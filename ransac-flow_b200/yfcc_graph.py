"""evalYFCC's pair (evaluation/evalYFCC/evaluation.py:179-274) from CUDA graphs, with one host read inside the pair (DESIGN §9).

  * search : the 11-image trunk, the four rotations' background maps, masked re-matchings and RANSAC calls, and
             ``rf_yfcc_rotation_select``, which writes one int32 record (winner, scores, rotations that drew, error flag,
             orientation class);
  * loop   : one per orientation class (0 / 180 degrees share the resized target's shape, 90 / 270 the transposed one): the
             winner's target, raw conv4 rows and background map copied by device index into static buffers, then
             ``maxCoarse + 1`` unconditional hypotheses gated by a device ``alive`` flag (``pipeline._hypothesis_loop``).

The host reads the search record, raises utils/outil.py:162's ``TypeError`` on its error flag, and otherwise runs the loop of
the winner's class.  RANSAC samples: the search draws T = 4 + maxCoarse + 1 tables up front, one ``ops.philox_words`` call
each, so table j is the j-th draw the eager path makes from the same generator state; a device slot chain
(``rf_ransac_homography_drawn``) hands each RANSAC call the table the reference would have drawn for it, also after calls
that drew nothing (fewer than 4 matches).  The generator advances by T tables per pair.
"""
import ctypes as C

import numpy as np
import torch

from . import ops, pipeline
from ._lib import check, lib, need_cuda, ptr, stream
from .ops import Ragged

REC_WINNER, REC_SCORES, REC_DRAWN, REC_ERROR, REC_CLASS, REC_WORDS = 0, 1, 5, 6, 7, 8     # include/ransacflow_b200.h


# --------------------------------------------------------------------------- kernel entries
def ransac_homography_drawn(match1, match2, tables, slot_in, slot_out, tolerance, M_dev, sample_mode, chunk=100):
    """``ops.ransac_homography`` on table ``*slot_in`` of ``tables`` (T, nbIter, 4) int64; writes ``*slot_out = *slot_in +
    (M >= 4)``.  ``slot_in`` / ``slot_out``: two different one-element int32 CUDA tensors.  Returns (H [9], nbInlier [1],
    mask [M], status [1])."""
    need_cuda(match1, match2, tables, slot_in, slot_out, M_dev)
    if tables.dim() != 3 or tables.shape[2] != 4 or tables.dtype != torch.int64 or not tables.is_contiguous():
        raise ValueError("ransac_homography_drawn: tables must be a contiguous (T, nbIter, 4) int64 tensor")
    for t in (slot_in, slot_out):
        if t.dtype != torch.int32 or t.numel() != 1:
            raise ValueError("ransac_homography_drawn: slots must be one int32 each")
    M = match1.shape[0]
    T, nbIter = int(tables.shape[0]), int(tables.shape[1])
    dev = match1.device
    H = torch.empty(9, device=dev, dtype=torch.float32)
    nb = torch.empty(1, device=dev, dtype=torch.int64)
    mask = torch.empty(max(M, 1), device=dev, dtype=torch.uint8)
    status = torch.empty(1, device=dev, dtype=torch.int32)
    wsz = lib.rf_ransac_workspace(nbIter)
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_ransac_homography_drawn(ptr(match1), ptr(match2), M, ptr(M_dev), ptr(tables), T, int(sample_mode), nbIter,
                                         float(tolerance), int(chunk), ptr(slot_in), ptr(slot_out), ptr(H), ptr(nb), ptr(mask),
                                         ptr(status), ptr(ws), wsz, stream()))
    return H, nb, mask[:M], status


def rotation_select(status, counts, masks, nbPoint=4, rec=None):
    """``rf_yfcc_rotation_select`` over four rotations: ``status`` / ``counts`` one int32 each, ``masks`` u8 inlier masks (their
    length bounds the count).  Returns ``rec`` (int32 [REC_WORDS], allocated when None)."""
    need_cuda(*status, *counts, *masks, rec)
    if not (len(status) == len(counts) == len(masks) == 4):
        raise ValueError("rotation_select: four rotations")
    for s, n, m in zip(status, counts, masks):
        if s.dtype != torch.int32 or n.dtype != torch.int32 or m.dtype != torch.uint8 or not m.is_contiguous():
            raise ValueError("rotation_select: int32 status / count and contiguous uint8 masks")
    if rec is None:
        rec = torch.empty(REC_WORDS, device=status[0].device, dtype=torch.int32)
    arr = lambda ts: (C.c_void_p * 4)(*[t.data_ptr() for t in ts])
    caps = (C.c_int * 4)(*[int(m.numel()) for m in masks])
    check(lib.rf_yfcc_rotation_select(arr(status), arr(counts), arr(masks), caps, int(nbPoint), ptr(rec), stream()))
    return rec


def select_copy(srcs, sel, dst):
    """``dst <- srcs[sel[0]]`` with the index read on the device (``rf_select_copy``); a None source copies nothing.  Every
    source has ``dst``'s size in bytes."""
    need_cuda(sel, dst, *[s for s in srcs if s is not None])
    nbytes = dst.numel() * dst.element_size()
    if not dst.is_contiguous() or not (1 <= len(srcs) <= 4) or sel.dtype != torch.int32:
        raise ValueError("select_copy: contiguous dst, 1 to 4 sources, an int32 index")
    for s in srcs:
        if s is not None and (not s.is_contiguous() or s.numel() * s.element_size() != nbytes):
            raise ValueError("select_copy: every source must be contiguous and of dst's size")
    src = (C.c_void_p * len(srcs))(*[None if s is None else s.data_ptr() for s in srcs])
    check(lib.rf_select_copy(src, len(srcs), ptr(sel), ptr(dst), nbytes, stream()))
    return dst


# --------------------------------------------------------------------------- sample tables
class DrawnTables:
    """The T sample tables of one pair and their slot chain: call i of the pair reads ``slots[i]`` and writes ``slots[i + 1]``.
    ``samples`` None: T ``ops.philox_words`` draws from ``generator`` (the reference's stream, ``SAMPLES_PHILOX64``); else a
    list of injected (nbIter, 4) tables, one per RANSAC call that draws in the reference's order (``SAMPLES_MOD``), padded with
    zeros (a call past the reference's last draw has fewer than 4 matches and reads nothing)."""

    def __init__(self, nbIter, nbPoint, T, device, generator=None, samples=None):
        if samples is None:
            self.tables = torch.empty((T, nbIter, nbPoint), dtype=torch.int64, device=device)
            for j in range(T):
                ops.philox_words(nbIter, nbPoint, device, generator, out=self.tables[j])
            self.mode = ops.SAMPLES_PHILOX64
        else:
            given = [np.asarray(s, dtype=np.int64) for s in samples][:T]
            n = given[0].shape[0] if given else nbIter
            host = np.zeros((T, n, nbPoint), dtype=np.int64)
            for j, s in enumerate(given):
                host[j] = s
            self.tables = torch.from_numpy(host).to(device)
            self.mode = ops.SAMPLES_MOD
        self.slots = torch.zeros(T + 1, dtype=torch.int32, device=device)

    def call(self, i):
        return _DrawnCall(self, i)


class _DrawnCall:
    """One RANSAC call of a slot chain, given to ``getCoarse_device`` / ``_ransac_device`` as its ``samples``."""

    def __init__(self, tables, i):
        self.t, self.i = tables, i

    def ransac(self, match1, match2, cnt, tolerance, chunk):
        s = self.t.slots
        return ransac_homography_drawn(match1, match2, self.t.tables, s[self.i:self.i + 1], s[self.i + 1:self.i + 2], tolerance, cnt,
                                       self.t.mode, chunk)


def slot_chain(counts, nbPoint=4):
    """The table every call of a chain reads, restated on the host: call i reads slot i, slot i + 1 = slot i + (M_i >= nbPoint)."""
    slots = [0]
    for m in counts:
        slots.append(slots[-1] + (1 if int(m) >= nbPoint else 0))
    return slots[:-1]


def orientation_classes(sizes):
    """The rotations each loop class serves, given the four rotated targets' (w, h): class c holds the rotations with rotation
    c's shape (0 / 180 and 90 / 270 degrees; all four for a square target)."""
    return {cls: [k for k in range(4) if tuple(sizes[k]) == tuple(sizes[cls])] for cls in (0, 1)}


# --------------------------------------------------------------------------- the two halves of a pair
_SRC_ATTRS = ("IsTensor", "_feats_rows", "featsMultiScale", "_src_planes", "WMultiScale", "HMultiScale", "_srcN", "_Is")


def _search_device(c, Is_u8, It_u8, maxCoarse, It_bg=None, segNet=False, samples=None):
    """The rotation search with no host read (evaluation.py:191-212): everything queued on the current stream.  ``It_bg``: a
    float32 (H, W) CUDA map of the unrotated target (``skyFromSeg``), or None; ``segNet``: segNet's map of ``It_u8`` instead.
    Returns the state the loop reads: the select record, the sample tables, the rotations' images / raw features /
    background maps, the source's features and the rotations each loop class serves."""
    c._set_rotated_pair(Is_u8, It_u8)
    dev = It_u8.device
    if segNet:
        It_bg = pipeline._require_segnet(c).run(It_u8)[0]
    draws = DrawnTables(c.nbIter, c.nbPoint, 4 + maxCoarse + 1, dev, c.sample_generator, samples)
    bgs, found = [], []
    for k in range(4):
        c._select_target(k)
        bg, Mt = pipeline._rotation_mask(It_bg, k, c.rotated_target_size(k))
        m1, m2, _, cnt = c._match_device(Mt)
        _, _, mask, status = draws.call(k).ransac(m1, m2, cnt, c.tolerance, 100)
        bgs.append(bg)
        found.append((status, cnt, mask, m1, m2))
    rec = rotation_select([f[0] for f in found], [f[1] for f in found], [f[2] for f in found], c.nbPoint)
    sizes = [c.rotated_target_size(k) for k in range(4)]
    classes = orientation_classes(sizes)
    return dict(rec=rec, draws=draws, rot=list(c._rot), bgs=bgs, found=found, sizes=sizes, classes=classes,
                src={a: c.__dict__[a] for a in _SRC_ATTRS if a in c.__dict__})


def _loop_device(c, network, S, cls, maxCoarse, maskRegionTh):
    """The hypothesis loop on the winner of ``S`` (``_search_device``), for the rotations of orientation class ``cls``: the
    winner's uint8 target, raw conv4 rows and background map are copied by the record's device index into buffers of this
    loop, then ``pipeline._hypothesis_loop`` runs ``maxCoarse + 1`` hypotheses, RANSAC calls 4.. of the slot chain.  Returns
    the packed records, the background map (or None), the target size (h, w), the flowDown8 shape and the loop's copies of the
    winner (``u8``, ``raw``: a captured loop writes them on every replay, so they live as long as this dict)."""
    ks = S["classes"][cls]
    k0 = ks[0]
    c.__dict__.update(S["src"])
    sel = S["rec"][REC_WINNER:REC_WINNER + 1]

    def take(bufs):
        dst = torch.empty_like(bufs[k0], memory_format=torch.contiguous_format)
        return select_copy([bufs[k] if k in ks else None for k in range(4)], sel, dst)
    u8 = take([r["u8"] for r in S["rot"]])
    raw = take([r["raw"].data for r in S["rot"]])
    bg = take(S["bgs"]) if S["bgs"][0] is not None else None
    c._set_static_target(u8, Ragged(raw, S["rot"][k0]["raw"].hw))
    recs, f8shape = pipeline._hypothesis_loop(c, network, maxCoarse, maskRegionTh, True, bg,
                                              [S["draws"].call(4 + k) for k in range(maxCoarse + 1)], region64=True)
    w, h = S["sizes"][k0]
    return dict(packed=torch.cat(recs), bg=bg, size=(h, w), f8shape=f8shape, u8=u8, raw=raw)


def _loop_pair(L):
    """A ``_loop_device`` result as the ``pipeline.DevicePair`` it is (no maps; ``bg`` the float32 background map or None)."""
    return pipeline.DevicePair(L["packed"], None, L["size"], L["f8shape"], L["bg"])


def unpack_record(rec):
    """The select record as (winner, the four scores, rotations that drew, error flag, orientation class) host ints."""
    rec = np.asarray(rec).reshape(-1)
    return (int(rec[REC_WINNER]), [int(v) for v in rec[REC_SCORES:REC_SCORES + 4]], int(rec[REC_DRAWN]), bool(rec[REC_ERROR]),
            int(rec[REC_CLASS]))


def _raise_on_error(rec):
    if unpack_record(rec)[3]:
        raise TypeError("'NoneType' object is not subscriptable")     # utils/outil.py:162 in the rotation search


def _result(rec, host, bg_host, size, f8shape, maxCoarse):
    """``align_pair_yfcc``'s dict (without the full-resolution maps) from the search's select record and the loop's records
    and background map."""
    winner, scores, _, _, _ = unpack_record(rec)
    out = pipeline._unpack_multi(host, size, f8shape, maxCoarse + 1, bg_host)
    out.setdefault("It_bg", np.ones(size, dtype=bool))
    out.update(angle=pipeline.YFCC_ANGLES[winner], nbInlierRot=scores)
    return out


def align_pair_yfcc_graph(coarseModel, network, Is, It, maxCoarse=10, maskRegionTh=0.01, segNet=False, It_bg=None, samples=None):
    """``align_pair_yfcc`` as the graphed path runs it, eagerly: the search queued with no host read, ONE read of its record,
    then the loop of the winner's orientation class, then one read of the loop's records.  Returns ``align_pair_yfcc``'s dict
    (H, flowDown8, matchDown8, nbMatch, angle, nbInlierRot, It_bg; ``flow12`` / ``match`` empty: the full-resolution maps stay
    on the device, as in ``align_pair_multi``).  ``Is`` / ``It``: PIL images, numpy arrays or uint8 (H, W, 3) tensors.
    ``segNet``: segNet's map of ``It`` masks the sky (a ``coarseModel`` built with ``segNet=True``); ``It_bg``: such a map
    given instead (float32 (H, W), CUDA or host).  ``samples``: injected (nbIter, 4) tables, one per RANSAC call that draws, in
    the reference's order.  Under ``torch.manual_seed(s)`` the pair equals ``align_pair_yfcc``'s; the generator then stands
    T = 4 + maxCoarse + 1 tables further on, not where the reference's would."""
    c = coarseModel
    with torch.no_grad():
        if It_bg is not None and not torch.is_tensor(It_bg):
            It_bg = torch.from_numpy(np.ascontiguousarray(It_bg, dtype=np.float32))
        if It_bg is not None and not It_bg.is_cuda:
            It_bg = It_bg.to(torch.device("cuda", torch.cuda.current_device()))
        S = _search_device(c, pipeline._as_device_u8(c, Is), pipeline._as_device_u8(c, It), maxCoarse, It_bg, segNet, samples)
        sel = pipeline._to_host(S["rec"]).copy()
        _raise_on_error(sel)
        L = _loop_device(c, network, S, unpack_record(sel)[4], maxCoarse, maskRegionTh)
        host, bg = pipeline._read_back(_loop_pair(L))
    return _result(sel, host, bg, L["size"], L["f8shape"], maxCoarse)


class GraphedYfccAligner(pipeline.GraphedAligner):
    """evalYFCC's pair as CUDA graphs per (source shape, target shape[, background shape]): the search graph and one loop graph
    per orientation class (one for a square target), sharing one memory pool and held by one LRU record.  ``enqueue`` replays
    the search graph, waits for its record alone, replays the loop graph of the winner's class and queues the D2H of its
    records; ``fetch`` returns ``align_pair_yfcc_graph``'s dict (``copy`` is accepted for the lanes' interface: no device map
    is returned).  ``It_bg`` (``prepare`` / ``enqueue`` / call): a float32 (H, W) background map of the target instead of
    segNet's.  It can be a ``ConcurrentAligner`` lane (``make_aligner``)."""

    def __init__(self, coarseModel, network, maxCoarse=10, maskRegionTh=0.01, segNet=False, warmup=2, max_graphs=4):
        """``segNet``: segNet's map of the target masks the sky inside the search graph (``align_pair_yfcc_graph(segNet=True)``)."""
        if segNet:
            pipeline._require_segnet(coarseModel)
        super().__init__(coarseModel, network, with_match21=True, warmup=warmup, max_graphs=max_graphs)
        self.maxCoarse, self.maskRegionTh, self.segNet = int(maxCoarse), maskRegionTh, bool(segNet)

    def _unpack(self, host, bg, maps, size, shapes, sel):
        return _result(sel, host, bg, size, shapes, self.maxCoarse)

    def _build(self, s_in, t_in, bg_in):
        search = lambda: _search_device(self.coarse, s_in, t_in, self.maxCoarse, bg_in, self.segNet)
        loop = lambda S, cls: _loop_device(self.coarse, self.net, S, cls, self.maxCoarse, self.maskRegionTh)

        def warm():
            S = search()
            for cls in sorted({min(S["classes"][c]) for c in (0, 1)}):          # one loop for a square target
                S["rec"][REC_WINNER].fill_(cls)                                # the selection forced to this class
                loop(S, cls)
        self.warm(warm)
        g, S, n_search = self.capture(search)
        loops, class_map = {}, {}
        for cls in (0, 1):
            first = min(S["classes"][cls])                      # the class of a square target's rotations 1 and 3 is 0's
            if first not in loops:
                gl, L, n = self.capture(lambda: loop(S, cls), pool=g.pool())
                loops[first] = dict(L, graph=gl, pair=_loop_pair(L), n_kernels=n)
            class_map[cls] = first
        return dict(graph=g, S=S, loops=loops, class_map=class_map, n_kernels=n_search,
                    host_rec=torch.empty(REC_WORDS, dtype=torch.int32).pin_memory())

    def enqueue(self, Is, It, It_bg=None):
        """Queue one pair on the CURRENT stream: input copies, the search graph, a D2H of its record and a wait for it (the one
        host read inside the pair; ``TypeError`` when RANSAC found no model in a rotation that drew), the loop graph of the
        winner's class and the D2H of its records.  Returns a ticket for ``fetch``."""
        c = self._replay(Is, It, It_bg)
        c["host_rec"].copy_(c["S"]["rec"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        sel = c["host_rec"].numpy().copy()
        _raise_on_error(sel)
        L = c["loops"][c["class_map"][unpack_record(sel)[4]]]
        L["graph"].replay()
        self.replayed_kernels += L["n_kernels"]
        return self._queue(L, sel)
