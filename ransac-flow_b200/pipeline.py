"""The per-pair path above the modules: ``PredFlowMask`` and the multi-hypothesis driver
loop of the evaluation scripts, and ``getFlow_all`` / ``getFlow`` of the getResults scripts,
restated on the library's kernels (no file IO, no metrics: those stay in the drivers).

  PredFlowMask : evaluation/evalHpatch/evaluation.py:23-55, evaluation/evalCorr/evaluation.py:29-59
  align_pair   : evaluation/evalHpatch/evaluation.py:172-243
  getFlow_all  : evaluation/evalHpatch/getResults.py:16-63 (after the np.load calls)
  KITTI        : evaluation/evalKITTI/evaluation.py:49-100,216-344 (two-level flow, small connected components),
                 evaluation/evalKITTI/getResults.py:95-141 (two-level recomposition)
"""
from typing import NamedTuple

import numpy as np
import torch

from . import _lib, model, ops, program
from .kornia_geometry import HomographyWarper
from .ops import Ragged


def base_grid(h, w, device="cuda"):
    """evaluation/evalHpatch/evaluation.py:187-189."""
    gy = torch.linspace(-1, 1, steps=h, device=device).view(1, -1, 1, 1).expand(1, h, w, 1)
    gx = torch.linspace(-1, 1, steps=w, device=device).view(1, 1, -1, 1).expand(1, h, w, 1)
    return torch.cat((gx, gy), dim=3).contiguous()


def fine_features(netFeatCoarse, img):
    """F.normalize(netFeatCoarse(img)) as a Ragged (rows = pixels)."""
    f = netFeatCoarse.forward_ragged(Ragged.from_nchw(img))
    return Ragged(ops.l2norm(f.data), f.hw)


def _fine_corr(network, IsSample, ItSample, featt, feat_box):
    """The fine features of the warped source and the target and their correlation pair: (corr12, [corr12 ; corr21], held).
    ``featt = None``: both images' features in one two-image batch (twice the tiles per FeatureExtractor launch, half the
    launches), the target's handed to ``feat_box`` (a dict, or None) for the next hypotheses; else the target's cached
    features (a Ragged or the reference's (1,256,h8,w8) tensor) and the source's alone.  ``held``: the features and volumes
    behind the pair, which the caller keeps until its heads have run (when they are freed sets the layout, and so the size,
    of a captured graph's memory pool)."""
    if featt is None:
        f = fine_features(network["netFeatCoarse"], torch.cat([IsSample, ItSample], dim=0))
        n = f.data.shape[0] // 2
        fs, ft = Ragged(f.data[:n], f.hw[:1]), Ragged(f.data[n:], f.hw[1:])
        if feat_box is not None:
            feat_box["featt"] = ft
    else:
        fs = fine_features(network["netFeatCoarse"], IsSample)
        ft = featt if isinstance(featt, Ragged) else Ragged.from_nchw(featt)
    k, ld = network["netCorr"].kernelSize, network["netFlowCoarse"].CORR_LD
    tc = model.fine_engine()            # 0 plain fp32, 1 TF32-rounded, 2 fp16, 4 split planes: the operand type of the heads
    if tc == ops.ENGINE_SPLIT:          # one launch: corr12 standalone + the two-image [corr12 ; corr21] tensor, split planes
        corr = ops.corr_neigh_pair_split(ft, fs, k, ld)
    else:                               # both volumes from one launch, already laid out as the two-image batch
        corr = ops.corr_neigh_pair(ft, fs, k, ld, tc)
    return corr[0], corr[-1], (fs, ft, corr)


def PredFlowMask_device(IsTensor, featt, flowCoarse, size, network, with_match21=False, align_corners=False, ItTensor=None, feat_box=None):
    """PredFlowMask without the device->host copies: returns CUDA tensors
    (flow12 (1,H,W,2), match (1,1,H,W), flowDown8 (1,2,h8,w8), matchDown8 (2,1,h8,w8) = [match12, match21]).
    ``featt = None`` with ``ItTensor``: the target's fine features are computed HERE, in one two-image batch with the warped
    source's (twice the tiles per FeatureExtractor launch, half the launches);
    ``feat_box`` (a dict) receives them for the next hypotheses."""
    with torch.no_grad():
        IsSample = ops.grid_sample(IsTensor, flowCoarse, align_corners)
        corr12, both, _held = _fine_corr(network, IsSample, ItTensor, featt, feat_box)
        # the two heads are independent: the flow head (one image: 152 tiles in its widest layer, more than one wave on 132
        # SMs) runs on the side stream and fills the tails of the matchability head's kernels (two images) and vice versa
        main, side = torch.cuda.current_stream(), _side_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            flowDown8 = network["netFlowCoarse"].forward_ragged(corr12)
        corr12.data.record_stream(side)
        mboth = network["netMatch"].forward_ragged(both)                    # (2,1,h8,w8): match12, match21 in one batch
        main.wait_stream(side)
        flowDown8.record_stream(main)
        flow12, match, _ = ops.compose_fine(flowDown8, mboth[0:1], mboth[1:2] if with_match21 else None, flowCoarse,
                                            clamp=True, align_corners=align_corners)
        return flow12, match, flowDown8, mboth


def PredFlowMask(IsTensor, featt, flowCoarse, grid, network, with_match21=False, align_corners=False):
    """Same inputs/outputs as the reference function (evaluation/evalHpatch/evaluation.py:23-55; ``with_match21``:
    evaluation/evalCorr/evaluation.py:54).  ``featt`` may be the (1,256,h8,w8) tensor the reference passes or a Ragged
    from ``fine_features``.  ``grid`` is only used for its size (the base grid is regenerated inside the fused
    composition kernel)."""
    H, W = grid.size()[1], grid.size()[2]
    flow12, match, flowDown8, mboth = PredFlowMask_device(IsTensor, featt, flowCoarse, (H, W), network, with_match21, align_corners)
    out = torch.cat([match.reshape(-1), flowDown8.reshape(-1), mboth.reshape(-1)]).cpu().numpy()   # one D2H
    n0, n1 = H * W, flowDown8.numel()
    return (flow12, out[:n0].reshape(H, W), out[n0:n0 + n1].reshape(tuple(flowDown8.shape)),
            out[n0 + n1:].reshape(1, 2, flowDown8.shape[2], flowDown8.shape[3]))


_pinned = {}
_side = {}


def _side_stream():
    d = torch.cuda.current_device()
    if d not in _side:
        _side[d] = torch.cuda.Stream(device=d)
    return _side[d]


def _to_host(t):
    """One asynchronous D2H into a cached pinned buffer + a stream synchronise."""
    key = (t.numel(), t.dtype)
    if key not in _pinned:
        _pinned[key] = torch.empty(t.numel(), dtype=t.dtype).pin_memory()
    h = _pinned[key]
    h.copy_(t.reshape(-1), non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return h.numpy()


class DevicePair(NamedTuple):
    """One pair's results as its device path leaves them, nothing read back: ``packed`` the records the host reads, ``maps``
    the device tensors handed to the caller (or None), ``size`` the target's (h, w), ``shapes`` the shapes the host needs to
    cut the records, ``bg`` the device background map (None without one)."""
    packed: torch.Tensor
    maps: object
    size: tuple
    shapes: tuple
    bg: object = None


def _read_back(pair):
    """The end of an eager entry point: one pinned D2H of the records and one of the background map (None without one)."""
    return _to_host(pair.packed).copy(), None if pair.bg is None else _to_host(pair.bg).copy()


def _single_device(coarseModel, network, Is, It, with_match21, samples=None):
    """Device part of the single-hypothesis path: everything queued on the current stream, nothing read back."""
    coarseModel.setPair(Is, It)
    Itw, Ith = coarseModel.target_size
    Hd, nb, mask, status, cnt = coarseModel.getCoarse_device(None, samples)
    flowCoarse = ops.warp_grid(Hd.view(1, 3, 3), Ith, Itw)
    # target and warped source through the FeatureExtractor as one two-image batch (bit-identical features)
    flow12, match, f8, mboth = PredFlowMask_device(coarseModel.IsTensor, None, flowCoarse, (Ith, Itw), network, with_match21,
                                                   ItTensor=coarseModel.ItTensor)
    packed = torch.cat([status.float(), cnt.float(), nb.float(), Hd, match.reshape(-1), f8.reshape(-1), mboth.reshape(-1)])
    return DevicePair(packed, flow12, (Ith, Itw), tuple(f8.shape))


def _unpack_single(host, flow12, size, f8shape):
    """The host side of ``_single_device``: ``align_pair_single``'s dict."""
    Ith, Itw = size
    st, n0, n8 = int(host[0]), Ith * Itw, int(np.prod(f8shape))
    if st != 0:                                    # the reference's `if bestPara is None: break` (evaluation.py:215-216)
        if st == 2:
            raise TypeError("'NoneType' object is not subscriptable")     # utils/outil.py:162
        return dict(H=np.zeros((0,)), flowDown8=np.zeros((0,)), matchDown8=np.zeros((0,)), flow12=[], match=[],
                    nbInlier=0, nbMatch=int(host[1]))
    H = host[3:12].reshape(1, 3, 3).astype(np.float32)
    o = 12
    return dict(H=H, flowDown8=host[o + n0:o + n0 + n8].reshape(f8shape),
                matchDown8=host[o + n0 + n8:].reshape(1, 2, f8shape[2], f8shape[3]),
                flow12=[flow12], match=[host[o:o + n0].reshape(Ith, Itw)], nbInlier=int(host[2]), nbMatch=int(host[1]))


def align_pair_single(coarseModel, network, Is, It, with_match21=False, samples=None):
    """The single-hypothesis case of the evaluation loop (maxCoarse = 0, no background mask) with NO host
    synchronisation until the results are fetched: matching, RANSAC (device-side match count), warp, fine flow and
    composition are queued back to back, then one pinned D2H brings back status, H, the matchability map and the /8
    tensors.  Same outputs as ``align_pair``; under ``torch.manual_seed(s)`` also the same RANSAC samples (the reference's
    stream, ``ops.philox_words``).  ``samples``: an injected (nbIter, 4) index table instead."""
    pair = _single_device(coarseModel, network, Is, It, with_match21, samples)
    return _unpack_single(_read_back(pair)[0], pair.maps, pair.size, pair.shapes)


def _as_tensor(a):
    return torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray) else a


def _clone(maps):
    """A copy of a result's device maps: a tensor, a list of (flow, match) tensors, or None."""
    if torch.is_tensor(maps):
        return maps.clone()
    return None if maps is None else [tuple(t.clone() for t in m) for m in maps]


class GraphedAligner:
    """``align_pair_single`` captured once in a CUDA graph per input size and replayed per pair: the ~140 kernel
    launches of a pair (pyramid, ResNet-50 trunk, matching, RANSAC, fine flow) cost one graph launch on the host.
    Inputs are copied into static device buffers (H2D when they are host tensors / arrays); the RANSAC samples are
    drawn inside the graph (torch's graph-safe Philox offsets), so successive replays use fresh samples.

    It is also the capture core of the other graphed pairs: a subclass gives the device work of its pair (``_device``,
    returning a ``DevicePair``) and its host unpacking (``_unpack``), or builds its own graphs from ``warm`` and ``capture``.
    Each record pins the layer-program entries its graphs point into; evicting it unpins them, and an entry goes with its
    last pin, whichever aligner holds the other graphs that point into it."""

    def __init__(self, coarseModel, network, with_match21=False, warmup=2, max_graphs=8):
        self.coarse, self.net, self.m21, self.warmup = coarseModel, network, with_match21, warmup
        self.coarse.device_preproc = True
        self.graphs = {}                # insertion-ordered: least recently used first
        self.max_graphs = max_graphs    # datasets with many image sizes (HPatches, MegaDepth, YFCC): LRU-bounded graph memory
        self.replayed_kernels = 0       # library kernels executed through graph replays (they bypass rf_launch_count)
        self.generator = None           # RANSAC sample stream: torch's default CUDA generator (the reference's stream)
        self._entries = set()           # (program, key) the graphs of the record being built point into

    def use_generator(self, generator):
        """Draw this aligner's RANSAC samples from ``generator`` (a CUDA torch.Generator of its own) instead of torch's default
        generator.  A replay copies its generator's seed and offset into device memory that the graph reads; graphs replayed
        concurrently on several streams must therefore not share a generator.  Call before the first graph is captured."""
        assert not self.graphs, "use_generator: graphs already captured with another generator"
        self.generator = generator
        self.coarse.sample_generator = generator

    def _device(self, s_in, t_in):
        """The device work of one pair, queued on the current stream: a ``DevicePair``."""
        return _single_device(self.coarse, self.net, s_in, t_in, self.m21)

    def _unpack(self, host, bg, maps, size, shapes):
        """The pair's dict from its host records, host background map (None without one) and device maps."""
        return _unpack_single(host, maps, size, shapes)

    def warm(self, fn):
        """``warmup`` eager runs of ``fn()`` on a side stream (function attributes, TMA maps, caches, layer programs: nothing a
        capture may do first), then a device barrier."""
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.no_grad(), torch.cuda.stream(side):
            for _ in range(self.warmup):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()

    def capture(self, fn, pool=None):
        """``fn()`` captured in a new CUDA graph (in the memory pool ``pool`` when given) that replays draw from this aligner's
        generator.  The layer-program entries the graph points into join those the record being built pins.  Returns (graph,
        ``fn()``'s result, library kernels in the graph)."""
        g = torch.cuda.CUDAGraph()
        if self.generator is not None:
            g.register_generator_state(self.generator)
        n0 = _lib.launch_count()
        with torch.no_grad(), program.recording() as used, torch.cuda.graph(g, pool=pool):
            res = fn()
        self._entries |= used
        return g, res, _lib.launch_count() - n0

    def _build(self, s_in, t_in, bg_in):
        """The record of one input size: the pair in one graph."""
        if bg_in is not None:
            raise TypeError("%s takes no background map" % type(self).__name__)
        self.warm(lambda: self._device(s_in, t_in))
        g, pair, n = self.capture(lambda: self._device(s_in, t_in))
        return dict(graph=g, pair=pair, flow12=pair.maps, n_kernels=n)      # flow12: the maps replays write (fetch's copy=False)

    def prepare(self, Is, It, It_bg=None):
        """Capture (once) the graphs for these input sizes, evicting the least recently used record beyond ``max_graphs``;
        returns their record."""
        inputs = [_as_tensor(a) for a in (Is, It, It_bg)]
        key = tuple(None if a is None else tuple(a.shape) for a in inputs)
        if key in self.graphs:
            self.graphs[key] = self.graphs.pop(key)            # most recently used last
            return self.graphs[key]
        while self.max_graphs and len(self.graphs) >= self.max_graphs:
            self._evict()
        dev = torch.device("cuda", torch.cuda.current_device())
        dtypes = (torch.uint8, torch.uint8, torch.float32)             # Is, It, It_bg
        static = [None if a is None else torch.empty(tuple(a.shape), dtype=d, device=dev).copy_(a) for a, d in zip(inputs, dtypes)]
        self._entries = set()
        rec = self._build(*static)
        for p, k in self._entries:
            p.pin(k)
        rec.update(inputs=static, pins=self._entries, prog_keys={(id(p), k) for p, k in self._entries})
        self.graphs[key] = rec
        return rec

    def _evict(self):
        """Drop the least recently used record, and unpin the layer-program entries its graphs point into: an entry no other
        live graph pins goes with it (a graph holds raw pointers into the entries' buffers, so neither may outlive the other)."""
        torch.cuda.synchronize()
        rec = self.graphs.pop(next(iter(self.graphs)))
        for p, k in rec["pins"]:
            p.unpin(k)

    def _replay(self, Is, It, It_bg=None):
        """Copy the inputs into their record's static buffers and replay its graph on the current stream; returns the record."""
        inputs = [_as_tensor(a) for a in (Is, It, It_bg)]
        rec = self.prepare(*inputs)
        for buf, a in zip(rec["inputs"], inputs):
            if a is not None:
                buf.copy_(a, non_blocking=True)
        rec["graph"].replay()
        self.replayed_kernels += rec["n_kernels"]
        return rec

    def _queue(self, L, *ctx):
        """Queue the D2H of ``L["pair"]``'s records and background map into L's own pinned buffers; returns the ticket (``ctx``:
        what ``_unpack`` takes after the shapes)."""
        pair = L["pair"]
        if "host" not in L:
            L["host"] = torch.empty(pair.packed.numel(), dtype=pair.packed.dtype).pin_memory()
            L["host_bg"] = None if pair.bg is None else torch.empty(pair.bg.numel(), dtype=pair.bg.dtype).pin_memory()
        L["host"].copy_(pair.packed.reshape(-1), non_blocking=True)
        if pair.bg is not None:
            L["host_bg"].copy_(pair.bg.reshape(-1), non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        return (L, done, ctx)

    def enqueue(self, Is, It, It_bg=None):
        """Queue one pair on the CURRENT stream without waiting for it: input copies (H2D when the images are pinned host
        tensors), one graph replay, one D2H of the packed results into this aligner's own pinned buffer.  Returns a
        ticket for ``fetch``.  The ticket's buffers are reused by the next ``enqueue`` with the same sizes."""
        return self._queue(self._replay(Is, It, It_bg))

    def fetch(self, ticket, copy=True):
        """Wait for a ticket and unpack it (the dict of the eager entry point: ``align_pair_single``'s here).  The device maps
        (``flow12``; KITTI's ``maps``) are the graph's static output buffers: they are cloned so that results collected over
        several replays stay valid (``copy=False`` returns the live buffers, overwritten by the next replay with these input
        sizes)."""
        L, done, ctx = ticket
        done.synchronize()
        pair = L["pair"]
        bg = None if pair.bg is None else L["host_bg"].numpy()
        return self._unpack(L["host"].numpy().copy(), bg, _clone(pair.maps) if copy else pair.maps, pair.size, pair.shapes, *ctx)

    def __call__(self, Is, It, copy=True, It_bg=None):
        """Is, It: uint8 (H, W, 3) torch tensors (CUDA, or pinned host for an asynchronous H2D) or numpy arrays.  ``It_bg``: a
        float32 (H, W) background map of the target, for the aligners that take one (``GraphedYfccAligner``)."""
        return self.fetch(self.enqueue(Is, It, It_bg), copy)


def _require_segnet(coarseModel):
    """``coarseModel``'s segNet; ``skyFromSeg``'s NotImplementedError without one."""
    seg = getattr(coarseModel, "segNet", None)
    if seg is None:
        raise NotImplementedError("skyFromSeg needs a CoarseAlign built with segNet=True")
    return seg


def _sky_background(coarseModel, It):
    """evaluation/evalCorr/evaluation.py:184-189 on the device: segNet's mask of the original target ``It`` (a path, PIL image or
    uint8 (H, W, 3) CUDA tensor), resized to the resized target like ``imresize(It_bg, (h, w)) < 128``.  Returns the bool
    (h, w) CUDA map (True = kept).  Nothing is read back to the host."""
    Itw, Ith = coarseModel.target_size
    return ops.imresize_keep(_require_segnet(coarseModel).run(It)[0], Ith, Itw)


def _multi_device(coarseModel, network, Is, It, maxCoarse, maskRegionTh, with_match21, samples=None, segNet=False):
    """The multi-hypothesis loop of evaluation/evalCorr/evaluation.py:211-243 with NO host control at all: every one of the
    ``maxCoarse + 1`` iterations is queued unconditionally; what the reference decides on the host - stop at the first failed
    RANSAC (:215-216), stop at the first hypothesis whose new-region matchability mean is below ``maskRegionTh`` (:226), update
    the mask (:236) - becomes a device-side ``alive`` flag that gates the mask update, and the host drops the hypotheses
    after the first dead one when it unpacks.  Accepted hypotheses are computed from exactly the state the reference's loop
    would have had; dead ones are wasted work (none when every hypothesis is accepted, the common case at maxCoarse = 10).
    One packed result tensor: per hypothesis [alive, status, nbMatch, nbInlier, H(9), flowDown8, matchDown8] - the tensors
    the drivers save (evaluation.py:244-260); the full-resolution maps stay on the device and are not returned.
    ``segNet`` (the drivers' ``--segNet``): the background map of the target (``_sky_background``) masks every hypothesis,
    the first included (:211-243 with ``It_bg``); it is the pair's ``bg``, a bool (h, w) CUDA map (True = kept)."""
    coarseModel.setPair(Is, It)
    keep = _sky_background(coarseModel, It) if segNet else None
    bg = keep.float() if segNet else None
    recs, f8shape = _hypothesis_loop(coarseModel, network, maxCoarse, maskRegionTh, with_match21, bg, samples)
    Itw, Ith = coarseModel.target_size
    return DevicePair(torch.cat(recs), None, (Ith, Itw), f8shape, keep)


def _hypothesis_loop(coarseModel, network, maxCoarse, maskRegionTh, with_match21, bg, samples, region64=False):
    """The ``maxCoarse + 1`` unconditional iterations of ``_multi_device`` on the target ``coarseModel`` currently holds, masked
    with ``bg`` (a float (h, w) CUDA map, 1 = kept; None: nothing masked).  ``samples[k]``: what hypothesis k's ``getCoarse_device``
    draws from (None: the generator).  ``region64``: the acceptance test compares the new-region mean with ``maskRegionTh`` in
    float64, as the host-steered loop does once the mean is on the host.  Returns (per-hypothesis records, flowDown8 shape)."""
    Itw, Ith = coarseModel.target_size
    dev = coarseModel.ItTensor.device
    Mask = torch.zeros((Ith, Itw), device=dev)
    alive = torch.ones((), device=dev, dtype=torch.bool)
    recs, featt, f8shape, box = [], None, None, {}
    for k in range(maxCoarse + 1):
        Mask, alive, featt, rec, f8shape = _hypothesis_step(coarseModel, network, k, Mask, alive, bg, featt, box, maskRegionTh,
                                                            with_match21, None if samples is None else samples[k], region64)
        recs.append(rec)
    return recs, f8shape


def _hypothesis_step(coarseModel, network, k, Mask, alive, bg, featt, box, maskRegionTh, with_match21, samples, region64=False):
    """Hypothesis ``k`` of ``_hypothesis_loop``: getCoarse masked by (Mask, bg), the fine flow, the acceptance test and the mask
    update gated by the ``alive`` flag.  Returns (Mask, alive, the target's fine features, the record, flowDown8 shape)."""
    Itw, Ith = coarseModel.target_size
    dev = coarseModel.ItTensor.device
    if bg is None:
        fgMask = (Mask > 0.5).float()                                # It_bg = 1 everywhere: (Mask + (1 - It_bg)) > 0.5
    else:
        fgMask = ((Mask + (1 - bg)) > 0.5).float()
    Hd, nb, mask, status, cnt = coarseModel.getCoarse_device(fgMask if k > 0 or bg is not None else None, samples)
    flowCoarse = ops.warp_grid(Hd.view(1, 3, 3), Ith, Itw)
    flow12, match, f8, mboth = PredFlowMask_device(coarseModel.IsTensor, featt, flowCoarse, (Ith, Itw), network, with_match21,
                                                   ItTensor=coarseModel.ItTensor, feat_box=box)
    if featt is None:
        featt = box["featt"]            # computed with the first hypothesis' warped source in one batch
    newreg = (match[0, 0] * (1 - fgMask)).mean()
    found = status[0] == 0
    if k > 0:
        region = (newreg.double() > maskRegionTh) if region64 else (newreg > maskRegionTh)
    else:
        region = torch.ones((), device=dev, dtype=torch.bool)
    ok = found & region
    alive = alive & ok
    # (evaluation.py:235 masks from the first hypothesis on; without a background the first mask is all zeros)
    matchFine = match[0, 0] if (k == 0 and bg is None) else match[0, 0] * (1 - fgMask)
    Mask = torch.where(alive, ((Mask + matchFine) >= 1.0).float(), Mask)
    rec = torch.cat([alive.float().reshape(1), status.float(), cnt.float(), nb.float(), Hd, f8.reshape(-1), mboth.reshape(-1)])
    return Mask, alive, featt, rec, tuple(f8.shape)


# the per-hypothesis record of the device loops (multi-hypothesis, KITTI, YFCC): [alive, status, nbMatch, nbInlier, H(9), payload]
_ALIVE, _STATUS, _NBMATCH, _NBINLIER, _H, _PAYLOAD = 0, 1, 2, 3, slice(4, 13), 13


def _accepted(host, nhyp):
    """The ``nhyp`` records of a device loop -> (n, the records of the hypotheses before the first dead one).  A RANSAC without
    a model (status 2) in a hypothesis the reference reaches raises utils/outil.py:162's ``TypeError``."""
    rows = host.reshape(nhyp, -1)
    if any(rows[i, _STATUS] == 2 and rows[:i, _ALIVE].all() for i in range(nhyp)):
        raise TypeError("'NoneType' object is not subscriptable")          # utils/outil.py:162
    n = 0
    while n < nhyp and rows[n, _ALIVE] > 0.5:
        n += 1
    return n, rows[:n]


def _split(rows, shapes):
    """Accepted records -> [H (n,3,3) float32] + their payload cut into one (n,) + shape[1:] array per per-hypothesis shape;
    np.zeros((0,)) for each when no hypothesis was accepted."""
    if len(rows) == 0:
        return [np.zeros((0,)) for _ in range(1 + len(shapes))]
    out, o = [rows[:, _H].reshape(-1, 3, 3).astype(np.float32)], _PAYLOAD
    for shape in shapes:
        m = int(np.prod(shape))
        out.append(rows[:, o:o + m].reshape((len(rows),) + tuple(shape[1:])))
        o += m
    return out


def _counts(rows):
    return dict(nbMatch=[int(v) for v in rows[:, _NBMATCH]], nbInlier=[int(v) for v in rows[:, _NBINLIER]])


def _unpack_multi(host, size, f8shape, nhyp, bg=None):
    """The host side of ``_multi_device``: the hypotheses up to the first dead one, in ``align_pair_multi``'s dict."""
    n, rows = _accepted(host, nhyp)
    out = dict(flow12=[], match=[], **_counts(rows))
    out["H"], out["flowDown8"], out["matchDown8"] = _split(rows, [f8shape, (1, 2) + tuple(f8shape[2:])])
    if bg is not None:
        out["It_bg"] = bg.reshape(size).astype(bool)
    return out


def align_pair_multi(coarseModel, network, Is, It, maxCoarse=10, maskRegionTh=0.01, with_match21=True, samples=None, segNet=False):
    """``align_pair_device`` without any host round trip inside the loop (see ``_multi_device``): one pinned D2H at the end.
    Returns H / flowDown8 / matchDown8 / nbMatch / nbInlier of the accepted hypotheses (what the drivers save).  ``segNet``:
    the sky of the target is masked as the drivers' ``--segNet`` masks it (the ``coarseModel`` needs ``segNet=True``), and the
    result has ``It_bg``, the (h, w) bool background map the drivers save as ``maskBG_*``."""
    pair = _multi_device(coarseModel, network, Is, It, maxCoarse, maskRegionTh, with_match21, samples, segNet)
    host, bg = _read_back(pair)
    return _unpack_multi(host, pair.size, pair.shapes, maxCoarse + 1, bg)


class GraphedMultiAligner(GraphedAligner):
    """The whole multi-hypothesis pair (``align_pair_multi``: trunk, matching, ``maxCoarse + 1`` x (RANSAC, warp, fine flow,
    acceptance test, mask update)) as ONE CUDA graph per input size: ~0.6 k kernels per pair at maxCoarse = 10 with no host
    work between them.  BASELINE config 4 (evalCorr / evalYFCC semantics) is measured through it."""

    def __init__(self, coarseModel, network, maxCoarse=10, maskRegionTh=0.01, with_match21=True, warmup=2, max_graphs=4, segNet=False):
        """``segNet`` (the drivers' ``--segNet``): segNet and the background-map resize run inside the graph, every hypothesis
        is masked with the background, and ``fetch`` also returns ``It_bg`` (``align_pair_multi(segNet=True)``)."""
        if segNet:
            _require_segnet(coarseModel)
        super().__init__(coarseModel, network, with_match21=with_match21, warmup=warmup, max_graphs=max_graphs)
        self.maxCoarse, self.maskRegionTh, self.segNet = maxCoarse, maskRegionTh, bool(segNet)

    def _device(self, s_in, t_in):
        return _multi_device(self.coarse, self.net, s_in, t_in, self.maxCoarse, self.maskRegionTh, self.m21, segNet=self.segNet)

    def _unpack(self, host, bg, maps, size, shapes):
        return _unpack_multi(host, size, shapes, self.maxCoarse + 1, bg)


class ConcurrentAligner:
    """``lanes`` independent GraphedAligners (each with its OWN CoarseAlign state, network activations, graph memory,
    pinned result buffer and stream) replayed side by side: pairs are independent (SURVEY 8e), and a single pair leaves
    SMs idle in its small layers (the /16 grids of the trunk's late layers, the 60 x 80 heads, RANSAC), which the other
    lanes' kernels fill.  ``make_models()`` must return a fresh ``(coarseModel, network)`` per lane (layer programs cache
    their activation buffers per module, so lanes cannot share modules).  Every lane draws its RANSAC samples from a CUDA
    generator of its own (``seed``): what a pair returns depends on the seed and on the pair's position in the sequence
    given to the aligner, never on how the lanes' replays interleave in time."""

    def __init__(self, make_models, lanes=2, with_match21=False, make_aligner=None, seed=0):
        """``make_aligner(coarseModel, network)`` (optional): the per-lane aligner, e.g. a ``GraphedMultiAligner``."""
        mk = make_aligner or (lambda c, n: GraphedAligner(c, n, with_match21=with_match21))
        self.lanes = [mk(*make_models()) for _ in range(lanes)]
        self.streams = [torch.cuda.Stream() for _ in range(lanes)]
        for a in self.lanes:
            a.use_generator(torch.Generator(device=torch.device("cuda", torch.cuda.current_device())))
        self.seed(seed)

    def seed(self, s):
        """Restart the lanes' sample streams: lane k's generator is seeded with s + k."""
        for k, a in enumerate(self.lanes):
            a.generator.manual_seed(s + k)

    @property
    def replayed_kernels(self):
        return sum(a.replayed_kernels for a in self.lanes)

    def prepare(self, Is, It):
        for a in self.lanes:                      # graph capture is serial
            a.prepare(Is, It)
        torch.cuda.synchronize()

    def enqueue(self, pairs):
        """pairs: up to ``lanes`` (Is, It) tuples -> tickets; lane k runs on its own stream, ordered after the work
        already queued on the current stream."""
        assert len(pairs) <= len(self.lanes)
        main = torch.cuda.current_stream()
        tickets = []
        for a, s, (Is, It) in zip(self.lanes, self.streams, pairs):
            a.prepare(Is, It)
            s.wait_stream(main)
            with torch.cuda.stream(s):
                tickets.append(a.enqueue(Is, It))
        for s in self.streams[:len(pairs)]:
            main.wait_stream(s)                   # later work on the current stream (e.g. the next batch) follows all lanes
        return tickets

    def fetch(self, tickets, copy=True):
        return [a.fetch(t, copy) for a, t in zip(self.lanes, tickets)]

    def __call__(self, pairs, copy=True):
        return self.fetch(self.enqueue(pairs), copy)

    def run(self, pairs, copy=True):
        """Any number of pairs through the lanes WITHOUT a barrier between rounds: lane k is refilled as soon as its previous
        pair has been fetched, so the lanes drift apart instead of starting every round in lock-step (their tails and launch
        gaps then overlap each other's work).  Results in the order of ``pairs``.  With ``copy=False`` a result's ``flow12`` is
        valid only until its lane is refilled."""
        main = torch.cuda.current_stream()
        L = len(self.lanes)
        for s in self.streams:
            s.wait_stream(main)
        tickets, owner, out = [None] * L, [None] * L, [None] * len(pairs)
        for i, (Is, It) in enumerate(pairs):
            k = i % L
            if tickets[k] is not None:
                out[owner[k]] = self.lanes[k].fetch(tickets[k], copy)
            with torch.cuda.stream(self.streams[k]):
                tickets[k], owner[k] = self.lanes[k].enqueue(Is, It), i
        for k in range(L):
            if tickets[k] is not None:
                out[owner[k]] = self.lanes[k].fetch(tickets[k], copy)
        for s in self.streams:
            main.wait_stream(s)
        return out


def align_pair(coarseModel, network, Is, It, maxCoarse=0, maskRegionTh=0.01, with_match21=False, It_bg=None):
    """One pair through the evaluation loop (evaluation/evalHpatch/evaluation.py:172-243).
    Returns dict(H (nH,3,3), flowDown8 (nH,2,h8,w8), matchDown8 (nH,2,h8,w8), flow12 [..], match [..])."""
    coarseModel.setPair(Is, It)
    Itw, Ith = coarseModel.target_size
    if It_bg is None:
        It_bg = np.ones((Ith, Itw), dtype=np.float32)
    featt = fine_features(network["netFeatCoarse"], coarseModel.ItTensor)
    grid = torch.empty((1, Ith, Itw, 2), device="meta")                    # size carrier only
    warper = HomographyWarper(Ith, Itw)
    Mask = np.zeros((Ith, Itw), dtype=np.float32)
    Hs, flows8, matches8, flows, matches = [], [], [], [], []
    nbCoarse = 0
    while nbCoarse <= maxCoarse:
        fgMask = ((Mask + (1 - It_bg)) > 0.5).astype(np.float32)
        bestPara = coarseModel.getCoarse(fgMask)
        if bestPara is None:
            break
        bestParaT = torch.from_numpy(bestPara).unsqueeze(0).cuda()
        flowCoarse = warper.warp_grid(bestParaT)
        flowFine, matchFine, f8, m8 = PredFlowMask(coarseModel.IsTensor, featt, flowCoarse, grid, network, with_match21)
        if (matchFine * (1 - fgMask)).mean() > maskRegionTh or nbCoarse == 0:
            Hs.append(bestPara[None])
            flows8.append(f8)
            matches8.append(m8)
            flows.append(flowFine)
            matches.append(matchFine)
            nbCoarse += 1
            matchFine = matchFine if len(matches8) == 0 else matchFine * (1 - fgMask)
            Mask = ((Mask + matchFine) >= 1.0).astype(np.float32)
        else:
            break
    cat = lambda l: np.concatenate(l, axis=0) if l else np.zeros((0,))
    return dict(H=cat(Hs), flowDown8=cat(flows8), matchDown8=cat(matches8), flow12=flows, match=matches)


def align_pair_device(coarseModel, network, Is, It, maxCoarse=0, maskRegionTh=0.01, with_match21=False, It_bg=None, samples=None):
    """The multi-hypothesis loop of evaluation/evalHpatch/evaluation.py:211-243 with the masks kept on the device:
    per hypothesis only the two scalars the host needs to steer the loop (RANSAC status, new-region matchability mean)
    cross the bus instead of the full-resolution matchability map, and the accepted results are fetched once at the
    end.  Same outputs as ``align_pair`` (plus ``nbMatch`` per hypothesis), and under a seed the same RANSAC samples per
    hypothesis.  ``samples``: optional list of injected (nbIter, 4) index tables, one per ``getCoarse`` call."""
    coarseModel.setPair(Is, It)
    return _hypotheses_device(coarseModel, network, maxCoarse, maskRegionTh, with_match21, It_bg, samples)


def _hypotheses_device(coarseModel, network, maxCoarse, maskRegionTh, with_match21, It_bg, samples, rewind_too_few=False):
    """The hypothesis loop of ``align_pair_device`` on the pair / target ``coarseModel`` currently holds.
    ``rewind_too_few``: a ``getCoarse`` with fewer than 4 matches returns None before RANSAC draws its samples (variant B
    :179-180, utils/outil.py:120), so the generator state the device draw advanced is put back (the stream of the next pair
    is then the reference's)."""
    Itw, Ith = coarseModel.target_size
    dev = coarseModel.ItTensor.device
    bg = torch.ones((Ith, Itw), device=dev) if It_bg is None else torch.as_tensor(It_bg, dtype=torch.float32, device=dev)
    featt = fine_features(network["netFeatCoarse"], coarseModel.ItTensor)
    Mask = torch.zeros((Ith, Itw), device=dev)
    acc = []
    nbCoarse = ncall = 0
    gen = None
    if rewind_too_few and samples is None:
        gen = coarseModel.sample_generator or torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
    while nbCoarse <= maxCoarse:
        fgMask = ((Mask + (1 - bg)) > 0.5).float()
        state = gen.get_state() if gen is not None else None
        Hd, nb, mask, status, cnt = coarseModel.getCoarse_device(fgMask if nbCoarse > 0 or It_bg is not None else None,
                                                                 None if samples is None else samples[ncall])
        ncall += 1
        # the fine stage is queued before the status is known (no host round trip between RANSAC and the networks); a failed
        # RANSAC leaves H = 0, whose warp grid is NaN: harmless (the results are dropped below) and finite work
        flowCoarse = ops.warp_grid(Hd.view(1, 3, 3), Ith, Itw)
        flow12, match, f8, mboth = PredFlowMask_device(coarseModel.IsTensor, featt, flowCoarse, (Ith, Itw), network, with_match21)
        newreg = (match[0, 0] * (1 - fgMask)).mean()
        ctl = _to_host(torch.cat([status.float(), newreg.reshape(1), cnt.float()])).copy()        # 12 bytes per hypothesis
        st = int(ctl[0])
        if st == 2:
            raise TypeError("'NoneType' object is not subscriptable")     # utils/outil.py:162
        if st == 3 and state is not None:
            gen.set_state(state)
        if st != 0:
            break                                                          # bestPara is None (evaluation.py:215-216)
        if float(ctl[1]) > maskRegionTh or nbCoarse == 0:
            acc.append((Hd, f8, mboth, flow12, match, int(ctl[2])))
            # evaluation.py:235 tests len(...) == 0 after the append: always masked (a no-op on the first hypothesis unless
            # a background mask is given)
            matchFine = match[0, 0] * (1 - fgMask)
            nbCoarse += 1
            Mask = ((Mask + matchFine) >= 1.0).float()
        else:
            break
    if not acc:
        return dict(H=np.zeros((0,)), flowDown8=np.zeros((0,)), matchDown8=np.zeros((0,)), flow12=[], match=[], nbMatch=[])
    packed = torch.cat([torch.cat([a[0], a[1].reshape(-1), a[2].reshape(-1), a[4].reshape(-1)]) for a in acc])
    host = _to_host(packed).copy().reshape(len(acc), -1)
    n8 = acc[0][1].numel()
    f8shape = tuple(acc[0][1].shape)
    return dict(H=host[:, :9].reshape(-1, 3, 3).astype(np.float32),
                flowDown8=host[:, 9:9 + n8].reshape((len(acc),) + f8shape[1:]),
                matchDown8=host[:, 9 + n8:9 + 2 * n8].reshape(len(acc), 2, f8shape[2], f8shape[3]),
                flow12=[a[3] for a in acc], match=[host[i, 9 + 2 * n8:].reshape(Ith, Itw) for i in range(len(acc))],
                nbMatch=[a[5] for a in acc])


# ------------------------------------------------------------------------------------------------------------------
# YFCC: four-rotation target search + re-matching hypothesis loop (evaluation/evalYFCC/evaluation.py:179-274)
# ------------------------------------------------------------------------------------------------------------------
YFCC_ANGLES = (0, 90, 180, 270)


def yfcc_background(It_bg, k, size):
    """evaluation/evalYFCC/evaluation.py:193 / :200 / :212 for rotation ``k``: the segNet map of the unrotated target (or
    None: all ones) rotated by ``np.rot90``, resized by SciPy 1.2's ``imresize`` (byte-scaling) to ``size`` = (w, h),
    ``< 128``.  float32 (h, w), 1 = kept (not sky): a CUDA tensor when ``It_bg`` is one (``ops.imresize_mask``, no host
    copy), else a numpy array."""
    from .dropin import imresize
    w, h = size
    if It_bg is None:                      # imresize of a constant map byte-scales to 0: every cell < 128
        return np.ones((h, w), dtype=np.float32)
    if torch.is_tensor(It_bg):
        return ops.imresize_mask(It_bg, h, w, rot=k)
    return (imresize(np.rot90(np.asarray(It_bg, dtype=np.float32), k), (h, w)) < 128).astype(np.float32)


def rotation_draws(counts, nbPoint=4):
    """The rotations (in the reference's order) whose ``getCoarse`` reaches ``outil.RANSAC`` and draws its samples: those
    with at least ``nbPoint`` matches (evalYFCC/coarseAlignFeatMatch.py:179-180 returns None before the draw)."""
    return [k for k in range(len(counts)) if int(counts[k]) >= nbPoint]


def rotation_scores(ran, status, inliers):
    """evaluation/evalYFCC/evaluation.py:203-206: the score of every rotation - the inlier count of RANSAC's hypothesis
    for the rotations ``ran`` (RF_RANSAC_* ``status``), 0 where RANSAC returned None or did not run.  RF_RANSAC_NO_MODEL
    raises where utils/outil.py:162 does."""
    scores = [0, 0, 0, 0]
    for k, st, n in zip(ran, status, inliers):
        if int(st) == 2:
            raise TypeError("'NoneType' object is not subscriptable")     # utils/outil.py:162
        scores[k] = int(n) if int(st) == 0 else 0
    return scores


def align_pair_yfcc(coarseModel, network, Is, It, maxCoarse=10, maskRegionTh=0.01, It_bg=None, samples=None):
    """One pair through evalYFCC's loop (evaluation/evalYFCC/evaluation.py:179-274) with a variant-B / C ``coarseModel``,
    eager and steered from the host like ``align_pair_device``:

      * rotation search (:191-212): the source pyramid and the four rotated targets through the trunk as one ragged batch,
        the four masked re-matchings, ONE host read of the four match counts, then RANSAC in rotation order for the
        rotations with at least 4 matches only (the reference returns None before RANSAC draws, so a seeded run consumes
        the reference's sample stream); the score is the inlier count of the winning hypothesis (= ``np.sum(InlierMask)``:
        mutual matches use each target cell once), 0 when RANSAC returns None; the first maximum wins;
      * the hypothesis loop of ``align_pair_device`` on the winning rotation: masked re-matching per ``getCoarse``,
        ``match12 * match21`` matchability (:32-62), 12 bytes per hypothesis to the host.

    ``Is`` / ``It``: PIL images or uint8 (H, W, 3) CUDA tensors.  ``It_bg``: ``skyFromSeg`` of the unrotated target (a host
    array, or the float32 CUDA mask of ``SegNet.run``, which then never leaves the device), or None (no ``--segNet``).  ``samples``: optional injected (nbIter, 4) index tables, one per RANSAC call in the reference's
    order.  Returns ``align_pair_device``'s dict plus ``angle``, ``nbInlierRot`` (the four scores) and ``It_bg`` (the
    resized boolean background map the driver saves as ``maskBG_``)."""
    with torch.no_grad():
        coarseModel._set_rotated_pair(Is, It)
        best, nbInlierRot, bg, calls = _rotation_search(coarseModel, It_bg, samples)
        rest = None
        if samples is not None:       # a last call with M < 4 draws nothing in the reference: any table serves it
            rest = list(samples[calls:]) + [np.zeros((coarseModel.nbIter, coarseModel.nbPoint), dtype=np.int64)]
        out = _hypotheses_device(coarseModel, network, maxCoarse, maskRegionTh, True, bg, rest, rewind_too_few=True)
    w, h = coarseModel.target_size
    if torch.is_tensor(bg):
        bg = bg.cpu().numpy()
    out.update(angle=YFCC_ANGLES[best], nbInlierRot=nbInlierRot,
               It_bg=(bg if bg is not None else np.ones((h, w), dtype=np.float32)).astype(bool))
    return out


def _rotation_search(c, It_bg, samples):
    """evaluation.py:195-212 on the rotations ``_set_rotated_pair`` computed: selects the winning rotation.  Returns (its index,
    the four scores, its background map (None without ``It_bg``), the number of RANSAC calls made)."""
    bgs, found = [], []
    for k in range(4):
        c._select_target(k)
        bg = yfcc_background(It_bg, k, c.rotated_target_size(k))
        bgs.append(bg)
        if It_bg is None:
            Mt = None
        elif torch.is_tensor(bg):
            Mt = ((1 - bg) > 0.5).float()
        else:
            Mt = ((1 - bg) > 0.5).astype(np.float32)
        m1, m2, _, cnt = c._match_device(Mt)
        found.append((m1, m2, cnt))
    counts = _to_host(torch.cat([f[2] for f in found])).copy()               # the one read the draw decision needs
    ran = rotation_draws(counts, c.nbPoint)
    res = []
    for n, k in enumerate(ran):
        m1, m2, cnt = found[k]
        _, _, mask, status = c._ransac_device(m1, m2, cnt, None if samples is None else samples[n])
        res.append(torch.cat([status, mask[:int(counts[k])].sum(dtype=torch.int32).reshape(1)]))
    res = _to_host(torch.cat(res)).copy().reshape(-1, 2) if res else np.zeros((0, 2), dtype=np.int32)
    nbInlierRot = rotation_scores(ran, res[:, 0], res[:, 1])
    best = int(np.argmax(nbInlierRot))                                          # np.argmax: the first maximum wins
    c._select_target(best)
    return best, nbInlierRot, (bgs[best] if It_bg is not None else None), len(ran)


def align_pair_yfcc_host(coarseModel, network, Is, It, maxCoarse=10, maskRegionTh=0.01, It_bg=None):
    """The drop-in path of evalYFCC: the driver's statements (evaluation/evalYFCC/evaluation.py:191-274) on the mirror
    ``CoarseAlignB`` (``setSource`` / ``setTarget`` / ``getCoarse``, host-synchronised, RANSAC samples from
    ``torch.randint`` on the CUDA generator) and ``PredFlowMask`` with ``match21``.  ``Is`` / ``It``: PIL images.  Same
    dict as ``align_pair_yfcc`` (without ``nbMatch``); the yardstick its device path is tested and timed against."""
    c = coarseModel
    with torch.no_grad():
        c.setSource(Is)
        ItList = [It] + [It.rotate(a, expand=True) for a in YFCC_ANGLES[1:]]
        nbInlier = []
        for k in range(4):
            c.setTarget(ItList[k])
            bg = yfcc_background(It_bg, k, c.It.size)
            bestPara, InlierMask = c.getCoarse(((1 - bg) > 0.5).astype(np.float32))
            nbInlier.append(0 if bestPara is None else int(np.sum(InlierMask)))
        best = int(np.argmax(nbInlier))
        c.setTarget(ItList[best])
        Itw, Ith = c.It.size
        bg = yfcc_background(It_bg, best, (Itw, Ith))
        featt = fine_features(network["netFeatCoarse"], c.ItTensor)
        grid = torch.empty((1, Ith, Itw, 2), device="meta")                     # size carrier only
        warper = HomographyWarper(Ith, Itw)
        Mask = np.zeros((Ith, Itw), dtype=np.float32)
        Hs, flows8, matches8, flows, matches = [], [], [], [], []
        nbCoarse = 0
        while nbCoarse <= maxCoarse:
            fgMask = ((Mask + (1 - bg)) > 0.5).astype(np.float32)
            bestPara, _ = c.getCoarse(fgMask)
            if bestPara is None:
                break
            flowCoarse = warper.warp_grid(torch.from_numpy(bestPara).unsqueeze(0).cuda())
            flowFine, matchFine, f8, m8 = PredFlowMask(c.IsTensor, featt, flowCoarse, grid, network, with_match21=True)
            if (matchFine * (1 - fgMask)).mean() > maskRegionTh or nbCoarse == 0:
                Hs.append(bestPara[None])
                flows8.append(f8)
                matches8.append(m8)
                flows.append(flowFine)
                matches.append(matchFine)
                nbCoarse += 1
                Mask = ((Mask + matchFine * (1 - fgMask)) >= 1.0).astype(np.float32)
            else:
                break
    cat = lambda l: np.concatenate(l, axis=0) if l else np.zeros((0,))
    return dict(H=cat(Hs), flowDown8=cat(flows8), matchDown8=cat(matches8), flow12=flows, match=matches, angle=YFCC_ANGLES[best],
                nbInlierRot=nbInlier, It_bg=bg.astype(bool))


def align2images(coarseModel, network, img1, img2, align_corners=False):
    """quick_start/align2images.py:53-97 without the matplotlib / file output: coarse homography from the variant-C
    CoarseAlign, coarse warp, fine flow (no clamp, align2images.py:91-94) and the finely aligned source.
    Note the reference calls ``netCorr(feat_source, feat_target)`` here (align2images.py:89, SURVEY A.3 #9)."""
    with torch.no_grad():
        coarseModel.setSource(img1)
        coarseModel.setTarget(img2)
        w, h = coarseModel.target_size
        bestPrm, inlierMask = coarseModel.getCoarse(np.zeros((h, w)))
        if bestPrm is None:
            return None
        Hd = torch.from_numpy(bestPrm).unsqueeze(0).cuda()
        flowCoarse = HomographyWarper(h, w).warp_grid(Hd)
        img1_coarse = ops.grid_sample(coarseModel.IsTensor, flowCoarse, align_corners)
        feat1 = fine_features(network["netFeatCoarse"], img1_coarse)
        feat2 = fine_features(network["netFeatCoarse"], coarseModel.ItTensor)
        k = network["netCorr"].kernelSize
        if model.fine_engine() == ops.ENGINE_SPLIT:
            corr12, _ = ops.corr_neigh_pair_split(feat1, feat2, k, network["netFlowCoarse"].CORR_LD, want_both=False)
        else:
            corr12 = ops.corr_neigh(feat1, feat2, k, network["netFlowCoarse"].CORR_LD, model.fine_engine())
        flowDown = network["netFlowCoarse"].forward_ragged(corr12)
        flow12, _, _ = ops.compose_fine(flowDown, None, None, flowCoarse, clamp=False, align_corners=align_corners, want_match=False)
        img1_fine = ops.grid_sample(coarseModel.IsTensor, flow12, align_corners)
        return dict(bestPrm=bestPrm, inlierMask=inlierMask, flowCoarse=flowCoarse, img1_coarse=img1_coarse, flowDown=flowDown,
                    flow12=flow12, img1_fine=img1_fine)


# ------------------------------------------------------------------------------------------------------------------
# KITTI: two-level fine flow (evaluation/evalKITTI/evaluation.py) and its recomposition (evalKITTI/getResults.py)
# ------------------------------------------------------------------------------------------------------------------
def PredFlowMask_kitti_device(IsSample, ItSample, flowCoarse, size, network, align_corners=False, featt=None, feat_box=None):
    """evaluation/evalKITTI/evaluation.py:49-81 without the device->host copy: both images' fine features are computed
    here (one ragged batch of two images), the matchability is always ``match12 * grid_sample(match21) * inside``, and
    ``flowCoarse`` (1,Hc,Wc,2) may live on another grid than the ``size`` = (H, W) outputs (the second level, :296-302).
    Returns CUDA tensors (flow12 (1,H,W,2), match (1,1,H,W), flowDown8 (1,2,h8,w8), matchDown8 (1,2,h8,w8)).
    ``featt`` (a Ragged): the target's fine features from an earlier batch, so only the source goes through the
    FeatureExtractor; ``feat_box`` (a dict) receives the target's features of this batch under "featt"."""
    with torch.no_grad():
        corr12, both, _held = _fine_corr(network, IsSample, ItSample, featt, feat_box)
        flowDown8 = network["netFlowCoarse"].forward_ragged(corr12)
        mboth = network["netMatch"].forward_ragged(both)                    # (2,1,h8,w8): match12, match21
        flow12, match, _ = ops.compose_fine(flowDown8, mboth[0:1], mboth[1:2], flowCoarse, clamp=True, align_corners=align_corners,
                                            size=size)
        return flow12, match, flowDown8, mboth.permute(1, 0, 2, 3).contiguous()


def PredFlowMask_kitti(IsSample, ItSample, flowCoarse, grid, network):
    """Same inputs / outputs as evaluation/evalKITTI/evaluation.py:49-81 (``match`` as a numpy (H, W) array, the /8
    tensors on the device)."""
    flow12, match, f8, m8 = PredFlowMask_kitti_device(IsSample, ItSample, flowCoarse, (grid.size()[1], grid.size()[2]), network)
    return flow12, match[0, 0].cpu().numpy(), f8, m8


def remove_small_cc(matchFine, match_th, cc_th):
    """evaluation/evalKITTI/evaluation.py:85-100 for a numpy (H, W) map, on the device (connected components by union-find)."""
    m = torch.from_numpy(np.ascontiguousarray(matchFine, dtype=np.float32)).cuda()
    return ops.remove_small_cc(m, match_th, cc_th).cpu().numpy()


def align_pair_kitti(coarseModel, network, Is, It, fineSize=650, cc_th=0.01, maskRegionTh=0.005, maxH=None, It_bg=None):
    """One pair through evaluation/evalKITTI/evaluation.py:216-344 (no file output): per hypothesis the coarse
    homography from ``coarseModel`` (variant A at ``coarseSize``), the first fine level on the half-size target, the
    second level on the ``fineSize`` target sampled on the ORIGINAL image's grid, small connected components of the
    matchability removed on the device, and the reference's mask update on the host.  ``Is`` / ``It``: PIL images.
    ``maxH`` caps the reference's ``while True``.  ``It_bg``: with ``--segNet``, the raw ``skyFromSeg`` map of the target (host
    array or CUDA tensor, :245-250), resized to the original size by ``ops.imresize_mask`` (byte-scaling; both PIL passes are
    skipped); it masks every hypothesis and is returned as ``It_bg`` (bool, for ``results.save_pair_kitti``).  Returns the four
    arrays the script saves (H (nH,3,3) 'Homograpy', flow_d2 'Finetune_D2', mask 'Finetune_Mask', flow 'Finetune') plus the
    per-hypothesis full-resolution maps."""
    from . import outil
    strideNet = 8
    to_t = lambda I: coarseModel._to_tensor01(coarseModel._to_device_u8(I))          # transforms.ToTensor()(I)[None].cuda()
    It_resize = outil.resizeImg(It, strideNet, fineSize)
    It_d2 = outil.resizeImg(It, strideNet, fineSize // 2)
    w_org, h_org = It.size
    tensor_s = to_t(Is)
    (w_r, h_r), tensor_resize = It_resize.size, to_t(It_resize)
    (w_d2, h_d2), tensor_d2 = It_d2.size, to_t(It_d2)
    coarseModel.setPair(Is, It)
    given = It_bg is not None
    if given:                    # :248 (the reference's It_bg_tensor at the d2 size, :247, is never used)
        It_bg = ops.imresize_mask(It_bg, h_org, w_org).cpu().numpy()
    else:
        It_bg = np.ones((h_org, w_org), dtype=np.float32)
    Mask = np.zeros((h_org, w_org), dtype=np.float32)
    Hs, D2, Msk, Fin, maps = [], [], [], [], []
    nbCoarse = 0
    while maxH is None or nbCoarse < maxH:
        fgMask = ((Mask + (1 - It_bg)) > 0.5).astype(np.float32)
        bestPara = coarseModel.getCoarse(fgMask)
        if bestPara is None:
            break
        with torch.no_grad():
            bp = torch.from_numpy(bestPara).unsqueeze(0).cuda()
            homography_d2 = ops.warp_grid(bp, h_d2, w_d2)
            homography_resize = ops.warp_grid(bp, h_r, w_r)
            IsSample_d2 = ops.grid_sample(tensor_s, homography_d2)
            _, _, flowFine_d2, _ = PredFlowMask_kitti_device(IsSample_d2, tensor_d2, homography_d2, (h_d2, w_d2), network)
            flowCoarse, _, _ = ops.compose_fine(flowFine_d2, None, None, homography_resize, clamp=True, want_match=False)     # :291-294
            IsSample = ops.grid_sample(tensor_s, flowCoarse)
            flowFine_org, match_org, f8, m8 = PredFlowMask_kitti_device(IsSample, tensor_resize, flowCoarse, (h_org, w_org), network)
            ops.remove_small_cc(match_org, 0.99, cc_th)                                                                        # :311
            matchFine = match_org[0, 0].cpu().numpy()
        if ((matchFine > 0.9999) * (1 - fgMask)).mean() > maskRegionTh or nbCoarse == 0:
            Hs.append(bestPara[None])
            D2.append(flowFine_d2.cpu().numpy())
            Msk.append(m8.cpu().numpy())
            Fin.append(f8.cpu().numpy())
            maps.append((flowFine_org, matchFine.copy()))
            nbCoarse += 1
            matchFine = matchFine * (1 - fgMask)              # :324 (len(Finetune_Mask) is never 0 here)
            Mask = ((Mask + matchFine) > 0.9999).astype(np.float32)
        else:
            break
    cat = lambda l: np.concatenate(l, axis=0) if l else np.zeros((0,))
    out = dict(H=cat(Hs), flow_d2=cat(D2), mask=cat(Msk), flow=cat(Fin), maps=maps, size=(h_org, w_org))
    if given:
        out["It_bg"] = It_bg.astype(bool)
    return out


def fine_sizes(w, h, strideNet, minSize):
    """The (w, h) ``outil.resizeImg(I, strideNet, minSize)`` resizes a w x h image to (utils/outil.py:6-19), from the size
    alone: the same float divisions and Python ``round`` (half to even)."""
    ratio = min(w / minSize, h / minSize)
    return round(w / ratio / strideNet) * strideNet, round(h / ratio / strideNet) * strideNet


_cmin_cache = {}


def kitti_region_cmin(n, maskRegionTh):
    """The smallest count c for which evalKITTI's acceptance test (evaluation.py:316), numpy's own
    ``((m > 0.9999) * (1 - fgMask)).mean() > maskRegionTh``, holds for an n-pixel map with c new matched pixels; n + 1 when no
    count does.  Found by bisection on that very expression (float32 mean, numpy's comparison rule), so the kernel only compares
    integers.  The mean depends on c alone while its partial sums are exact, i.e. for n < 2**24.  Cached per (n, maskRegionTh)."""
    n = int(n)
    key = (n, float(maskRegionTh))
    if key not in _cmin_cache:
        assert 0 < n < 2 ** 24, "kitti_region_cmin: the float32 mean is exact only below 2**24 pixels"
        fg = np.zeros(n, dtype=np.float32)

        def accepted(c):
            m = np.zeros(n, dtype=np.float32)
            m[:c] = 1
            return bool(((m > 0.9999) * (1 - fg)).mean() > maskRegionTh)

        lo, hi = 0, n + 1                      # accepted(hi) is taken as true; find the first true in [lo, hi]
        while lo < hi:
            mid = (lo + hi) // 2
            if accepted(mid):
                hi = mid
            else:
                lo = mid + 1
        _cmin_cache[key] = lo
    return _cmin_cache[key]


def _kitti_device(coarseModel, network, Is_u8, It_u8, fineSize, cc_th, maskRegionTh, maxH, segNet=False, samples=None):
    """evaluation/evalKITTI/evaluation.py:216-336 for one pair with NO host control: everything is queued on the current stream
    and nothing is read back, so the whole pair can be captured in one CUDA graph.
      * the two fine-level targets are resized by the device LANCZOS (``outil.resizeImg`` to ``fineSize`` and ``fineSize // 2``);
      * the target's fine features are computed once per level, in the first hypothesis' two-image batch (``feat_box``);
      * ``maxH`` iterations run unconditionally: getCoarse (masked by fgMask), the two warp grids, the d2 level, its composition
        to the resized grid, the org level, ``remove_small_cc`` and ``ops.kitti_region_step``, which turns the reference's
        acceptance test and mask update (:316-326) into a device ``alive`` flag.  Hypotheses after the first dead one are
        computed but dropped by the host when it unpacks.
    ``Is_u8`` / ``It_u8``: uint8 (H, W, 3) CUDA images.  ``segNet``: the background of :245-250 is segNet's map of the target,
    byte-scaled to the original size (``ops.imresize_mask``).  Returns (packed records, per-hypothesis (flow (1,H,W,2),
    match (H,W)) CUDA maps, (h_org, w_org), (flow_d2 shape, flow shape)[, the uint8 (h_org, w_org) background map]), the
    fields of a ``DevicePair`` in order; one record per hypothesis: [alive, status, nbMatch, nbInlier, H(9), Finetune_D2,
    Finetune_Mask, Finetune]."""
    with torch.no_grad():
        h_org, w_org = int(It_u8.shape[0]), int(It_u8.shape[1])
        w_r, h_r = fine_sizes(w_org, h_org, 8, fineSize)
        w_d2, h_d2 = fine_sizes(w_org, h_org, 8, fineSize // 2)
        to_t = coarseModel._to_tensor01
        tensor_s = to_t(Is_u8)
        tensor_resize = to_t(ops.resize_lanczos_u8(It_u8, w_r, h_r))
        tensor_d2 = to_t(ops.resize_lanczos_u8(It_u8, w_d2, h_d2))
        coarseModel.setPair(Is_u8, It_u8)
        dev = It_u8.device
        if segNet:
            bg = ops.imresize_mask(_require_segnet(coarseModel).run(It_u8)[0], h_org, w_org)              # :248
        else:
            bg = torch.ones((h_org, w_org), device=dev)
        Mask = torch.zeros((h_org, w_org), device=dev)
        fgMask = ((Mask + (1 - bg)) > 0.5).float()
        alive = torch.ones(1, device=dev, dtype=torch.int32)
        cmin = kitti_region_cmin(h_org * w_org, maskRegionTh)
        box_d2, box_r = {}, {}
        recs, maps, shapes = [], [], None
        for k in range(maxH):
            Hd, nb, _, status, cnt = coarseModel.getCoarse_device(fgMask, None if samples is None else samples[k])
            bp = Hd.view(1, 3, 3)
            homography_d2 = ops.warp_grid(bp, h_d2, w_d2)
            homography_resize = ops.warp_grid(bp, h_r, w_r)
            IsSample_d2 = ops.grid_sample(tensor_s, homography_d2)
            _, _, flowFine_d2, _ = PredFlowMask_kitti_device(IsSample_d2, tensor_d2, homography_d2, (h_d2, w_d2), network,
                                                             featt=box_d2.get("featt"), feat_box=box_d2)
            flowCoarse, _, _ = ops.compose_fine(flowFine_d2, None, None, homography_resize, clamp=True, want_match=False)
            IsSample = ops.grid_sample(tensor_s, flowCoarse)
            flowFine_org, match_org, f8, m8 = PredFlowMask_kitti_device(IsSample, tensor_resize, flowCoarse, (h_org, w_org), network,
                                                                        featt=box_r.get("featt"), feat_box=box_r)
            ops.remove_small_cc(match_org, 0.99, cc_th)
            match = match_org.view(h_org, w_org)
            rec = ops.kitti_region_step(match, Mask, bg, fgMask, status, alive, k == 0, cmin)
            recs.append(torch.cat([rec[:1].float(), status.float(), cnt.float(), nb.float(), Hd, flowFine_d2.reshape(-1),
                                   m8.reshape(-1), f8.reshape(-1)]))
            maps.append((flowFine_org, match))
            shapes = (tuple(flowFine_d2.shape), tuple(f8.shape))
        packed = torch.cat(recs)
    out = (packed, maps, (h_org, w_org), shapes)
    return out + (bg.to(torch.uint8),) if segNet else out


def _unpack_kitti(host, maps, size, shapes, maxH, bg=None):
    """The host side of ``_kitti_device``: the hypotheses up to the first dead one, in ``align_pair_kitti_graph``'s dict."""
    n, rows = _accepted(host, maxH)
    out = dict(maps=list(maps[:n]), size=tuple(size), capped=n == maxH, **_counts(rows))
    d2shape, f8shape = shapes
    out["H"], out["flow_d2"], out["mask"], out["flow"] = _split(rows, [d2shape, f8shape, f8shape])
    if bg is not None:
        out["It_bg"] = bg.reshape(size).astype(bool)
    return out


def _as_device_u8(coarseModel, I):
    """A PIL image, numpy array or uint8 (H, W, 3) tensor as a uint8 CUDA image."""
    if torch.is_tensor(I):
        return I if I.is_cuda else I.cuda()
    return coarseModel._to_device_u8(I)


def align_pair_kitti_graph(coarseModel, network, Is, It, fineSize=650, cc_th=0.01, maskRegionTh=0.005, maxH=5, segNet=False, samples=None):
    """``align_pair_kitti`` without any host round trip inside the pair (``_kitti_device``, run eagerly), then one pinned D2H of
    the records.  ``Is`` / ``It``: PIL images, numpy arrays or uint8 (H, W, 3) tensors.  ``maxH`` is required: the reference's
    ``while True`` becomes ``maxH`` unconditional iterations.  Returns ``align_pair_kitti``'s dict (``maps``: the accepted
    hypotheses' (flow, match) as CUDA tensors) plus ``nbMatch`` / ``nbInlier`` per hypothesis and ``capped`` (all ``maxH``
    hypotheses accepted: the reference might have gone on); with ``segNet`` also ``It_bg``.  Under ``torch.manual_seed(s)`` the
    RANSAC samples are the reference's; the hypotheses after the first dead one still draw theirs.  ``samples``: optional
    injected (nbIter, 4) tables, one per hypothesis."""
    if maxH is None or int(maxH) < 1:
        raise ValueError("align_pair_kitti_graph: maxH must be a positive hypothesis cap")
    maxH = int(maxH)
    pair = DevicePair(*_kitti_device(coarseModel, network, _as_device_u8(coarseModel, Is), _as_device_u8(coarseModel, It), fineSize,
                                     cc_th, maskRegionTh, maxH, segNet, samples))
    host, bg = _read_back(pair)
    return _unpack_kitti(host, pair.maps, pair.size, pair.shapes, maxH, bg)


class GraphedKittiAligner(GraphedAligner):
    """evalKITTI's pair (``align_pair_kitti_graph``: trunk, matching, ``maxH`` x (RANSAC, two fine levels, remove_small_cc,
    acceptance test and mask update)) as ONE CUDA graph per pair of input sizes, with the LRU eviction of ``GraphedAligner``.
    It can be a ``ConcurrentAligner`` lane (``make_aligner``).  ``fetch`` returns ``align_pair_kitti_graph``'s dict; its
    ``maps`` are cloned from the graph's static buffers (``copy=False``: the live buffers, overwritten by the next replay with
    these input sizes)."""

    def __init__(self, coarseModel, network, fineSize=650, cc_th=0.01, maskRegionTh=0.005, maxH=5, segNet=False, warmup=2, max_graphs=4):
        if segNet:
            _require_segnet(coarseModel)
        if maxH is None or int(maxH) < 1:
            raise ValueError("GraphedKittiAligner: maxH must be a positive hypothesis cap")
        super().__init__(coarseModel, network, warmup=warmup, max_graphs=max_graphs)
        self.fineSize, self.cc_th, self.maskRegionTh, self.maxH, self.segNet = fineSize, cc_th, maskRegionTh, int(maxH), bool(segNet)

    def _device(self, s_in, t_in):
        return DevicePair(*_kitti_device(self.coarse, self.net, s_in, t_in, self.fineSize, self.cc_th, self.maskRegionTh, self.maxH,
                                         self.segNet))

    def _unpack(self, host, bg, maps, size, shapes):
        return _unpack_kitti(host, maps, size, shapes, self.maxH, bg)


def getFlow_all_kitti(param, flowd2, flow, match, outH, outW, th=1.0, cc_th=0.01, multiH=True, interpolate=False):
    """evaluation/evalKITTI/getResults.py:95-141 after its np.load calls: param (nH,3,3) 'Homograpy', flowd2 (nH,2,.,.)
    'Finetune_D2', flow (nH,2,.,.) 'Finetune', match (nH,2,.,.) 'Finetune_Mask' -> (flowGlobal (1,outH,outW,2), binary match
    map), both CUDA.  The two levels are composed with the fused kernel, small connected components are removed on the
    device, the first-hypothesis-wins merge is elementwise torch.  ``interpolate``: the EDT hole filling of :87-93
    (``ops.fill_nearest_matched``: exact nearest matched pixel; between equidistant ones the choice may differ from scipy's)."""
    param = torch.as_tensor(param, dtype=torch.float32).cuda()
    flowd2 = torch.as_tensor(flowd2, dtype=torch.float32).cuda()
    flow = torch.as_tensor(flow, dtype=torch.float32).cuda()
    match = torch.as_tensor(match, dtype=torch.float32).cuda()
    homography_org = ops.warp_grid(param, outH, outW)
    fl, ms = [], []
    for i in range(flow.shape[0]):
        fd2, _, _ = ops.compose_fine(flowd2[i:i + 1], None, None, homography_org[i:i + 1], clamp=True, want_match=False)     # :104-107
        f12, m, _ = ops.compose_fine(flow[i:i + 1], match[i:i + 1, 0:1], match[i:i + 1, 1:2], fd2, clamp=True)              # :110-123
        fl.append(f12)
        ms.append(m)
    m = ops.remove_small_cc(torch.cat(ms, dim=0).contiguous(), 0.99, cc_th).permute(0, 2, 3, 1)
    f = torch.clamp(torch.cat(fl, dim=0), min=-1, max=1)
    flowGlobal = f[:1].clone()
    mb = m[:1] >= th
    if multiH:
        for i in range(1, len(m)):
            tmp = (m.narrow(0, i, 1) >= th) * (~mb)
            mb = mb + tmp
            tmp = tmp.expand_as(flowGlobal)
            flowGlobal[tmp] = f.narrow(0, i, 1)[tmp]
    if interpolate:
        flowGlobal = ops.fill_nearest_matched(flowGlobal, mb)
    return flowGlobal, mb


def merge_first_wins(f, m, th, multiH=True):
    """The first-hypothesis-wins merge every getResults script ends with (evaluation/evalCorr/getResults.py:121-134):
    f (nH,H,W,2) clamped flows, m (nH,H,W,1) matchabilities -> (flowGlobal (1,H,W,2), matchGlobal (1,H,W,1), binary map).
    Elementwise torch on the tensors' device."""
    flowGlobal, matchGlobal = f[:1].clone(), m[:1].clone()
    mb = m[:1] >= th
    if multiH:
        for i in range(1, len(m)):
            tmp = (m.narrow(0, i, 1) >= th) * (~mb)
            matchGlobal[tmp] = m.narrow(0, i, 1)[tmp]
            mb = mb + tmp
            tmp = tmp.expand_as(flowGlobal)
            flowGlobal[tmp] = f.narrow(0, i, 1)[tmp]
    return flowGlobal, matchGlobal, mb


def getFlow_corr(flow, param, match, th=0.95, multiH=True):
    """evaluation/evalCorr/getResults.py:78-134 ``getFlow`` (= evalYFCC/getResults.py:150-190 ``_getFlow``) after its np.load
    calls: flow (nH,2,h8,w8), param (nH,3,3), match (nH,2,h8,w8) -> (flowGlobal (1,8h8,8w8,2), matchGlobal (1,8h8,8w8,1)), CUDA:
    x8 upsampling, ``match12 * grid_sample(match21) * inside`` from the fused composition kernel, then ``merge_first_wins``."""
    flowGlobal, matchGlobal, _ = getFlow_corr_binary(flow, param, match, th, multiH)
    return flowGlobal, matchGlobal


def getFlow_corr_binary(flow, param, match, th=0.95, multiH=True):
    """``getFlow_corr`` plus the merge's binary map (1,8h8,8w8,1) bool, which evalYFCC's ``_getFlow`` returns instead of the
    matchability (evalYFCC/getResults.py:178-187)."""
    flow = torch.as_tensor(flow, dtype=torch.float32).cuda()
    param = torch.as_tensor(param, dtype=torch.float32).cuda()
    match = torch.as_tensor(match, dtype=torch.float32).cuda()
    H, W = int(flow.shape[2]) * 8, int(flow.shape[3]) * 8
    coarse = ops.warp_grid(param, H, W)
    fl, ms = [], []
    for i in range(flow.shape[0]):
        f12, m, _ = ops.compose_fine(flow[i:i + 1], match[i:i + 1, 0:1], match[i:i + 1, 1:2], coarse[i:i + 1], clamp=True)
        fl.append(f12)
        ms.append(m)
    f = torch.clamp(torch.cat(fl, dim=0), min=-1, max=1)
    m = torch.cat(ms, dim=0).permute(0, 2, 3, 1)
    return merge_first_wins(f, m, th, multiH)


def getFlow_all(flow, param, match, outH, outW, th=0.95, multiH=True, with_match21=False):
    """evaluation/evalHpatch/getResults.py:16-63 on device tensors: flow (nH,2,h8,w8), param (nH,3,3),
    match (nH,2,h8,w8) -> flowGlobal (1,outH,outW,2).  The reference runs this on CPU tensors; the
    composition here is the fused kernel, the first-hypothesis-wins merge is elementwise torch."""
    flow = torch.as_tensor(flow, dtype=torch.float32).cuda()
    param = torch.as_tensor(param, dtype=torch.float32).cuda()
    match = torch.as_tensor(match, dtype=torch.float32).cuda()
    coarse = ops.warp_grid(param, outH, outW)
    fl, ms = [], []
    for i in range(flow.shape[0]):
        f12, m, _ = ops.compose_fine(flow[i:i + 1], match[i:i + 1, 0:1], match[i:i + 1, 1:2] if with_match21 else None,
                                     coarse[i:i + 1], clamp=True)
        fl.append(f12)
        ms.append(m)
    f = torch.clamp(torch.cat(fl, dim=0), min=-1, max=1)
    m = torch.cat(ms, dim=0).permute(0, 2, 3, 1)
    flowGlobal = f[:1].clone()
    if multiH:
        mb = m[:1] >= th
        for i in range(1, len(m)):
            tmp = (m.narrow(0, i, 1) >= th) * (~mb)
            mb = mb + tmp
            tmp = tmp.expand_as(flowGlobal)
            flowGlobal[tmp] = f.narrow(0, i, 1)[tmp]
    return flowGlobal


# evalYFCC's pair from CUDA graphs (its kernel entries live with it, in yfcc_graph)
from .yfcc_graph import GraphedYfccAligner, align_pair_yfcc_graph  # noqa: E402,F401

# train/generate_coarse_aligned_pair.ipynb's pair (its kernel entry lives with it, in train_pairs)
from .train_pairs import GraphedTrainPairAligner, TrainPairModel, align_train_pair  # noqa: E402,F401
