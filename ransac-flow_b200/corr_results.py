"""evalCorr's getResults.py (the MegaDepth-1600 and RobotCar PCK tables) on the device: the multi-hypothesis composition, the
first-hypothesis-wins merge and alignmentError evaluated at the annotated keypoints only, with the counts of the whole dataset
accumulated on the device and read once, at the end.

  image_size / pair_keypoints  : getResults.py:210-237 (``ResizeMinResolution`` / ``ResizeMinResolution_megadepth``): the
                                 sizes come from the image headers (``Image.open(path).size``); nothing is decoded or resized
  CorrScores                   : the dataset's ``precAllAlign`` / ``validAlign`` (:178-183) as one device accumulator, the
                                 missing-pair rule (:242-246) and the errors the reference raises
  score_pair                   : :239-253 for one pair from the dict ``pipeline.align_pair*`` returns (what ``results.save_pair``
                                 writes), queued with nothing read back
  get_results                  : :196-256 over a DataFrame and the ``.npy`` files evaluation.py wrote
  evaluate                     : evaluation/evalCorr/evaluation.py's loop (``pipeline.align_pair_multi``) and the scoring in one
                                 pass, writing no files unless asked to
  python -m ransac_flow_b200.corr_results : getResults.py's command line; with ``--resumePth`` it aligns in-process

The keypoint kernel (``corr_keypoints``, ``rf_corr_keypoints``) reproduces the reference's arithmetic and its quirks
(DESIGN.md section 12): the ``<=`` compare, the int64 truncation and numpy's index rule, the flow read through
``.view(1, 1, Ith, Itw)``, and for a matchability threshold > 0 the broadcast of the (1, H, W, 1) threshold map with the
(1, 1, H, W) inside map, which raises for a non-square map and counts each selected keypoint once per inside pixel of a row
for a square one.
"""
import os

import numpy as np
import PIL.Image as Image
import torch

from . import pipeline, results
from ._lib import check, lib, need_cuda, ptr, stream
from .ops import _staging_for, _view
from .validation import resize_min_resolution_size, scale_keypoints

MIN_SIZE, STRIDE_NET = 480, 16                                               # getResults.py:171-172 (minSize's default)
PIXEL_GRID = np.around(np.logspace(0, np.log10(36), 8).reshape(-1, 8))       # getResults.py:185
NO_ERROR = 2 ** 31 - 1                                                       # the error word before any out-of-range index
_I32 = np.iinfo(np.int32)


# --------------------------------------------------------------------------- host rules
def image_path(testDir, scene, name):
    """getResults.py:204,215: ``testDir/scene/name``, or ``testDir/name`` when the scene is ``'/'``."""
    return os.path.join(os.path.join(testDir, scene), name) if scene != "/" else os.path.join(testDir, name)


def image_size(path):
    """(w, h) of an image from its header (PIL reads no pixels); a file PIL cannot open raises as ``Image.open`` does."""
    with Image.open(path) as im:
        return im.size


def pair_keypoints(df, i, testDir, dataset, minSize=MIN_SIZE, sizes=None):
    """Row i as getResults.py:200-222 reads it, in its order: (Xs, Ys, Xt, Yt) float32 in the resized images, (Isw, Ish) and
    (Itw, Ith).  MegaDepth keeps the keypoints strictly inside both resized images.  ``sizes``: the two original (w, h), if
    already known (the headers are read otherwise)."""
    scene = df["scene"][i]
    if sizes is None:
        ws, hs = image_size(image_path(testDir, scene, df["source_image"][i]))
    else:
        ws, hs = sizes[0]
    Isw, Ish = resize_min_resolution_size(ws, hs, minSize, STRIDE_NET)
    Xs, Ys = scale_keypoints(df["XA"][i], df["YA"][i], ws, hs, Isw, Ish)
    if sizes is None:
        wt, ht = image_size(image_path(testDir, scene, df["target_image"][i]))
    else:
        wt, ht = sizes[1]
    Itw, Ith = resize_min_resolution_size(wt, ht, minSize, STRIDE_NET)
    Xt, Yt = scale_keypoints(df["XB"][i], df["YB"][i], wt, ht, Itw, Ith)
    if dataset != "RobotCar":
        valid = (Xs > 0) * (Xs < Isw) * (Ys > 0) * (Ys < Ish) * ((Xt > 0) * (Xt < Itw) * (Yt > 0) * (Yt < Ith))
        Xs, Ys, Xt, Yt = Xs[valid], Ys[valid], Xt[valid], Yt[valid]
    return (Xs, Ys, Xt, Yt), (Isw, Ish), (Itw, Ith)


def truncate_keypoints(Xs, Ys, Xt, Yt):
    """alignmentError's ``astype(np.int64)`` (getResults.py:26), as int32 rows (xa, ya, xb, yb): beyond the int32 range an
    index is out of range and a distance beyond every threshold either way."""
    with np.errstate(invalid="ignore"):
        cols = np.stack([np.asarray(a).astype(np.int64) for a in (Xs, Ys, Xt, Yt)], axis=1).reshape(-1, 4)
    return np.ascontiguousarray(np.clip(cols, _I32.min, _I32.max).astype(np.int32))


def _keys(matchabilityTH):
    """The dict keys of precAllAlign / validAlign (equal thresholds share one) and each threshold's key index."""
    keys, slots = [], []
    for t in matchabilityTH:
        for k, key in enumerate(keys):
            if key == t:
                slots.append(k)
                break
        else:
            keys.append(t)
            slots.append(len(keys) - 1)
    return keys, slots


def _broadcast_error(H, W):
    return RuntimeError("The size of tensor a (%d) must match the size of tensor b (%d) at non-singleton dimension 2" % (W, H))


def _view_error(Ith, Itw, n):
    return RuntimeError("shape '[1, 1, %d, %d]' is invalid for input of size %d" % (Ith, Itw, n))


# --------------------------------------------------------------------------- kernel entry
CORR_MAX_MTH = 8                                                             # RF_CORR_MAX_MTH


def corr_keypoints(flowDown8, matchDown8, H, size_t, size_s, kpts, count, counts, err, thresholds, mth, slots, th, multiH,
                   onlyCoarse=False, pair=0, flow_out=None, match_out=None, hyp_out=None, dist_out=None):
    """``rf_corr_keypoints``: evalCorr/getResults.py's getFlow (getFlow_Coarse with ``onlyCoarse``), the per-threshold binary
    map and alignmentError at the keypoints of one pair.  flowDown8 / matchDown8 (nH, 2, h8, w8) and H (nH, 9) or (nH, 3, 3)
    fp32 on the device (flowDown8 is read for its shape only with ``onlyCoarse``, matchDown8 may then be None); ``size_t`` =
    (Ith, Itw) of the target, ``size_s`` = (hA, wA) of the source; kpts int32 (capacity, 4) = (xa, ya, xb, yb), ``count`` an
    int32 [1] on the device; ``counts`` an int64 accumulator of at least max(slots) + 1 rows of len(thresholds) + 1 counts and
    ``err`` an int32 [1] error word.  ``mth``: the matchability thresholds in order, ``slots`` their accumulator rows.
    Optional per-keypoint outputs: flow_out (capacity, 2) fp32, match_out (capacity,) fp32, hyp_out (capacity,) int32,
    dist_out (capacity, len(mth)) fp64."""
    need_cuda(flowDown8, matchDown8, H, kpts, count, counts, err, flow_out, match_out, hyp_out, dist_out)
    t = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float64).reshape(-1))
    m = np.ascontiguousarray(np.asarray(mth, dtype=np.float64).reshape(-1))
    sl = np.ascontiguousarray(np.asarray(slots, dtype=np.int32).reshape(-1))
    if flowDown8.dtype != torch.float32 or flowDown8.dim() != 4 or flowDown8.shape[1] != 2 or not flowDown8.is_contiguous():
        raise ValueError("corr_keypoints: flowDown8 must be a contiguous float32 (nH, 2, h8, w8) tensor")
    nH, _, h8, w8 = flowDown8.shape
    if matchDown8 is None and not onlyCoarse:
        raise ValueError("corr_keypoints: matchDown8 is required without onlyCoarse")
    if matchDown8 is not None and (matchDown8.dtype != torch.float32 or tuple(matchDown8.shape) != tuple(flowDown8.shape)
                                   or not matchDown8.is_contiguous()):
        raise ValueError("corr_keypoints: matchDown8 must be a contiguous float32 tensor shaped as flowDown8")
    if H.dtype != torch.float32 or H.numel() != 9 * nH or not H.is_contiguous():
        raise ValueError("corr_keypoints: H must be %d contiguous float32 values" % (9 * nH))
    if kpts.dtype != torch.int32 or kpts.dim() != 2 or kpts.shape[1] != 4 or not kpts.is_contiguous():
        raise ValueError("corr_keypoints: kpts must be a contiguous int32 (n, 4) tensor")
    if count.dtype != torch.int32 or count.numel() != 1 or err.dtype != torch.int32 or err.numel() != 1:
        raise ValueError("corr_keypoints: count and err must be one int32 each")
    if not 1 <= m.size <= CORR_MAX_MTH or sl.size != m.size or sl.min() < 0 or sl.max() >= m.size:
        raise ValueError("corr_keypoints: 1..%d matchability thresholds, each with a row in [0, %d)" % (CORR_MAX_MTH, m.size))
    if counts.dtype != torch.int64 or not counts.is_contiguous() or counts.numel() < (int(sl.max()) + 1) * (t.size + 1):
        raise ValueError("corr_keypoints: counts must be a contiguous int64 accumulator of (rows, T + 1) counts")
    cap, J = int(kpts.shape[0]), int(m.size)
    for name, o, shape, dt in (("flow_out", flow_out, (cap, 2), torch.float32), ("match_out", match_out, (cap,), torch.float32),
                               ("hyp_out", hyp_out, (cap,), torch.int32), ("dist_out", dist_out, (cap, J), torch.float64)):
        if o is not None and (tuple(o.shape) != shape or o.dtype != dt or not o.is_contiguous()):
            raise ValueError("corr_keypoints: %s must be a contiguous %s %s tensor" % (name, dt, shape))
    check(lib.rf_corr_keypoints(ptr(flowDown8), ptr(matchDown8), ptr(H), int(nH), int(h8), int(w8), int(size_t[0]), int(size_t[1]),
                                int(size_s[1]), int(size_s[0]), ptr(kpts), ptr(count), cap, int(pair), float(np.float32(th)),
                                int(bool(multiH)), int(bool(onlyCoarse)), t.ctypes.data, int(t.size), m.ctypes.data, sl.ctypes.data,
                                J, ptr(counts), ptr(err), ptr(flow_out), ptr(match_out), ptr(hyp_out), ptr(dist_out), stream()))


# --------------------------------------------------------------------------- the dataset accumulator
class CorrScores:
    """getResults.py's ``precAllAlign`` / ``validAlign`` over a dataset: one int64 device accumulator of (keys, T + 1) counts
    followed by the error word (its low 32 bits: the first pair with an out-of-range keypoint index, ``NO_ERROR`` if none).
    Pairs are queued on the current stream with nothing read back; ``result`` reads the device once."""

    def __init__(self, matchabilityTH=(0,), th=0.95, multiH=False, onlyCoarse=False, device=None):
        self.mth = list(matchabilityTH)
        if not 1 <= len(self.mth) <= CORR_MAX_MTH:
            raise ValueError("CorrScores: 1..%d matchability thresholds" % CORR_MAX_MTH)
        self.keys, self.slots = _keys(self.mth)
        self.th, self.multiH, self.onlyCoarse = th, bool(multiH), bool(onlyCoarse)
        self.T = PIXEL_GRID.size
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.acc = torch.zeros(len(self.keys) * (self.T + 1) + 1, dtype=torch.int64, device=self.device)
        self.acc[-1] = NO_ERROR
        self.counts = self.acc[:-1].view(len(self.keys), self.T + 1)
        self.err = self.acc[-1:].view(torch.int32)[:1]
        self.valid_host = [0] * len(self.keys)          # the missing pairs' ``validAlign[0] += len(Xs)``

    def missing(self, n):
        """getResults.py:242-246, a pair with no files: ``precAllAlign[0] = precAllAlign[th] + 0`` (``th``: the last
        matchability threshold) and ``validAlign[0] += n``; KeyError(0) when 0 is not a threshold."""
        k0 = next((k for k, key in enumerate(self.keys) if key == 0), None)
        if k0 is None:
            raise KeyError(0)
        kl = self.slots[-1]
        if kl != k0:
            self.counts[k0, :self.T].copy_(self.counts[kl, :self.T])
        self.valid_host[k0] += int(n)

    def pair_error(self, h8, w8, size_t):
        """The RuntimeError the reference raises for a pair before it reads any keypoint, with the number of thresholds it
        scores first: (count, error or None).  The flow's view as Ith x Itw needs the same number of pixels; a threshold > 0
        needs a square map (the broadcast of getResults.py:250)."""
        H, W = 8 * h8, 8 * w8
        Ith, Itw = size_t
        for q, t in enumerate(self.mth):
            if t > 0 and H != W:
                return q, _broadcast_error(H, W)
            if Ith * Itw != H * W:
                return q, _view_error(Ith, Itw, H * W)
        return len(self.mth), None

    def queue(self, flow, param, match, kpts, size_t, size_s, pair=0, dist_out=None, flow_out=None, match_out=None, hyp_out=None):
        """One pair's hypotheses (numpy flow / match (nH, 2, h8, w8), param (nH, 3, 3); ``match`` unused with onlyCoarse) and
        int32 keypoint rows, uploaded in one copy and scored.  ``size_t`` = (Ith, Itw), ``size_s`` = (Ish, Isw).  Raises the
        pair's RuntimeError (after queuing the thresholds the reference scores before it).  ``dist_out``: (n, thresholds)
        fp64 on the device, written when the pair raises nothing."""
        flow = np.ascontiguousarray(flow, dtype=np.float32)
        param = np.ascontiguousarray(param, dtype=np.float32).reshape(-1, 9)
        if self.onlyCoarse:                              # getFlow_Coarse: hypothesis 0's homography; the flow gives h8, w8
            flow, param = flow[:1], param[:1]
        nH, _, h8, w8 = flow.shape
        stop, error = self.pair_error(h8, w8, size_t)
        kpts = np.ascontiguousarray(np.asarray(kpts, dtype=np.int32).reshape(-1, 4))
        n = kpts.shape[0]
        if stop > 0 and n > 0:
            parts = [flow, param, np.array([n], np.int32), kpts]
            if not self.onlyCoarse:
                parts.append(np.ascontiguousarray(match, dtype=np.float32).reshape(flow.shape))
            with torch.no_grad(), torch.cuda.device(self.device):
                dev, o = _staging_for(self.device).upload(parts, self.device)
                f8 = _view(dev, o[0], torch.float32, flow.shape)
                Hm = _view(dev, o[1], torch.float32, (nH, 9))
                cnt = _view(dev, o[2], torch.int32, (1,))
                kp = _view(dev, o[3], torch.int32, (n, 4))
                m8 = None if self.onlyCoarse else _view(dev, o[4], torch.float32, flow.shape)
                corr_keypoints(f8, m8, Hm, size_t, size_s, kp, cnt, self.acc, self.err, PIXEL_GRID, self.mth[:stop],
                                   self.slots[:stop], self.th, self.multiH, self.onlyCoarse, pair, flow_out, match_out, hyp_out,
                                   dist_out if stop == len(self.mth) else None)
        if error is not None:
            raise error

    def read(self):
        """(counts (keys, T + 1), first failing pair or None) from one device read."""
        host = self.acc.cpu().numpy()
        err = int(host[-1:].view(np.int32)[0])
        return host[:-1].reshape(len(self.keys), self.T + 1), (None if err == NO_ERROR else err)

    def raise_pending(self, pair):
        """Called when pair ``pair`` raised on the host: raise instead the IndexError of a pair up to this one, which the
        reference met first (a pair's RuntimeError comes after the thresholds queued before it)."""
        _, err = self.read()
        if err is not None and err <= pair:
            raise IndexError("pair %d: a keypoint index is out of bounds of the flow or matchability map" % err) from None

    def result(self):
        """{threshold: (precAllAlign / validAlign (float64 8-vector), validAlign)} for each matchability threshold, as the
        reference's final loop (getResults.py:255-257) computes it; IndexError for the first pair with an out-of-range index."""
        counts, err = self.read()
        if err is not None:
            raise IndexError("pair %d: a keypoint index is out of bounds of the flow or matchability map" % err)
        out = {}
        for k, key in enumerate(self.keys):
            prec = np.zeros(self.T) + counts[k, :self.T]
            valid = int(counts[k, self.T]) + self.valid_host[k]
            with np.errstate(invalid="ignore", divide="ignore"):
                out[key] = (prec / valid, valid)
        return out


# --------------------------------------------------------------------------- one pair, the files, the dataset
def score_pair(out, kpts, sizes, scores, pair=0, dist_out=None, flow_out=None, match_out=None, hyp_out=None):
    """getResults.py:239-253 for one pair from the dict ``pipeline.align_pair*`` returns (H, flowDown8, matchDown8: the
    tensors ``results.save_pair`` writes), queued into ``scores`` (a ``CorrScores``) with nothing read back.  ``kpts``: the
    (Xs, Ys, Xt, Yt) float32 arrays of ``pair_keypoints``; ``sizes`` = ((Isw, Ish), (Itw, Ith)).  A pair without hypotheses
    is a pair with no files.  Optional per-keypoint outputs: see ``corr_keypoints``."""
    (Isw, Ish), (Itw, Ith) = sizes
    if len(out["H"]) == 0:
        scores.missing(len(kpts[0]))
        return
    scores.queue(out["flowDown8"], np.asarray(out["H"]).reshape(-1, 9), out["matchDown8"], truncate_keypoints(*kpts), (Ith, Itw),
                 (Ish, Isw), pair, dist_out, flow_out, match_out, hyp_out)


def _pair_files(i, finePth, coarsePth, maskPth, flowList, onlyCoarse):
    """getFlow / getFlow_Coarse's file reads (getResults.py:78-98,136-148): (flow, param, match) or None.  getFlow also
    loads the pair's ``maskBG`` file and fails without it; getFlow_Coarse reads no matchability."""
    nbH = results.find_nbH(i, flowList)
    if nbH is None:
        return None
    tag = "{}_{}H.npy".format(i, nbH)
    flow = np.load(os.path.join(finePth, "flow_" + tag)).astype(np.float32)
    param = np.load(os.path.join(coarsePth, "flow_" + tag)).astype(np.float32)
    if onlyCoarse:
        return flow, param, None
    match = np.load(os.path.join(finePth, "mask_" + tag)).astype(np.float32)
    bg = os.path.join(maskPth, "maskBG_" + tag)
    if not os.path.exists(bg):
        raise FileNotFoundError("[Errno 2] No such file or directory: '%s'" % bg)
    return flow, param, match


def get_results(df, testDir, finePth, coarsePth, multiH, th, matchabilityTH, dataset, onlyCoarse=False, minSize=MIN_SIZE,
                maskPth=None, dist_out=None):
    """getResults.py:178-257 over the DataFrame ``df`` and the ``.npy`` files of evaluation.py: {threshold: (precision
    8-vector, validAlign)}.  Every pair of ``df`` is read (``--beginIndex`` / ``--endIndex`` are ignored, as in the
    reference).  The device is read once, at the end; an error raises what the reference raises first.  ``dist_out``: a
    list that receives each pair's (n, len(matchabilityTH)) fp64 distances (NaN where a keypoint is not selected)."""
    scores = CorrScores(matchabilityTH, th, multiH, onlyCoarse)
    flowList = os.listdir(finePth)
    maskPth = finePth if maskPth is None else maskPth
    dists = []
    i = 0
    try:
        for i in range(len(df)):
            kpts, (Isw, Ish), (Itw, Ith) = pair_keypoints(df, i, testDir, dataset, minSize)
            files = _pair_files(i, finePth, coarsePth, maskPth, flowList, onlyCoarse)
            if files is None:
                scores.missing(len(kpts[0]))
                dists.append(None)
                continue
            flow, param, match = files
            d = None
            if dist_out is not None:
                d = torch.full((len(kpts[0]), len(scores.mth)), float("nan"), dtype=torch.float64, device=scores.device)
            scores.queue(flow, param.reshape(-1, 9), match, truncate_keypoints(*kpts), (Ith, Itw), (Ish, Isw), i, dist_out=d)
            dists.append(d)
    except Exception:
        scores.raise_pending(i)
        raise
    res = scores.result()
    if dist_out is not None:
        dist_out.extend(None if d is None else d.cpu().numpy() for d in dists)
    return res


def evaluate(df, testDir, coarseModel, network, dataset, matchabilityTH=(0,), th=0.95, multiH=False, onlyCoarse=False,
             maxCoarse=10, maskRegionTh=0.01, segNet=False, minSize=MIN_SIZE, outDir=None, beginIndex=0, endIndex=None):
    """evaluation/evalCorr/evaluation.py's loop (each pair through ``pipeline.align_pair_multi``, eager, one read per pair)
    and getResults.py's scoring in one pass, with no files: ``get_results``' dict.  Pairs ``beginIndex`` .. ``endIndex`` - 1
    are aligned; getResults.py reads every row, so the rows outside that range are scored as it scores a pair with no
    files (their keypoints counted into ``validAlign[0]``), and the table equals the one evaluation.py over the same range
    followed by getResults.py prints.  ``outDir``: also write evaluation.py's ``outDir_Coarse`` / ``outDir_Fine`` files
    (``results.save_pair``).  ``coarseModel`` / ``network``: as evaluation.py builds them (``netMatch`` included)."""
    endIndex = len(df) if endIndex is None else endIndex
    if outDir is not None:
        outCoarse, outFine = outDir + "_Coarse", outDir + "_Fine"
        for d in (outCoarse, outFine):
            if not os.path.exists(d):
                os.mkdir(d)
    scores = CorrScores(matchabilityTH, th, multiH, onlyCoarse)
    i = 0
    try:
        with torch.no_grad():
            for i in range(len(df)):
                if not beginIndex <= i < endIndex:
                    kpts, _, _ = pair_keypoints(df, i, testDir, dataset, minSize)
                    scores.missing(len(kpts[0]))
                    continue
                scene = df["scene"][i]
                Is = Image.open(image_path(testDir, scene, df["source_image"][i])).convert("RGB")
                It = Image.open(image_path(testDir, scene, df["target_image"][i])).convert("RGB")
                out = pipeline.align_pair_multi(coarseModel, network, Is, It, maxCoarse, maskRegionTh, with_match21=True, segNet=segNet)
                if outDir is not None:
                    results.save_pair(outCoarse, outFine, i, out, out.get("It_bg"))
                kpts, sizes_s, sizes_t = pair_keypoints(df, i, testDir, dataset, minSize, sizes=(Is.size, It.size))
                score_pair(out, kpts, (sizes_s, sizes_t), scores, pair=i)
    except Exception:
        scores.raise_pending(i)
        raise
    return scores.result()


# --------------------------------------------------------------------------- CLI
def build_parser():
    """getResults.py:152-172's arguments and sub-commands, plus evaluation.py's model arguments for ``--resumePth``."""
    import argparse
    p = argparse.ArgumentParser(description="evalCorr getResults (MegaDepth / RobotCar PCK) on the GPU")
    p.add_argument("--multiH", action="store_true", help="multiple homograhy or not")
    p.add_argument("--onlyCoarse", action="store_true", help="only Coarse")
    p.add_argument("--minSize", type=int, default=480, help="min size")
    p.add_argument("--matchabilityTH", type=float, nargs="+", default=[0], help="matchability threshold list")
    p.add_argument("--coarsePth", type=str, help="prediction file coarse flow ")
    p.add_argument("--finePth", type=str, help="prediction file fine flow")
    p.add_argument("--maskPth", type=str, help="prediction file mask")
    p.add_argument("--th", type=float, default=0.95, help="threshold")
    p.add_argument("--dataset", type=str, default="MegaDepth", help="RobotCar or megadepth")
    # evaluation.py's arguments: with --resumePth the pairs are aligned in this process instead of read from files
    p.add_argument("--resumePth", type=str, help="align in-process with this checkpoint instead of reading --finePth/--coarsePth")
    p.add_argument("--kernelSize", type=int, default=7, help="kernel Size")
    p.add_argument("--coarseIter", type=int, default=10000, help="nb iteration in RANSAC")
    p.add_argument("--maskRegionTh", type=float, default=0.01, help="if mask region smaller than this value, stop doing homography")
    p.add_argument("--maxCoarse", type=int, default=10, help="maximum number of coarse alignment")
    p.add_argument("--coarsetolerance", type=float, default=0.05, help="tolerance coarse in RANSAC")
    p.add_argument("--nbScale", type=int, default=7, choices=[3, 5, 7], help="nb scales ")
    p.add_argument("--outDir", type=str, help="also write evaluation.py's files (outDir_Coarse / outDir_Fine)")
    p.add_argument("--segNet", action="store_true", help="whether to use seg net to remove the sky?")
    p.add_argument("--imageNet", action="store_true", help="whether to use seg net imagenet feature?")
    p.add_argument("--scaleR", type=float, default=2, help="scale range ")
    p.add_argument("--engine", default="f16x3", choices=["f16x3", "fp32"], help="fine-network engine")
    sub = p.add_subparsers(title="test dataset", dest="subcommand")
    rc = sub.add_parser("RobotCar", help="parser for training arguments")
    rc.add_argument("--testDir", type=str, default="../../data/RobotCar/imgs/", help="RGB image directory")
    rc.add_argument("--testCSV", type=str, default="../../data/RobotCar/test6511.csv", help="RGB image directory")
    md = sub.add_parser("MegaDepth", help="parser for training arguments")
    md.add_argument("--testDir", type=str, default="../../data/MegaDepth/Test/test1600Pairs", help="RGB image directory")
    md.add_argument("--testCSV", type=str, default="../../data/MegaDepth/Test/test1600Pairs.csv", help="RGB image directory")
    md.add_argument("--beginIndex", type=int, default=0, help="begin index")
    md.add_argument("--endIndex", type=int, default=1600, help="end index")
    return p


def load_models(args):
    """evaluation.py's networks and CoarseAlign from its arguments."""
    from . import coarseAlignFeatMatch, model
    model.set_engine(args.engine)
    network = {"netFeatCoarse": model.FeatureExtractor(), "netCorr": model.CorrNeigh(args.kernelSize),
               "netFlowCoarse": model.NetFlowCoarse(args.kernelSize), "netMatch": model.NetMatchability(args.kernelSize)}
    for key in network:
        network[key].cuda()
    param = torch.load(args.resumePth, map_location="cpu")
    for key in list(param.keys()):
        network[key].load_state_dict(param[key])
        network[key].eval()
    coarseModel = coarseAlignFeatMatch.CoarseAlign(args.nbScale, args.coarseIter, args.coarsetolerance, "Homography", args.minSize,
                                                   2, False, args.scaleR, args.imageNet, args.segNet)
    return coarseModel, network


def print_results(res, matchabilityTH):
    """getResults.py:255-257."""
    for th in matchabilityTH:
        msg = "\nthreshold {:.1f}, precision ".format(th)
        print(msg, res[th][0], res[th][1])


def main(argv=None):
    import pandas as pd
    args = build_parser().parse_args(argv)
    if args.subcommand is None:
        raise SystemExit("corr_results: a dataset sub-command (MegaDepth or RobotCar) is required")
    df = pd.read_csv(args.testCSV, dtype=str)
    print("Evaluation for pixel grid : \n")
    print("-->  ", PIXEL_GRID, "\n")
    if args.resumePth:
        coarseModel, network = load_models(args)
        end = getattr(args, "endIndex", len(df))
        res = evaluate(df, args.testDir, coarseModel, network, args.dataset, args.matchabilityTH, args.th, args.multiH,
                       args.onlyCoarse, args.maxCoarse, args.maskRegionTh, args.segNet, args.minSize, args.outDir,
                       getattr(args, "beginIndex", 0), min(end, len(df)))
    else:
        if args.finePth is None or args.coarsePth is None:
            raise SystemExit("corr_results: --finePth and --coarsePth are required without --resumePth")
        res = get_results(df, args.testDir, args.finePth, args.coarsePth, args.multiH, args.th, args.matchabilityTH, args.dataset,
                          args.onlyCoarse, args.minSize, args.maskPth)
    print_results(res, args.matchabilityTH)
    return res


if __name__ == "__main__":
    main()
