"""MegaDepth validation (train/validation.py) on the device: the ``valPrec@8`` that train.py computes after every epoch
(train.py:271) and that picks ``BestModel.pth`` (train.py:289), for scoring and choosing fine-flow checkpoints.

  ResizeMinResolution : validation.py:16-29 (PIL LANCZOS to min side 480, ``round(w / ratio) // 16 * 16`` with Python's
                        half-to-even ``round`` and a FLOOR to the stride: not ``pipeline.fine_sizes``); keypoints scaled as
                        float32 arrays, truncated later by ``int()``
  validate_pair       : validation.py:74-110 for one pair with nothing read back: the original uint8 images resized on the
                        device (``ops.resize_lanczos_u8``), ``rf_affine_sample_u8`` (affine_grid + ToTensor + grid_sample of the
                        source, written into the source's half of the two-image batch) and ``rf_preproc_u8`` (the target's
                        half), the two-image fine features + ``l2norm``, the one volume ``CorrNeigh(featt, featsSample)``, the
                        ``NetFlowCoarse`` trunk + ``softmax_flow``, and ``rf_val_keypoints``: the x8 upsampling, the grid, the
                        clamp, the composition with the affine grid and ``alignmentError`` at the keypoints only
  validation          : validation.py:56-110 over a DataFrame; one device read, at the end

Decoding, CSV parsing and the keypoint truncation stay on the host, as the reference does them; with no synchronisation in
the loop, decoding the next pair overlaps the GPU.  Each pair's inputs go up in one copy from a ring of pinned staging
buffers, each reused only after the event recorded behind its copy has completed.

The grid the flow is added to is the reference's CPU ``torch.linspace`` (validation.py:93-95); ATen's AVX2 / AVX-512 CPU
kernel computes it with one FMA per value, as the kernels' ``lin11`` does.  The affine grid's product with theta is a cuBLAS
``bmm`` in the reference, so the composed flow matches it to a few ulps, not bit for bit.
"""
import os

import numpy as np
import PIL.Image as Image
import torch

from . import model, ops
from ._lib import check, lib, need_cuda, ptr, stream
from .ops import Ragged

MIN_SIZE, STRIDE_NET = 480, 16                                              # validation.py:60-61
PIXEL_GRID = np.around(np.logspace(0, np.log10(36), 8).reshape(-1, 8))      # validation.py:64: [1, 2, 3, 5, 8, 13, 22, 36]
NO_ERROR = 2 ** 31 - 1                                                      # the error word before any out-of-range index
_I32 = np.iinfo(np.int32)


# --------------------------------------------------------------------------- host rules (the reference's, on numpy)
def resize_min_resolution_size(w, h, minSize=MIN_SIZE, strideNet=STRIDE_NET):
    """validation.py:22-24: the (w, h) ``ResizeMinResolution`` resizes a w x h image to."""
    ratio = min(w / float(minSize), h / float(minSize))
    new_w, new_h = round(w / ratio), round(h / ratio)
    return new_w // strideNet * strideNet, new_h // strideNet * strideNet


def scale_keypoints(x, y, w, h, new_w, new_h):
    """validation.py:18-19,26-29: the ``;``-separated coordinate strings of a w x h image as float32 arrays, scaled to
    new_w x new_h (float32 times a Python float stays float32)."""
    x = np.array(list(map(float, x.split(";")))).astype(np.float32)
    y = np.array(list(map(float, y.split(";")))).astype(np.float32)
    return x * (new_w / float(w)), y * (new_h / float(h))


def ResizeMinResolution(minSize, I, x, y, strideNet):
    """validation.py:16-29 (PIL image in, PIL image and float32 keypoints out)."""
    w, h = I.size
    new_w, new_h = resize_min_resolution_size(w, h, minSize, strideNet)
    x, y = scale_keypoints(x, y, w, h, new_w, new_h)
    return I.resize((new_w, new_h), resample=Image.LANCZOS), x, y


def _index(i, size, dim):
    """torch's rule for one integer index: [-size, size) is valid, a negative one wraps once."""
    if not -size <= i < size:
        raise IndexError("index %d is out of bounds for dimension %d with size %d" % (i, dim, size))
    return i + size if i < 0 else i


def alignmentError(wB, hB, wA, hA, XA, YA, XB, YB, flow, pixelGrid):
    """validation.py:33-53 on a full (1, hB, wB, 2) flow (CPU or CUDA): the estimate in fp32, the distance in fp64, the
    strict compare with ``pixelGrid``.  Returns (counts per threshold, number of keypoints)."""
    f = flow.detach().reshape(hB, wB, 2).cpu().numpy() if torch.is_tensor(flow) else np.asarray(flow).reshape(hB, wB, 2)
    one, half = np.float32(1), np.float32(0.5)
    xaH, yaH, xa, ya = [], [], [], []
    for j in range(len(XB)):
        a, b, xb, yb = int(XA[j]), int(YA[j]), int(XB[j]), int(YB[j])
        r, c = _index(yb, hB, 2), _index(xb, wB, 3)
        xaH.append((f[r, c, 0] + one) * half * np.float32(wA - 1))
        yaH.append((f[r, c, 1] + one) * half * np.float32(hA - 1))
        xa.append(a)
        ya.append(b)
    dx = np.array(xaH, dtype=np.float64) - np.array(xa, dtype=np.float64)
    dy = np.array(yaH, dtype=np.float64) - np.array(ya, dtype=np.float64)
    pixelDiff = np.sqrt(dx * dx + dy * dy)
    return np.sum(pixelDiff.reshape((-1, 1)) < pixelGrid, axis=0), len(pixelDiff)


def truncate_keypoints(XA, YA, XB, YB, hB, wB):
    """alignmentError's ``int()`` of each coordinate (validation.py:42), as int32 rows (xa, ya, xb, yb).  Raises what the
    reference raises on its own: the IndexError of a short coordinate array, or the ValueError / OverflowError of ``int()``
    on a non-finite coordinate, after the IndexError of an earlier keypoint's out-of-range target index."""
    n = len(XB)
    for arr in (XA, YA, YB):
        if len(arr) < n:
            raise IndexError("index %d is out of bounds for axis 0 with size %d" % (len(arr), len(arr)))
    cols = np.stack([np.asarray(a[:n], dtype=np.float32) for a in (XA, YA, XB, YB)], axis=1).reshape(n, 4)
    bad = ~np.isfinite(cols).all(axis=1)
    if bad.any():
        j0 = int(np.argmax(bad))
        for j in range(j0):
            _index(int(cols[j, 3]), hB, 2), _index(int(cols[j, 2]), wB, 3)
        [int(v) for v in cols[j0]]                                  # the reference's own ValueError / OverflowError
    t = np.trunc(cols.astype(np.float64))
    return np.clip(t, _I32.min, _I32.max).astype(np.int32)         # beyond int32 a target index is out of range either way


def check_theta(theta):
    """``inPklCoarse[i]`` as the reference's ``F.affine_grid`` + ``F.grid_sample`` accept it: a (2, 3) float32 array."""
    t = theta if torch.is_tensor(theta) else torch.from_numpy(np.asarray(theta))
    if not t.is_floating_point():                                       # F.affine_grid's checks, in its order
        raise ValueError("Expected theta to have floating point type, but got %s" % t.dtype)
    if tuple(t.shape) != (2, 3):
        raise ValueError("Expected a batch of 2D affine matrices of shape Nx2x3 for size [1, 3, H, W]. Got %s."
                         % str(t.unsqueeze(0).shape))
    if t.dtype != torch.float32:                                        # then F.grid_sample's
        raise RuntimeError("grid_sampler(): expected input and grid to have same dtype, but input has float and grid has %s"
                           % str(t.dtype).replace("torch.", ""))
    return t


# --------------------------------------------------------------------------- kernel entries
def affine_sample_u8(theta, src, h, w, out=None):
    """``F.grid_sample(ToTensor(src), F.affine_grid(theta, (1, 3, h, w)))`` in one kernel, as fp32 NHWC rows [h * w, 3]:
    theta 6 float32 values on the device (read there), ``src`` a uint8 (Hin, Win, 3) CUDA image."""
    need_cuda(theta, src, out)
    if theta.dtype != torch.float32 or theta.numel() != 6 or not theta.is_contiguous():
        raise ValueError("affine_sample_u8: theta must be 6 contiguous float32 values")
    if src.dtype != torch.uint8 or src.dim() != 3 or src.shape[2] != 3 or not src.is_contiguous():
        raise ValueError("affine_sample_u8: src must be a contiguous uint8 (H, W, 3) image")
    if out is None:
        out = torch.empty((h * w, 3), device=src.device, dtype=torch.float32)
    elif out.dtype != torch.float32 or out.numel() != h * w * 3 or not out.is_contiguous():
        raise ValueError("affine_sample_u8: out must be %d contiguous float32 values" % (h * w * 3))
    check(lib.rf_affine_sample_u8(ptr(theta), ptr(src), int(src.shape[0]), int(src.shape[1]), int(h), int(w), ptr(out), stream()))
    return out


def new_counts(device=None):
    """A fresh accumulator for ``val_keypoints``: int64 [T + 2] on the device, the T + 1 counts (keypoints below each of
    ``PIXEL_GRID``'s T thresholds, then the keypoints scored) followed by the error word (its low 32 bits: the first pair
    with an out-of-range target index, ``NO_ERROR`` if none)."""
    acc = torch.zeros(PIXEL_GRID.size + 2, dtype=torch.int64, device=device or torch.device("cuda", torch.cuda.current_device()))
    acc[-1] = NO_ERROR
    return acc


def val_keypoints(flowDown8, theta, size_t, size_s, kpts, count, counts, pair=0, dist_out=None, flow_out=None,
                  thresholds=PIXEL_GRID):
    """``rf_val_keypoints``: flowDown8 (1, 2, h8, w8) fp32; theta 6 float32; ``size_t`` = (H, W) of the target, ``size_s`` =
    (hA, wA) of the resized source; kpts int32 (capacity, 4) = (xa, ya, xb, yb) and ``count`` an int32 [1], both on the
    device; ``counts`` a ``new_counts`` accumulator.  ``dist_out`` (capacity,) fp64 / ``flow_out`` (capacity, 4) fp32:
    optional per-keypoint distances / (clamped fine flow, composed flow) pairs."""
    need_cuda(flowDown8, theta, kpts, count, counts, dist_out, flow_out)
    th = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float64).reshape(-1))
    if flowDown8.dtype != torch.float32 or flowDown8.dim() != 4 or tuple(flowDown8.shape[:2]) != (1, 2) or not flowDown8.is_contiguous():
        raise ValueError("val_keypoints: flowDown8 must be a contiguous float32 (1, 2, h8, w8) tensor")
    if theta.dtype != torch.float32 or theta.numel() != 6 or not theta.is_contiguous():
        raise ValueError("val_keypoints: theta must be 6 contiguous float32 values")
    if kpts.dtype != torch.int32 or kpts.dim() != 2 or kpts.shape[1] != 4 or not kpts.is_contiguous():
        raise ValueError("val_keypoints: kpts must be a contiguous int32 (n, 4) tensor")
    if count.dtype != torch.int32 or count.numel() != 1:
        raise ValueError("val_keypoints: count must be one int32")
    if counts.dtype != torch.int64 or counts.numel() != th.size + 2 or not counts.is_contiguous():
        raise ValueError("val_keypoints: counts must be a contiguous int64 [T + 2] accumulator (new_counts)")
    cap = int(kpts.shape[0])
    for name, t, shape in (("dist_out", dist_out, (cap,)), ("flow_out", flow_out, (cap, 4))):
        if t is not None and (tuple(t.shape) != shape or t.dtype != (torch.float64 if name == "dist_out" else torch.float32)
                              or not t.is_contiguous()):
            raise ValueError("val_keypoints: %s must be a contiguous %s tensor" % (name, shape))
    _, _, h8, w8 = flowDown8.shape
    err = counts[-1:].view(torch.int32)[:1]                                 # the error word: the low half of the last entry
    check(lib.rf_val_keypoints(ptr(flowDown8), int(h8), int(w8), ptr(theta), int(size_t[0]), int(size_t[1]), int(size_s[1]),
                               int(size_s[0]), ptr(kpts), ptr(count), cap, int(pair), th.ctypes.data, int(th.size), ptr(counts),
                               ptr(err), ptr(dist_out), ptr(flow_out), stream()))


def read_counts(host):
    """(counts [T + 1], first failing pair or None) of an accumulator read back to the host."""
    host = np.asarray(host, dtype=np.int64)
    err = int(host[-1:].view(np.int32)[0])
    return host[:-1], (None if err == NO_ERROR else err)


# --------------------------------------------------------------------------- pinned staging
class _Staging:
    """A ring of pinned host buffers, each uploaded with one asynchronous copy per pair and reused only once the event
    recorded behind that copy has completed."""

    def __init__(self, slots=3):
        self.bufs = [None] * slots
        self.events = [None] * slots
        self.k = 0

    def upload(self, parts, device):
        """``parts``: numpy arrays; returns their bytes on ``device`` (one uint8 tensor) and each part's byte offset (16-byte
        aligned)."""
        offs, n = [], 0
        for a in parts:
            offs.append(n)
            n += (a.nbytes + 15) // 16 * 16
        k = self.k
        self.k = (k + 1) % len(self.bufs)
        if self.events[k] is not None and not self.events[k].query():
            self.events[k].synchronize()                 # only when the GPU is this many pairs behind the host
        if self.bufs[k] is None or self.bufs[k].numel() < n:
            self.bufs[k] = torch.empty(max(n, 1 << 20), dtype=torch.uint8).pin_memory()
        host = self.bufs[k].numpy()
        for a, o in zip(parts, offs):
            host[o:o + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
        dev = torch.empty(max(n, 16), dtype=torch.uint8, device=device)
        dev[:n].copy_(self.bufs[k][:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        self.events[k] = ev
        return dev, offs


_staging = {}


def _staging_for(device):
    d = torch.device(device).index
    if d not in _staging:
        _staging[d] = _Staging()
    return _staging[d]


def _view(dev, off, dtype, shape):
    n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
    return dev[off:off + n].view(dtype).view(shape)


# --------------------------------------------------------------------------- the pair
def validate_pair(network, Is_u8, It_u8, theta, kpts, counts, pair=0, dist_out=None, flow_out=None):
    """validation.py:74-110 for one pair, queued on the current stream with nothing read back.  ``Is_u8`` / ``It_u8``: the
    ORIGINAL source / target as uint8 (H, W, 3) numpy arrays; ``theta`` the (2, 3) float32 ``inPklCoarse[i]``; ``kpts`` int32
    (n, 4) = ``truncate_keypoints`` of the keypoints scaled to the resized images; ``counts`` a ``new_counts`` accumulator;
    ``pair`` the index an out-of-range keypoint records.  ``dist_out`` / ``flow_out``: see ``val_keypoints``."""
    theta = check_theta(theta)
    Is_u8, It_u8 = np.asarray(Is_u8, dtype=np.uint8), np.asarray(It_u8, dtype=np.uint8)
    kpts = np.ascontiguousarray(np.asarray(kpts, dtype=np.int32).reshape(-1, 4))
    n = kpts.shape[0]
    ws, hs = resize_min_resolution_size(Is_u8.shape[1], Is_u8.shape[0])
    wt, ht = resize_min_resolution_size(It_u8.shape[1], It_u8.shape[0])
    device = counts.device
    with torch.no_grad(), torch.cuda.device(device):
        dev, o = _staging_for(device).upload([Is_u8, It_u8, theta.numpy(), np.array([n], np.int32), kpts], device)
        Is = _view(dev, o[0], torch.uint8, Is_u8.shape)
        It = _view(dev, o[1], torch.uint8, It_u8.shape)
        th = _view(dev, o[2], torch.float32, (6,))
        cnt = _view(dev, o[3], torch.int32, (1,))
        kp = _view(dev, o[4], torch.int32, (n, 4))
        Isr = ops.resize_lanczos_u8(Is, ws, hs, non_blocking=True)
        Itr = ops.resize_lanczos_u8(It, wt, ht, non_blocking=True)
        P = ht * wt
        x = torch.empty((2 * P, 3), device=device, dtype=torch.float32)     # [IsSample ; ItTensor], NHWC rows
        affine_sample_u8(th, Isr, ht, wt, out=x[:P])
        check(lib.rf_preproc_u8(ptr(Itr), P, 0, ptr(x[P:]), stream()))
        f = network["netFeatCoarse"].forward_ragged(Ragged(x, [(ht, wt)] * 2))
        f = Ragged(ops.l2norm(f.data), f.hw)
        m = f.data.shape[0] // 2
        featsSample, featt = Ragged(f.data[:m], f.hw[:1]), Ragged(f.data[m:], f.hw[1:])
        k, ld = network["netCorr"].kernelSize, network["netFlowCoarse"].CORR_LD
        tc = model.fine_engine()
        if tc == ops.ENGINE_SPLIT:                                            # corr21 = netCorr(featt, featsSample)
            corr21, _ = ops.corr_neigh_pair_split(featt, featsSample, k, ld, want_both=False)
        else:
            corr21 = ops.corr_neigh(featt, featsSample, k, ld, tc)
        flowDown8 = network["netFlowCoarse"].forward_ragged(corr21)
        if n:
            val_keypoints(flowDown8, th, (ht, wt), (hs, ws), kp, cnt, counts, pair, dist_out, flow_out)
    return flowDown8


def pair_inputs(df, i, valDir, inPklCoarse):
    """Row i of the DataFrame as the reference reads it, in its order, so that a bad row raises what the reference raises
    first: the two images and their keypoints (validation.py:74-90), ``inPklCoarse[i]`` as ``F.affine_grid`` and
    ``F.grid_sample`` check it (:97-99), then the keypoints' ``int()`` (:42).  Returns the two RGB images as uint8 arrays,
    theta and the int32 keypoint rows in the resized images."""
    scene = df["scene"][i]
    Is = np.asarray(Image.open(os.path.join(os.path.join(valDir, scene), df["source_image"][i])).convert("RGB"))
    It = np.asarray(Image.open(os.path.join(os.path.join(valDir, scene), df["target_image"][i])).convert("RGB"))
    ws, hs = resize_min_resolution_size(Is.shape[1], Is.shape[0])
    wt, ht = resize_min_resolution_size(It.shape[1], It.shape[0])
    Xs, Ys = scale_keypoints(df["XA"][i], df["YA"][i], Is.shape[1], Is.shape[0], ws, hs)
    Xt, Yt = scale_keypoints(df["XB"][i], df["YB"][i], It.shape[1], It.shape[0], wt, ht)
    theta = check_theta(inPklCoarse[i])
    return Is, It, theta, truncate_keypoints(Xs, Ys, Xt, Yt, ht, wt)


def queue_validation(df, valDir, inPklCoarse, network, acc, dists=None, prog=None):
    """The loop of ``validation``: every row queued on the current stream into the accumulator ``acc`` (``new_counts``),
    nothing read back.  ``dists``: a list that receives each pair's device fp64 distances; ``prog[0]``: the row in progress."""
    dev = acc.device
    for i in range(len(df)):
        if prog is not None:
            prog[0] = i
        Is, It, theta, kpts = pair_inputs(df, i, valDir, inPklCoarse)
        d = torch.empty(len(kpts), dtype=torch.float64, device=dev) if dists is not None else None
        validate_pair(network, Is, It, theta, kpts, acc, pair=i, dist_out=d)
        if dists is not None:
            dists.append(d)


def validation(df, valDir, inPklCoarse, network, trainMode, dist_out=None):
    """validation.py:56-110: the float64 8-vector ``precAllAlign / totalAlign`` over the whole DataFrame (``nan`` without a
    keypoint, as numpy gives).  ``network``: dict of this package's ``model`` modules; ``trainMode`` is accepted and ignored,
    as in the reference.  The device is read once, at the end; an out-of-range keypoint raises IndexError for the first pair
    that has one, where the reference raises.  ``dist_out``: a list that receives each pair's fp64 distances."""
    for key in list(network.keys()):
        network[key].eval()
    acc = new_counts()
    dists = [] if dist_out is not None else None
    prog = [0]
    try:
        queue_validation(df, valDir, inPklCoarse, network, acc, dists, prog)
    except Exception:
        _, err = read_counts(acc.cpu().numpy())          # an earlier pair's out-of-range index is what the reference raised
        if err is not None and err < prog[0]:
            raise IndexError("pair %d: a keypoint index is out of bounds of the target" % err) from None
        raise
    counts, err = read_counts(acc.cpu().numpy())          # the one read of the loop
    if err is not None:
        raise IndexError("pair %d: a keypoint index is out of bounds of the target" % err)
    if dist_out is not None:
        dist_out.extend(d.cpu().numpy() for d in dists)
    precAllAlign = np.zeros(PIXEL_GRID.size) + counts[:-1]
    totalAlign = int(counts[-1])
    with np.errstate(invalid="ignore"):
        return precAllAlign / totalAlign


# --------------------------------------------------------------------------- CLI
def load_network(pth, kernelSize=7):
    """A train.py checkpoint's fine networks (``netFeatCoarse``, ``netCorr``, ``netFlowCoarse``) in this package's modules."""
    param = torch.load(pth, map_location="cpu")
    network = {"netFeatCoarse": model.FeatureExtractor(), "netCorr": model.CorrNeigh(kernelSize),
               "netFlowCoarse": model.NetFlowCoarse(kernelSize)}
    for key, net in network.items():
        if key in param:                                 # CorrNeigh has no parameters
            net.load_state_dict(param[key])
        net.cuda()
        net.eval()
    return network


def main(argv=None):
    import argparse
    import pickle

    import pandas as pd
    p = argparse.ArgumentParser(description="MegaDepth validation (train/validation.py) of fine-flow checkpoints on the GPU")
    p.add_argument("--valImgDir", required=True, help="validation image directory (one sub-directory per scene)")
    p.add_argument("--valCSV", required=True, help="csv of correspondences (scene, source_image, target_image, XA, YA, XB, YB)")
    p.add_argument("--inPklCoarse", required=True, help="pickled list of the 2 x 3 float32 coarse affine transformations")
    p.add_argument("--resumePth", required=True, nargs="+", help="checkpoints to score")
    p.add_argument("--kernelSize", type=int, default=7)
    p.add_argument("--engine", default="f16x3", choices=["f16x3", "fp32"])
    args = p.parse_args(argv)
    model.set_engine(args.engine)
    df = pd.read_csv(args.valCSV, dtype=str)
    with open(args.inPklCoarse, "rb") as f:
        inPklCoarse = pickle.load(f)
    best, bestPrec = None, 0
    for pth in args.resumePth:
        prec = validation(df, args.valImgDir, inPklCoarse, load_network(pth, args.kernelSize), None)
        print("%s\tPrec@[1,2,3,5,8,13,22,36] %s\tvalPrec@8 : %.9f" % (pth, " ".join("%.6f" % v for v in prec), prec[4]), flush=True)
        if prec[4] > bestPrec:                           # train.py:289
            best, bestPrec = pth, prec[4]
    print("best\t%s\tvalPrec@8 : %.9f" % (best, bestPrec) if best is not None else "best\tnone", flush=True)
    return best


if __name__ == "__main__":
    main()
