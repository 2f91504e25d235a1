"""Generate tests/golden/validation_megadepth.npz by running the reference's train/validation.py on the CPU:

    python -m oracle.gen_validation_golden          # needs the reference checkout ($RF_REFERENCE)

Harness-side shims only (``gen_golden.cpu_as_cuda``): ``Image.open`` serves synthetic ``synth.make_pair`` images by file
name, the networks are ``gen_golden._ref_networks``' seeded fine weights, the DataFrame and the coarse affine list are built
here.  The per-keypoint distances are captured by wrapping the module's ``alignmentError``: the wrapper restates its loop on
the same arguments (fp32 estimate, fp64 distance) and then calls the original.  No reference source is stored; only inputs
and outputs.

Five pairs: landscape, portrait, square, a source whose resize rule meets an exact half (128 x 166: 622.5, Python's
half-to-even ``round`` then a floor to 16), and a source and target of different sizes.  One theta maps partly outside the
image; keypoints include the last row and column of the resized target and a negative target index (torch wraps it).  The
reference's ``ResizeMinResolution`` sizes for a sweep of (w, h) are stored beside them.  The images are not stored: they are
``synth.make_pair``'s, regenerated from each pair's spec and checked against its SHA-256.
"""
import hashlib
import os
import sys

import numpy as np
import pandas as pd
import PIL.Image as Image
import torch

from . import synth
from .gen_golden import REF, _load, _ref_networks, cpu_as_cuda, ref_model, save

#            source (w, h), target (w, h), make_pair seed, theta (2 x 3)
PAIRS = [((320, 240), (320, 240), 1, [[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]]),
         ((240, 320), (240, 320), 2, [[0.97, -0.02, -0.04], [0.03, 1.01, 0.02]]),
         ((200, 200), (200, 200), 3, [[1.30, 0.05, 0.35], [-0.04, 1.25, -0.30]]),        # partly outside the source
         ((128, 166), (128, 166), 4, [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]),
         ((300, 225), (240, 300), 5, [[0.95, 0.04, 0.01], [0.02, 1.03, 0.05]])]
N_KPTS = 60
SWEEP = [(w, h) for w in (100, 128, 200, 240, 333, 480, 481, 500, 640, 719, 1024, 1600) for h in (90, 166, 240, 321, 480, 600, 853, 1200)]


def pair_images(spec):
    """The synthetic (source, target) of a pair spec (ws, hs, wt, ht, seed): the images are regenerated, not stored."""
    ws0, hs0, wt0, ht0, seed = [int(v) for v in spec]
    return synth.make_pair(seed, hs0, ws0)[0], synth.make_pair(seed, ht0, wt0)[1]


def pair_digest(src, tgt):
    return hashlib.sha256(np.ascontiguousarray(src).tobytes() + np.ascontiguousarray(tgt).tobytes()).hexdigest()


def _fmt(a):
    return ";".join("%.4f" % v for v in a)


def _keypoints(rs, src_wh, tgt_wh, theta):
    """Target keypoints spread over the target (plus its last column and row, and one negative x), and source keypoints at
    theta's image of them with a few pixels of noise, in the ORIGINAL images' coordinates."""
    (ws0, hs0), (wt0, ht0) = src_wh, tgt_wh
    xb = rs.uniform(0, wt0 - 1, N_KPTS)
    yb = rs.uniform(0, ht0 - 1, N_KPTS)
    xb[0], yb[0] = wt0 - 1e-3, rs.uniform(0, ht0 - 1)        # last column of the resized target
    xb[1], yb[1] = rs.uniform(0, wt0 - 1), ht0 - 1e-3        # last row
    xb[2], yb[2] = wt0 - 1e-3, ht0 - 1e-3                    # the corner
    xb[3] = -0.7                                             # int() -> -1 after scaling: torch wraps to the last column
    gx, gy = 2 * xb / (wt0 - 1) - 1, 2 * yb / (ht0 - 1) - 1
    t = np.asarray(theta, dtype=np.float64)
    px, py = t[0, 0] * gx + t[0, 1] * gy + t[0, 2], t[1, 0] * gx + t[1, 1] * gy + t[1, 2]
    xa = (px + 1) / 2 * (ws0 - 1) + rs.normal(0, 4, N_KPTS)
    ya = (py + 1) / 2 * (hs0 - 1) + rs.normal(0, 4, N_KPTS)
    return xa, ya, xb, yb


def main():
    sys.path[:0] = [os.path.join(REF, "train"), REF]      # validation.py imports model.model from the checkout's root,
    sys.modules.setdefault("downsample", _load("downsample", os.path.join(REF, "model", "downsample.py")))   # and it downsample
    with cpu_as_cuda():
        import validation as V
    net = _ref_networks(ref_model())
    rs = np.random.RandomState(2024)
    images, rows, thetas, srcs, tgts = {}, [], [], [], []
    for i, ((ws0, hs0), (wt0, ht0), seed, theta) in enumerate(PAIRS):
        s, t = pair_images((ws0, hs0, wt0, ht0, seed))
        images["s%d.png" % i], images["t%d.png" % i] = s, t
        srcs.append(s)
        tgts.append(t)
        xa, ya, xb, yb = _keypoints(rs, (ws0, hs0), (wt0, ht0), theta)
        rows.append(dict(scene="scene%d" % (i % 2), source_image="s%d.png" % i, target_image="t%d.png" % i,
                         XA=_fmt(xa), YA=_fmt(ya), XB=_fmt(xb), YB=_fmt(yb)))
        thetas.append(np.asarray(theta, dtype=np.float32))
    df = pd.DataFrame(rows, dtype=str)

    dists, kpts = [], []
    real_err, real_open = V.alignmentError, Image.open

    def wrapped(wB, hB, wA, hA, XA, YA, XB, YB, flow, pixelGrid):
        estimX = flow.narrow(3, 1, 1).view(1, 1, hB, wB)
        estimY = flow.narrow(3, 0, 1).view(1, 1, hB, wB)
        estimY = (estimY + 1) * 0.5 * (wA - 1)
        estimX = (estimX + 1) * 0.5 * (hA - 1)
        d, k = [], []
        for j in range(len(XB)):
            xa, ya, xb, yb = int(XA[j]), int(YA[j]), int(XB[j]), int(YB[j])
            d.append(((estimY[0, 0, yb, xb].item() - xa) ** 2 + (estimX[0, 0, yb, xb].item() - ya) ** 2) ** 0.5)
            k.append((xa, ya, xb, yb))
        dists.append(np.array(d, dtype=np.float64))
        kpts.append(np.array(k, dtype=np.int32))
        return real_err(wB, hB, wA, hA, XA, YA, XB, YB, flow, pixelGrid)

    V.alignmentError = wrapped
    Image.open = lambda path, *a, **k: Image.fromarray(images[os.path.basename(path)])
    try:
        with cpu_as_cuda(), torch.no_grad():
            prec = V.validation(df, "/nonexistent", thetas, net, "grad")
            sweep = []
            for (w, h) in SWEEP:
                I, _, _ = V.ResizeMinResolution(480, Image.new("RGB", (w, h)), "0", "0", 16)
                sweep.append((w, h) + I.size)
    finally:
        V.alignmentError, Image.open = real_err, real_open
        del sys.path[:2]
    arrs = dict(prec=np.asarray(prec, dtype=np.float64), sweep=np.array(sweep, dtype=np.int64), n_pairs=np.int64(len(PAIRS)),
                feat_seed=np.int64(0), flow_seed=np.int64(1))
    for i in range(len(PAIRS)):
        (ws0, hs0), (wt0, ht0), seed, _ = PAIRS[i]
        arrs["spec%d" % i] = np.array([ws0, hs0, wt0, ht0, seed], dtype=np.int64)
        arrs["sha%d" % i] = np.array(pair_digest(srcs[i], tgts[i]))
        arrs["theta%d" % i] = thetas[i]
        arrs["dist%d" % i], arrs["kpts%d" % i] = dists[i], kpts[i]
        for c in ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB"):
            arrs["%s%d" % (c, i)] = np.array(rows[i][c])
    save("validation_megadepth", **arrs)


if __name__ == "__main__":
    main()
