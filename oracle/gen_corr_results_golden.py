"""Generate tests/golden/corr_results.npz by running the reference's evaluation/evalCorr/getResults.py as a script on the CPU:

    python -m oracle.gen_corr_results_golden        # needs the reference checkout ($RF_REFERENCE)

Each case runs the script with ``runpy`` under its own argv, over synthetic PNG images and ``.npy`` hypothesis files written
to a temporary directory.  Harness-side shims only: kornia is absent, so the oracle's ``Warper`` (``warp_oracle.warp_grid``)
stands in for ``kornia.geometry.HomographyWarper``, as ``gen_golden`` does; ``tqdm`` is replaced by a pass-through that,
when the script's loop starts, wraps the script's ``alignmentError`` to record, per call, the matchability threshold, the
selected keypoint indices (``np.where``'s, repeats included) and their distances (restated from the same arguments:
fp32 estimate, fp64 distance), then calls the original.  No reference source is stored; only inputs and outputs.

The images are regenerated from seeds and checked against their SHA-256; the ``.npy`` files, the CSV rows, the printed
lines, the final dictionaries and any exception are stored.  Cases: MegaDepth and RobotCar, ``--multiH`` on and off,
``--onlyCoarse``, ``--matchabilityTH 0 0.5`` on a square map (the broadcast quirk) and on a non-square one (its
RuntimeError), a target of the flow's pixel count in another shape (the flow read through ``.view(1, 1, Ith, Itw)`` at the
flat index) and of another pixel count (the view's RuntimeError), a pair with no files first and in the middle, the KeyError of that rule, and an out-of-range RobotCar index.
Hypothesis counts 1, 3 and 11, one non-finite H and one hypothesis mapping partly outside; keypoints that the MegaDepth
filter drops, on the last row and column, and a negative RobotCar index that wraps.
"""
import contextlib
import hashlib
import importlib.machinery
import io
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import pandas as pd
import PIL.Image as Image
import torch

from . import warp_oracle as WO
from .corr_results_oracle import digest, image
from .gen_golden import REF, save

MIN_SIZE = 64
N_PAIRS = 5
N_KPTS = 40
NH = [1, 3, 11, 3, 3]               # pair 3: hypothesis 1 has a non-finite H; pair 4: hypothesis 0 maps partly outside
SHAPES = {"ns": [((100, 80), (120, 90))] * N_PAIRS,            # both resize to 80 x 64 at minSize 64: h8, w8 = 8, 10
          "sq": [((90, 90), (70, 70))] * N_PAIRS,              # 64 x 64: h8 = w8 = 8
          "tr": [((100, 80), (90, 112))] * N_PAIRS,            # the target resizes to 64 x 80: the 80 x 64 flow's pixel count
          "pc": [((100, 80), (70, 70))] * N_PAIRS}             # the target resizes to 64 x 64, the flow is 80 x 64
FLOW_SIZE = {"ns": (8, 10), "sq": (8, 8), "tr": (8, 10), "pc": (8, 10)}    # (h8, w8) of each shape's hypothesis files
SEED_OFFSET = {"ns": 0, "sq": 50, "tr": 100, "pc": 150}
CASES = [("md_multi", "ns", "md", "MegaDepth", [2], ["--multiH", "--th", "0.5"]),
         ("md_single", "ns", "md", "MegaDepth", [2], []),
         ("rc_multi", "ns", "rc", "RobotCar", [0], ["--multiH", "--th", "0.5", "--dataset", "RobotCar"]),
         ("md_coarse", "ns", "md", "MegaDepth", [], ["--onlyCoarse"]),
         ("sq_mth", "sq", "md", "MegaDepth", [1], ["--multiH", "--th", "0.5", "--matchabilityTH", "0", "0.5"]),
         ("ns_mth", "ns", "md", "MegaDepth", [], ["--multiH", "--matchabilityTH", "0", "0.5"]),
         ("keyerr", "sq", "md", "MegaDepth", [1], ["--matchabilityTH", "0.5"]),
         ("rc_index", "ns", "rcbad", "RobotCar", [], ["--dataset", "RobotCar"]),
         ("view_index", "tr", "md", "MegaDepth", [1], ["--multiH", "--th", "0.5"]),
         ("md_flat", "tr", "mdv", "MegaDepth", [1], ["--multiH", "--th", "0.5"]),
         ("view_err", "pc", "md", "MegaDepth", [], ["--multiH"])]


def _fmt(a):
    return ";".join("%.4f" % v for v in a)


def keypoints(rs, src, tgt, kind):
    """Target keypoints over the original target (its last row and column included) and source keypoints near their
    scaled positions (``mdv``: in the top three quarters of the target).  ``md``: a few outside either image (the MegaDepth filter drops them); ``rc``: one x of -2, which
    truncates to -1 after scaling and wraps; ``rcbad``: also one x beyond the image (numpy's IndexError)."""
    (ws, hs), (wt, ht) = src, tgt
    xb, yb = rs.uniform(0, wt - 1, N_KPTS), rs.uniform(0, ht - 1, N_KPTS)
    xb[0], xb[1], yb[2] = wt - 1e-3, wt - 1e-3, ht - 1e-3
    yb[1] = ht - 1e-3
    xa = xb * ws / wt + rs.normal(0, 1.5, N_KPTS)
    ya = yb * hs / ht + rs.normal(0, 1.5, N_KPTS)
    if kind == "mdv":                                        # target rows inside the transposed flow map as well
        yb *= 0.75
        ya *= 0.75
    if kind in ("md", "mdv"):
        xb[3], ya[4], xa[5], yb[6] = -0.5, hs + 2.0, 0.0, ht + 0.5
    else:
        xb[3] = -2.0
        if kind == "rcbad":
            xb[7] = wt + 50.0
    return xa, ya, xb, yb


def hypotheses(rs, nH, h8, w8, pair):
    Hs = np.stack([np.eye(3) + rs.uniform(-0.04, 0.04, (3, 3)) for _ in range(nH)])
    if pair == 3:
        Hs[1] = np.nan
    if pair == 4:
        Hs[0, 0, 2] += 0.45
    flow = rs.normal(0, 0.03, (nH, 2, h8, w8))
    match = rs.uniform(0, 1, (nH, 2, h8, w8))
    return Hs.astype(np.float32), flow.astype(np.float32), match.astype(np.float32)


class Warper:                          # kornia is absent: the oracle's restatement stands in
    def __init__(self, h, w):
        self.h, self.w = h, w

    def warp_grid(self, H):
        return WO.warp_grid(H, self.h, self.w)


def run_case(script, argv, calls):
    """Run the script once; returns (stdout, exception repr or '')."""
    def tqdm(it, *a, **k):
        g = sys._getframe(1).f_globals
        real = g["alignmentError"]

        def wrapped(wB, hB, wA, hA, XA, YA, XB, YB, flow, match2, pixelGrid):
            estimX = flow.narrow(3, 1, 1).view(1, 1, hB, wB)
            estimY = flow.narrow(3, 0, 1).view(1, 1, hB, wB)
            estimY = ((estimY + 1) * 0.5 * (wA - 1)).squeeze().numpy()
            estimX = ((estimX + 1) * 0.5 * (hA - 1)).squeeze().numpy()
            match = match2.squeeze().numpy()
            xa, ya, xb, yb = XA.astype(np.int64), YA.astype(np.int64), XB.astype(np.int64), YB.astype(np.int64)
            index = np.where(match[yb, xb] > 0.5)[0]
            d = ((estimY[yb[index], xb[index]] - xa[index]) ** 2 + (estimX[yb[index], xb[index]] - ya[index]) ** 2) ** 0.5
            calls.append((g["i"], g["th"], index.astype(np.int64), np.asarray(d, dtype=np.float64)))
            return real(wB, hB, wA, hA, XA, YA, XB, YB, flow, match2, pixelGrid)
        g["alignmentError"] = wrapped
        return iter(it)

    saved = {k: sys.modules.get(k) for k in ("kornia", "kornia.geometry", "tqdm")}
    geo = types.ModuleType("kornia.geometry")
    geo.HomographyWarper = Warper
    kornia = types.ModuleType("kornia")
    kornia.geometry = geo
    tq = types.ModuleType("tqdm")
    tq.__spec__ = importlib.machinery.ModuleSpec("tqdm", None)
    tq.tqdm = tqdm
    sys.modules.update({"kornia": kornia, "kornia.geometry": geo, "tqdm": tq})
    old_argv, out, err = sys.argv, io.StringIO(), ""
    sys.argv = ["getResults.py"] + argv
    try:
        with contextlib.redirect_stdout(out), np.errstate(all="ignore"):
            runpy.run_path(script, run_name="__main__")
    except Exception as e:          # the reference's own error is part of the golden
        err = "%s: %s" % (type(e).__name__, e)
    finally:
        sys.argv = old_argv
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return out.getvalue(), err


def main():
    script = os.path.join(REF, "evaluation", "evalCorr", "getResults.py")
    rs = np.random.RandomState(2026)
    arrs = dict(min_size=np.int64(MIN_SIZE), n_pairs=np.int64(N_PAIRS), cases=np.array([c[0] for c in CASES]))
    data = {}
    for shape in SHAPES:
        for p in range(N_PAIRS):
            (ws, hs), (wt, ht) = SHAPES[shape][p]
            sseed, tseed = 1000 + 2 * p + SEED_OFFSET[shape], 1001 + 2 * p + SEED_OFFSET[shape]
            arrs["img_%s_%d" % (shape, p)] = np.array([ws, hs, sseed, wt, ht, tseed], dtype=np.int64)
            arrs["sha_%s_%d" % (shape, p)] = np.array([digest(image(sseed, ws, hs)), digest(image(tseed, wt, ht))])
            h8, w8 = FLOW_SIZE[shape]
            Hs, flow, match = hypotheses(rs, NH[p], h8, w8, p)
            data[shape, p] = (Hs, flow, match)
            arrs["H_%s_%d" % (shape, p)], arrs["flow_%s_%d" % (shape, p)], arrs["match_%s_%d" % (shape, p)] = Hs, flow, match
        for kind in sorted({c[2] for c in CASES if c[1] == shape}):
            rows = []
            for p in range(N_PAIRS):
                xa, ya, xb, yb = keypoints(rs, *SHAPES[shape][p], kind)
                rows.append(dict(scene="scene%d" % (p % 2) if kind == "md" else "/", source_image="s%d.png" % p,
                                 target_image="t%d.png" % p, XA=_fmt(xa), YA=_fmt(ya), XB=_fmt(xb), YB=_fmt(yb)))
            for c in ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB"):
                arrs["csv_%s_%s_%s" % (shape, kind, c)] = np.array([r[c] for r in rows])
    with tempfile.TemporaryDirectory() as tmp:
        for name, shape, kind, sub, missing, extra in CASES:
            root = os.path.join(tmp, name)
            imgs, fine, coarse = os.path.join(root, "imgs"), os.path.join(root, "fine"), os.path.join(root, "coarse")
            for d in (fine, coarse, os.path.join(imgs, "scene0"), os.path.join(imgs, "scene1")):
                os.makedirs(d)
            cols = {c: list(arrs["csv_%s_%s_%s" % (shape, kind, c)]) for c in ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB")}
            pd.DataFrame(cols, dtype=str).to_csv(os.path.join(root, "test.csv"), index=False)
            for p in range(N_PAIRS):
                ws, hs, sseed, wt, ht, tseed = [int(v) for v in arrs["img_%s_%d" % (shape, p)]]
                d = imgs if cols["scene"][p] == "/" else os.path.join(imgs, cols["scene"][p])
                Image.fromarray(image(sseed, ws, hs)).save(os.path.join(d, "s%d.png" % p))
                Image.fromarray(image(tseed, wt, ht)).save(os.path.join(d, "t%d.png" % p))
                if p in missing:
                    continue
                Hs, flow, match = data[shape, p]
                tag = "%d_%dH.npy" % (p, len(Hs))
                np.save(os.path.join(fine, "flow_" + tag), flow)
                np.save(os.path.join(fine, "mask_" + tag), match)
                np.save(os.path.join(fine, "maskBG_" + tag), np.ones((8 * flow.shape[2], 8 * flow.shape[3]), bool))
                np.save(os.path.join(coarse, "flow_" + tag), Hs)
            argv = extra + ["--minSize", str(MIN_SIZE), "--finePth", fine, "--coarsePth", coarse] + \
                   [sub, "--testDir", imgs, "--testCSV", os.path.join(root, "test.csv")]
            calls = []
            with torch.no_grad():
                stdout, err = run_case(script, argv, calls)
            lines = [l for l in stdout.splitlines() if not l.startswith("Namespace(")]
            arrs["%s_meta" % name] = np.array([shape, kind, sub, ",".join(str(m) for m in missing), " ".join(extra), err])
            arrs["%s_stdout" % name] = np.array(lines)
            arrs["%s_ncalls" % name] = np.int64(len(calls))
            for k, (i, th, index, d) in enumerate(calls):
                arrs["%s_call%d_pair_th" % (name, k)] = np.array([i, th], dtype=np.float64)
                arrs["%s_call%d_index" % (name, k)] = index
                arrs["%s_call%d_dist" % (name, k)] = d
            print(name, err or "ok", len(calls), "calls")
    save("corr_results", **arrs)


if __name__ == "__main__":
    main()
