"""Throughput of evalCorr's getResults on the device (``corr_results.get_results``) against today's per-pair path on the same
files, and the time of ``rf_corr_keypoints`` against the dense composition and merge it replaces.

    python tools/corr_results_profile.py [--pairs 24] [--nH 3] [--kpts 400] [--out result.json]

  pairs/s   : ``corr_results.get_results`` over a synthetic MegaDepth-shaped dataset (960 x 720 PNG files, resized to
              640 x 480: 60 x 80 ``.npy`` hypothesis files with ``--nH`` hypotheses, ``--kpts`` keypoints per pair, ``--multiH``
              at th 0.95), against getResults.py's per-pair statements on this package's modules: both images decoded and
              LANCZOS-resized on the host, ``results.getFlow_from_files`` (the dense composition and merge on the device, the
              maps copied to the host) and ``results.alignment_error``.  One warm-up pass each, then the timed pass, each ended
              by a device synchronise.  Both must print the same table.
  kernels   : CUDA events around 100 calls each at 480 x 640 with nH = 1 and 11: ``rf_corr_keypoints`` against
              ``pipeline._compose_all`` + ``merge_first_wins`` + the gather at the keypoints (on the device, nothing copied).

Prints one JSON object with the GPU's name and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import PIL.Image as Image
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ransac_flow_b200 as rf  # noqa: E402

CR = rf.corr_results


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def hypotheses(rs, nH, h8, w8):
    Hs = np.stack([np.eye(3) + rs.uniform(-0.05, 0.05, (3, 3)) for _ in range(nH)]).astype(np.float32)
    flow = rs.normal(0, 0.03, (nH, 2, h8, w8)).astype(np.float32)
    match = rs.uniform(0, 1, (nH, 2, h8, w8)).astype(np.float32)
    return Hs, flow, match


def dataset(root, pairs, nH, kpts):
    import pandas as pd
    rs = np.random.RandomState(0)
    fine, coarse = os.path.join(root, "fine"), os.path.join(root, "coarse")
    for d in (fine, coarse, os.path.join(root, "imgs", "scene0")):
        os.makedirs(d, exist_ok=True)
    rows = []
    f = lambda a: ";".join("%.3f" % v for v in a)
    for p in range(pairs):
        for name in ("s%d.png" % p, "t%d.png" % p):
            Image.fromarray(rs.randint(0, 256, (720, 960, 3), dtype=np.uint8)).save(os.path.join(root, "imgs", "scene0", name))
        xb, yb = rs.uniform(1, 958, kpts), rs.uniform(1, 718, kpts)
        rows.append(dict(scene="scene0", source_image="s%d.png" % p, target_image="t%d.png" % p,
                         XA=f(xb + rs.normal(0, 6, kpts)), YA=f(yb + rs.normal(0, 6, kpts)), XB=f(xb), YB=f(yb)))
        Hs, flow, match = hypotheses(rs, nH, 60, 80)
        tag = "%d_%dH.npy" % (p, nH)
        np.save(os.path.join(fine, "flow_" + tag), flow)
        np.save(os.path.join(fine, "mask_" + tag), match)
        np.save(os.path.join(fine, "maskBG_" + tag), np.ones((480, 640), bool))
        np.save(os.path.join(coarse, "flow_" + tag), Hs)
    return pd.DataFrame(rows, dtype=str), os.path.join(root, "imgs"), fine, coarse


def today(df, testDir, fine, coarse, multiH, th):
    """getResults.py's loop with matchabilityTH [0] as it runs today: decode + LANCZOS resize, the dense getFlow, the host
    alignmentError."""
    prec, valid = np.zeros(8), 0
    flowList = os.listdir(fine)
    for i in range(len(df)):
        path = lambda n: CR.image_path(testDir, df["scene"][i], n)
        Is = Image.open(path(df["source_image"][i])).convert("RGB")
        It = Image.open(path(df["target_image"][i])).convert("RGB")
        ws, hs = CR.resize_min_resolution_size(*Is.size)
        wt, ht = CR.resize_min_resolution_size(*It.size)
        Is, It = Is.resize((ws, hs), resample=Image.LANCZOS), It.resize((wt, ht), resample=Image.LANCZOS)
        (Xs, Ys, Xt, Yt), _, _ = CR.pair_keypoints(df, i, testDir, "MegaDepth", sizes=((960, 720), (960, 720)))
        flow, match = rf.results.getFlow_from_files(i, fine, flowList, coarse, fine, multiH, th)
        c, n = rf.results.alignment_error(wt, ht, ws, hs, Xs, Ys, Xt, Yt, flow, torch.ones(match.size()), CR.PIXEL_GRID)
        prec, valid = prec + c, valid + n
    return prec / valid


def pairs_per_s(fn, pairs):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return pairs / (time.perf_counter() - t), out


def kernel_times(nH, kpts, reps=100):
    rs = np.random.RandomState(nH)
    Hs, flow, match = hypotheses(rs, nH, 60, 80)
    H, W = 480, 640
    kp = np.stack([rs.randint(0, W, kpts), rs.randint(0, H, kpts), rs.randint(0, W, kpts), rs.randint(0, H, kpts)], 1).astype(np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    f8, m8, Hm, kd = dev(flow), dev(match), dev(Hs).reshape(-1, 9), dev(kp)
    cnt = torch.tensor([kpts], dtype=torch.int32, device="cuda")
    sc = CR.CorrScores([0], 0.95, True, False)
    yb, xb = kd[:, 3].long(), kd[:, 2].long()

    def device():
        CR.corr_keypoints(f8, m8, Hm, (H, W), (H, W), kd, cnt, sc.acc, sc.err, CR.PIXEL_GRID, [0], [0], 0.95, True, False)

    def dense():
        f, m = rf.pipeline._compose_all(f8, Hm.view(-1, 3, 3), m8, H, W)
        fg, mg, _ = rf.pipeline.merge_first_wins(f, m.permute(0, 2, 3, 1), 0.95, True)
        return fg[0, yb, xb], mg[0, yb, xb]

    out = {}
    for name, fn in (("rf_corr_keypoints", device), ("compose_all_merge_gather", dense)):
        for _ in range(5):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        out[name + "_us"] = a.elapsed_time(b) * 1000.0 / reps
    return dict(size="480x640", nH=nH, kpts=kpts, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=24)
    ap.add_argument("--nH", type=int, default=3)
    ap.add_argument("--kpts", type=int, default=400)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "corr_results_profile needs a GPU"
    res = dict(gpu_info(), pairs=args.pairs, nH=args.nH, kpts_per_pair=args.kpts)
    with tempfile.TemporaryDirectory() as root:
        df, imgs, fine, coarse = dataset(root, args.pairs, args.nH, args.kpts)
        res["device_pairs_per_s"], r_dev = pairs_per_s(
            lambda: CR.get_results(df, imgs, fine, coarse, True, 0.95, [0], "MegaDepth"), args.pairs)
        res["today_pairs_per_s"], p_today = pairs_per_s(lambda: today(df, imgs, fine, coarse, True, 0.95), args.pairs)
        res["prec_device"], res["prec_today"] = list(map(float, r_dev[0][0])), list(map(float, p_today))
    res["kernels"] = [kernel_times(1, args.kpts), kernel_times(11, args.kpts)]
    res["gpu_after"] = gpu_info()["nvidia_smi"]
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
