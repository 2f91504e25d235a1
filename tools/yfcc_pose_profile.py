"""Time evalYFCC's pose metric on the device: rf_yfcc_matches + rf_essential_ransac + rf_recover_pose per pair, on seeded
synthetic 480 x 640 composed flows with N ~ 10 k / 100 k / 300 k matched pixels (outlier ratios 0.1 / 0.5), through the same
calls as ``results.yfcc_pose`` (match buffers of H * W rows, N on the device), with CUDA events (median of repeated
runs after warm-up).  Reports the RANSAC iterations used, the models scored, and fp64 Sampson evaluations per second; times
cv2.findEssentialMat + cv2.recoverPose on the same points when cv2 is importable.

    python tools/yfcc_pose_profile.py [--reps 10] [--out results.json] [--method ransac|8point]

``--method 8point`` times the non-RANSAC branch instead (results.yfcc_pose_8point's calls): the three moment passes and the
one-warp tail of rf_fundamental_8point alone, and the whole matches + findFundamentalMat + recoverPose path, next to
cv2.findFundamentalMat + cv2.recoverPose when cv2 is importable.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ransac_flow_b200 as rf  # noqa: E402

THR = 0.0005


H_IMG, W_IMG = 480, 640        # the driver's target size at minSize 480: the match buffers hold H * W rows


def flow_inputs(N, outlier, seed):
    """A 480 x 640 composed flow / binary map with N matched pixels (a random subset, row-major order as the driver reads them)
    following a smooth-depth two-view scene, a fraction ``outlier`` of them displaced at random; the intrinsics as norm_kp's
    (cx, cy, fx, fy)."""
    rs = np.random.RandomState(seed)
    H, W = H_IMG, W_IMG
    norm = ((W - 1) / 2.0, (H - 1) / 2.0, 500.0, 500.0)
    ang = rs.uniform(-0.1, 0.1, 3)
    Kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]])
    import scipy.linalg
    R = scipy.linalg.expm(Kx)
    t = rs.uniform(-0.4, 0.4, 3)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    d = 4 + 0.8 * np.sin(xs / W * 3) + 0.6 * np.cos(ys / H * 2)
    X = np.stack([(xs - norm[0]) / norm[2] * d, (ys - norm[1]) / norm[3] * d, d], -1) @ R.T + t
    xa = norm[2] * X[..., 0] / X[..., 2] + norm[0]
    ya = norm[3] * X[..., 1] / X[..., 2] + norm[1]
    flow = np.stack([2 * xa / (W - 1) - 1, 2 * ya / (H - 1) - 1], -1)
    mask = np.zeros(H * W, np.uint8)
    sel = rs.choice(H * W, N, replace=False)
    mask[sel] = 1
    out = rs.choice(sel, int(round(outlier * N)), replace=False)
    flow.reshape(-1, 2)[out] = rs.uniform(-1, 1, (len(out), 2))
    return (torch.from_numpy(flow.astype(np.float32)).cuda(), torch.from_numpy(mask.reshape(H, W)).cuda(), norm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    ap.add_argument("--method", default="ransac", choices=["ransac", "8point"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ops = rf.ops
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    try:
        import cv2
    except ImportError:
        cv2 = None
    rows = []
    if args.method == "8point":
        return profile_8point(args, ops, q, cv2)
    for N in (10000, 100000, 300000):
        for outlier in (0.1, 0.5):
            flow, mask, norm = flow_inputs(N, outlier, seed=N + int(outlier * 10))
            size = (W_IMG, H_IMG)

            def once():
                # results.yfcc_pose's device path: the RANSAC and recoverPose buffers have H * W rows, N of them matches
                pts1, pts2, Nd = ops.yfcc_matches(flow, mask, 0, size, size, norm, norm)
                rec, m = ops.essential_ransac(pts1, pts2, Nd, THR)
                ops.recover_pose(pts1, pts2, m, rec)
                return rec, pts1, pts2, Nd

            for _ in range(3):
                once()
            torch.cuda.synchronize()
            times = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                rec, P1, P2, Nd = once()
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
            r = ops.read_pose_record(rec)
            assert r["status"] == ops.POSE_OK
            # models scored = candidates of the iterations inside the scored 64-iteration blocks
            blocks = (min(r["niters"], 1000) + 63) // 64
            idx = ops.essential_samples(Nd)
            E, n = ops.essential_five_point(P1, P2, idx)
            ncand = n.cpu().numpy()
            models = int(ncand[:blocks * 64].sum())
            ms = float(np.median(times))
            row = dict(N=N, outlier=outlier, median_ms=ms, min_ms=float(np.min(times)), niters=r["niters"], models_scored=models,
                       sampson_per_s=models * N / (ms * 1e-3), ransac_count=r["ransac_count"], pose_count=r["pose_count"])
            assert int(Nd) == N
            p1, p2 = P1[:N].cpu().numpy(), P2[:N].cpu().numpy()
            if cv2 is not None:
                t0 = time.perf_counter()
                Ec, mc = cv2.findEssentialMat(p1, p2, method=cv2.RANSAC, threshold=THR)
                t1 = time.perf_counter()
                cv2.recoverPose(Ec[:3], p1, p2, mask=mc)
                t2 = time.perf_counter()
                row.update(cv2_findEssentialMat_s=t1 - t0, cv2_recoverPose_s=t2 - t1, cv2_count=int(mc.sum()))
            rows.append(row)
            print(json.dumps(row), flush=True)
    res = dict(gpu=q, rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(q)


def cuda_median(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def profile_8point(args, ops, q, cv2):
    lib, ptr = rf._lib.lib, rf._lib.ptr
    rows = []
    size = (W_IMG, H_IMG)
    for N in (10000, 100000, 300000):
        flow, mask, norm = flow_inputs(N, 0.3, seed=N + 3)
        pts1, pts2, Nd = ops.yfcc_matches(flow, mask, 0, size, size, norm, norm)
        cap = int(pts1.shape[0])
        rec = ops.pose_record(pts1.device)
        m = torch.zeros(cap, device=pts1.device, dtype=torch.uint8)
        wsz = lib.rf_fundamental_8point_workspace(cap)
        ws = torch.empty(wsz, device=pts1.device, dtype=torch.uint8)
        out = torch.empty(51, device=pts1.device, dtype=torch.float64)
        st = rf._lib.stream()

        def fundamental():
            rf._lib.check(lib.rf_fundamental_8point(ptr(pts1), ptr(pts2), cap, ptr(Nd), ptr(rec), ptr(m), ptr(ws), wsz, st))

        def moments():
            rf._lib.check(lib.rf_fundamental_moments(ptr(pts1), ptr(pts2), cap, ptr(Nd), ptr(out), ptr(ws), wsz, st))

        def whole():
            p1, p2, n = ops.yfcc_matches(flow, mask, 0, size, size, norm, norm)
            r, mk = ops.fundamental_8point(p1, p2, n)
            ops.recover_pose(p1, p2, mk, r)
            return r

        t_f, t_m, t_all = cuda_median(fundamental, args.reps), cuda_median(moments, args.reps), cuda_median(whole, args.reps)
        r = ops.read_pose_record(whole())
        assert int(Nd) == N and r["status"] == ops.POSE_OK
        row = dict(N=N, outlier=0.3, fundamental_8point_ms=t_f, moment_passes_ms=t_m, tail_ms_estimate=t_f - t_m,
                   yfcc_pose_8point_path_ms=t_all, pose_count=r["pose_count"])
        if cv2 is not None:
            p1, p2 = pts1[:N].cpu().numpy(), pts2[:N].cpu().numpy()
            t0 = time.perf_counter()
            F, mc = cv2.findFundamentalMat(p1, p2, method=cv2.FM_8POINT)
            t1 = time.perf_counter()
            cv2.recoverPose(F[:3], p1, p2, mask=mc)
            t2 = time.perf_counter()
            row.update(cv2_findFundamentalMat_s=t1 - t0, cv2_recoverPose_s=t2 - t1)
        rows.append(row)
        print(json.dumps(row), flush=True)
    res = dict(gpu=q, method="8point", rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(q)


if __name__ == "__main__":
    main()
