"""Throughput of the training-pair generator (train/generate_coarse_aligned_pair.ipynb at its settings: minSize 480, nbIter
10000, tolerance 0.05) on synthetic 720 x 480 pairs (``synthdata.make_pair(i, 480, 720)``, the size of the notebook's sample
images) with seeded weights:

    python tools/train_pairs_profile.py [--pairs 8] [--runs 3] [--warmup 1] [--engine f16x3] [--calls 2000]

Pairs/s of ``align_train_pair`` (eager, one pinned read per pair), ``GraphedTrainPairAligner`` (one graph per input size), a
two-lane ``ConcurrentAligner`` of them, and ``results.write_train_pairs`` through the two lanes including host JPEG coding
(into a temporary directory).  Medians over ``--runs`` passes after ``--warmup``; every pass ends in a device synchronise.

Also: the fused ``rf_warp_sample_u8`` against the composition it replaces (warp_grid -> preproc_u8 -> grid_sample -> x 255
truncated), each timed with CUDA events over ``--calls`` back-to-back calls at the pair's size (480 x 720 from a 480 x 720
target); the library kernels per graph; the reserved memory the captures grow (``torch.cuda.memory_reserved`` around the first
``prepare``); the kept pairs; and the GPU's name and power limit (read only).  One JSON line.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.yfcc_profile import gpu_info  # noqa: E402


def event_ms(fn, calls):
    """Mean ms per call of ``fn()`` over ``calls`` back-to-back calls, between two CUDA events."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--engine", default="f16x3")
    ap.add_argument("--calls", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_pairs_profile needs a CUDA device")
    import ransac_flow_b200 as rf
    import synthdata as S
    from ransac_flow_b200 import dropin, pipeline, results
    dropin.select_engine(args.engine)
    rsd = S.resnet50_conv4_state(0)
    make = lambda: rf.train_pairs.TrainPairModel(rsd)
    pairs = [S.make_pair(i, 480, 720)[:2] for i in range(args.pairs)]
    dev_pairs = [tuple(torch.from_numpy(a).cuda() for a in p) for p in pairs]
    sync = torch.cuda.synchronize
    res = {k: [] for k in ("eager", "graphed", "lanes2", "write")}
    torch.manual_seed(0)
    with torch.no_grad():
        model = make()
        sync()
        r0 = torch.cuda.memory_reserved()
        ga = pipeline.GraphedTrainPairAligner(make())
        ga.prepare(*dev_pairs[0])
        sync()
        graph_reserved = torch.cuda.memory_reserved() - r0
        n_kernels = next(iter(ga.graphs.values()))["n_kernels"]
        ca = pipeline.ConcurrentAligner(lambda: (make(), None), lanes=2, make_aligner=pipeline.GraphedTrainPairAligner)
        ca.prepare(*dev_pairs[0])
        kept = None
        for it in range(args.warmup + args.runs):
            sync()
            t0 = time.perf_counter()
            outs = [rf.pipeline.align_train_pair(model, s, t) for s, t in dev_pairs]
            sync()
            t1 = time.perf_counter()
            for s, t in dev_pairs:
                ga(s, t)
            sync()
            t2 = time.perf_counter()
            ca.run(dev_pairs)
            sync()
            t3 = time.perf_counter()
            with tempfile.TemporaryDirectory() as d:
                index = results.write_train_pairs(ca, pairs, os.path.join(d, "pairs"))
            sync()
            t4 = time.perf_counter()
            if it >= args.warmup:
                n = len(pairs)
                for k, dt in zip(("eager", "graphed", "lanes2", "write"), (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
                    res[k].append(n / dt)
            kept = [o["kept"] for o in outs]
        # the fused kernel against its composition, at the pair's size
        H = torch.from_numpy(np.array([[1.05, 0.02, 0.03], [-0.01, 0.98, -0.02], [0.02, 0.01, 1.0]], np.float32)).reshape(-1).cuda()
        src = dev_pairs[0][1].contiguous()
        h, w = int(src.shape[0]), int(src.shape[1])

        def unfused():
            grid = rf.ops.warp_grid(H.view(1, 3, 3), h, w)
            t = rf.ops.preproc_u8(src.reshape(-1, 3), normalize=False).view(1, h, w, 3).permute(0, 3, 1, 2)
            return (rf.ops.grid_sample(t, grid) * 255).to(torch.uint8)[0].permute(1, 2, 0).contiguous()
        fused_ms = event_ms(lambda: rf.train_pairs.warp_sample_u8(H, src, h, w), args.calls)
        unfused_ms = event_ms(unfused, args.calls)
        assert torch.equal(rf.train_pairs.warp_sample_u8(H, src, h, w), unfused())
    name, power, clock = gpu_info()
    med = lambda v: round(float(np.median(v)), 3)
    print(json.dumps({"pairs_per_s": {"align_train_pair": med(res["eager"]), "GraphedTrainPairAligner": med(res["graphed"]),
                                      "ConcurrentAligner_2_lanes": med(res["lanes2"]), "write_train_pairs_2_lanes_jpeg": med(res["write"])},
                      "warp_sample_u8_us": {"fused": round(1e3 * fused_ms, 2), "unfused_composition": round(1e3 * unfused_ms, 2)},
                      "graph_kernels": n_kernels, "graph_reserved_mib": round(graph_reserved / 2 ** 20, 1), "kept": kept,
                      "engine": args.engine, "image": [480, 720], "pairs": len(pairs), "runs": args.runs,
                      "gpu": name, "power_limit": power, "max_sm_clock": clock}))


if __name__ == "__main__":
    main()
