"""Time evalKITTI's pair (BASELINE config 5: 376 x 1241, coarseSize 800, nbScale 3, scaleR 1.2, fineSize 650, maxH = 5) with and
without host control inside the pair.

    python tools/kitti_profile.py [--pairs 8] [--runs 5] [--warmup 2] [--out FILE]

  * ``align_pair_kitti`` on PIL images (host LANCZOS of both fine-level targets, one host read per hypothesis, the mask update
    in numpy): host-clock median per pair, each call synchronised;
  * ``align_pair_kitti_graph`` (the same pair queued with no host read, one D2H at the end), eager: the same clock;
  * ``GraphedKittiAligner`` (that pair as one CUDA graph): the same clock, plus the kernels per graph and the graph's memory
    (the growth of the allocator's reserved bytes over the capture);
  * ``ConcurrentAligner`` with 2 and 4 lanes of ``GraphedKittiAligner``: pairs/s over --pairs pairs (host clock around
    ``ConcurrentAligner.run``, synchronised), median of --runs windows;
  * ``ops.kitti_region_step`` alone at 376 x 1241: CUDA events around a graph of 200 calls, median of 5 replays.

Seeded synthetic weights and pairs (synthdata.make_pair); the engine is f16x3, as bench.py's default.  The GPU's name, power limit
and maximum SM clock are read (read only) in the same run and printed with the numbers.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def host_ms(fn, runs, warmup):
    """Median host-clock milliseconds of ``fn()`` followed by a device synchronise."""
    out = []
    for it in range(warmup + runs):
        torch.manual_seed(1000 + it)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if it >= warmup:
            out.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=8)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kitti_profile needs a CUDA device")
    import PIL.Image as Image
    import ransac_flow_b200 as rf
    import synthdata as S
    from segnet_profile import gpu_info
    name, power, clock = gpu_info()
    rf.model.set_engine("f16x3")
    rf.outil.corr_precision = 2
    P = rf.pipeline
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "size": "376x1241", "maxH": 5, "fineSize": 650}
    rsd = S.resnet50_conv4_state(0)

    def make_models():
        net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7), "netFlowCoarse": rf.model.NetFlowCoarse(7),
               "netMatch": rf.model.NetMatchability(7)}
        net["netFeatCoarse"].load_state_dict(S.feature_extractor_state(0))
        net["netFlowCoarse"].load_state_dict(S.net_flow_coarse_state(1))
        net["netMatch"].load_state_dict(S.net_matchability_state(2))
        for mod in net.values():
            mod.cuda()
            mod.eval()
        c = rf.CoarseAlignA(3, 1000, 0.05, "Homography", 800, 2, False, 1.2, True, False, resnet_state_dict=rsd, verbose=False)
        return c, net

    raw = [S.make_pair(i, 376, 1241)[:2] for i in range(4)]
    pil = [(Image.fromarray(s), Image.fromarray(t)) for s, t in raw]
    dev = [(torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda()) for s, t in raw]
    c, net = make_models()
    hyp = {}

    # ---- one pair at a time
    k = [0]

    def eager():
        Is, It = pil[k[0] % len(pil)]
        k[0] += 1
        hyp.setdefault("eager", []).append(len(P.align_pair_kitti(c, net, Is, It, maxH=5)["H"]))
    ms_eager = host_ms(eager, args.runs * len(pil), args.warmup)

    def queued():
        s, t = dev[k[0] % len(dev)]
        k[0] += 1
        hyp.setdefault("graph_eager", []).append(len(P.align_pair_kitti_graph(c, net, s, t, maxH=5)["H"]))
    ms_queued = host_ms(queued, args.runs * len(dev), args.warmup)

    ga = P.GraphedKittiAligner(c, net, maxH=5)
    torch.cuda.synchronize()
    r0 = torch.cuda.memory_reserved()
    rec = ga.prepare(*dev[0])
    torch.cuda.synchronize()
    graph_mb = (torch.cuda.memory_reserved() - r0) / 2 ** 20

    def graphed():
        s, t = dev[k[0] % len(dev)]
        k[0] += 1
        ga(s, t, copy=False)
    ms_graph = host_ms(graphed, args.runs * len(dev), args.warmup)
    res["one_pair"] = {"align_pair_kitti_ms": round(ms_eager, 2), "align_pair_kitti_graph_ms": round(ms_queued, 2),
                       "GraphedKittiAligner_ms": round(ms_graph, 2),
                       "pairs_per_s": {"align_pair_kitti": round(1e3 / ms_eager, 2), "align_pair_kitti_graph": round(1e3 / ms_queued, 2),
                                       "GraphedKittiAligner": round(1e3 / ms_graph, 2)},
                       "hypotheses_per_pair": {key: float(np.mean(v)) for key, v in hyp.items()}}
    res["graph"] = {"kernels": rec["n_kernels"], "reserved_mb_over_capture": round(graph_mb, 1)}
    del ga
    torch.cuda.synchronize()

    # ---- lanes
    lanes = {}
    work = [dev[i % len(dev)] for i in range(args.pairs)]
    for L in (2, 4):
        ca = P.ConcurrentAligner(make_models, lanes=L, seed=1000, make_aligner=lambda cc, nn: P.GraphedKittiAligner(cc, nn, maxH=5))
        ca.prepare(*dev[0])
        ms = host_ms(lambda: ca.run(work, copy=False), args.runs, 1)
        lanes["%d_lanes" % L] = {"pairs_per_s": round(1e3 * args.pairs / ms, 2), "ms_per_pair": round(ms / args.pairs, 2)}
        del ca
        torch.cuda.synchronize()
    res["ConcurrentAligner"] = lanes

    # ---- the fused acceptance / mask step alone
    H, W = 376, 1241
    rs = np.random.RandomState(0)
    match = torch.from_numpy(rs.rand(H, W).astype(np.float32)).cuda()
    Mask = torch.zeros((H, W), device="cuda")
    bg = torch.ones((H, W), device="cuda")
    fg = torch.zeros((H, W), device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    al = torch.ones(1, dtype=torch.int32, device="cuda")
    cmin = P.kitti_region_cmin(H * W, 0.005)
    for _ in range(10):
        rf.ops.kitti_region_step(match, Mask, bg, fg, st, al, True, cmin)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()                      # 200 steps in one graph: the device time, not the host's launch rate
    with torch.cuda.graph(g):
        for _ in range(200):
            rf.ops.kitti_region_step(match, Mask, bg, fg, st, al, True, cmin)
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 200)
    res["kitti_region_step_ms"] = round(float(np.median(times)), 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
