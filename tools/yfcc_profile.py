"""Throughput of evalYFCC's pair loop: ``pipeline.align_pair_yfcc`` (device-resident rotation search + hypothesis loop) and
the host-steered drop-in path (``pipeline.align_pair_yfcc_host``: the ``CoarseAlignB`` mirror plus the driver's statements)
on the same synthetic pairs, at the driver's defaults (nbScale 7, scaleR 2, minSize 480, coarseIter 10000, tolerance 0.05,
maxCoarse 10, maskRegionTh 0.01, no segNet).

    python tools/yfcc_profile.py [--pairs 4] [--runs 3] [--warmup 1] [--engine f16x3] [--maskRegionTh 0.01]

``--maskRegionTh 1.0`` rejects every hypothesis after the first (the pair ends early: the eager paths compute two, the
loop graphs all eleven).

Pairs: ``synthdata.make_rotated_pair(i, 480, 640, i % 4)`` (targets rotated by 0 / 90 / 180 / 270 degrees), seeded
synthetic weights.  The device path gets uint8 CUDA images, the drop-in path PIL images (what the driver opens).  Per pass
over the pairs: pairs/s of each path, and the device path split into its stages - the 11-image trunk (pyramid, rotations,
resizing, ResNet-50 conv4), the rotation search (4 correlations + RANSAC) and the hypothesis loop - each timed with a host
clock between device synchronisations (the stages read back to the host anyway).  Medians over ``--runs`` passes after
``--warmup`` passes; one JSON line with the GPU's name and power limit (read only) and the peak device memory the first
11-image batch allocates (torch's allocator statistics).

The graphed arms on the same pairs: ``align_pair_yfcc_graph`` (the graphed path's device work run eagerly, one host read of
the search record per pair), ``GraphedYfccAligner`` (a search graph and one loop graph per orientation class per input size)
and a two-lane ``ConcurrentAligner`` of them; with the kernels per graph, the reserved memory the captures grow
(``torch.cuda.memory_reserved`` around the first ``prepare`` of every input size) and the hypotheses accepted per pair.  The
loop graphs run all ``maxCoarse + 1`` hypotheses whatever the pair accepts.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in q.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def networks(rf, S):
    net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7),
           "netFlowCoarse": rf.model.NetFlowCoarse(7), "netMatch": rf.model.NetMatchability(7)}
    net["netFeatCoarse"].load_state_dict(S.feature_extractor_state(0))
    net["netFlowCoarse"].load_state_dict(S.net_flow_coarse_state(1))
    net["netMatch"].load_state_dict(S.net_matchability_state(2))
    for m in net.values():
        m.cuda()
        m.eval()
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--engine", default="f16x3")
    ap.add_argument("--maskRegionTh", type=float, default=0.01)
    args = ap.parse_args()
    th = args.maskRegionTh
    if not torch.cuda.is_available():
        raise SystemExit("yfcc_profile needs a CUDA device")
    import PIL.Image as Image
    import ransac_flow_b200 as rf
    import synthdata as S
    from ransac_flow_b200 import dropin, pipeline
    dropin.select_engine(args.engine)
    net = networks(rf, S)
    make = lambda: rf.CoarseAlignB(7, 10000, 0.05, "Homography", 480, 1, True, True, True, False, 2,
                                   resnet_state_dict=S.resnet50_conv4_state(0), verbose=False)
    dev_model, host_model = make(), make()
    pairs = [S.make_rotated_pair(i, 480, 640, i % 4)[:2] for i in range(args.pairs)]
    dev_pairs = [tuple(torch.from_numpy(a).cuda() for a in p) for p in pairs]
    pil_pairs = [tuple(Image.fromarray(a) for a in p) for p in pairs]
    sync = torch.cuda.synchronize
    res = {k: [] for k in ("device", "trunk", "search", "hypotheses", "host", "graph_eager", "graphed", "lanes2")}
    angles, nH = None, None
    torch.manual_seed(0)
    with torch.no_grad():
        # peak memory of the 11-image batch on a model that has not run yet: activation slots, trunk output, features
        sync()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        dev_model._set_rotated_pair(*dev_pairs[0])
        sync()
        trunk_peak = torch.cuda.max_memory_allocated() - base
        for it in range(args.warmup + args.runs):
            sync()
            t0 = time.perf_counter()
            outs = [pipeline.align_pair_yfcc(dev_model, net, s, t, maskRegionTh=th) for s, t in dev_pairs]
            sync()
            t1 = time.perf_counter()
            st = np.zeros(3)
            for s, t in dev_pairs:                   # the same work, stage by stage
                a = time.perf_counter()
                dev_model._set_rotated_pair(s, t)
                sync()
                b = time.perf_counter()
                _, _, bg, _ = pipeline._rotation_search(dev_model, None, None)
                sync()
                c = time.perf_counter()
                pipeline._hypotheses_device(dev_model, net, 10, th, True, bg, None, rewind_too_few=True)
                sync()
                st += (b - a, c - b, time.perf_counter() - c)
            sync()
            t2 = time.perf_counter()
            for s, t in pil_pairs:
                pipeline.align_pair_yfcc_host(host_model, net, s, t, maskRegionTh=th)
            sync()
            t3 = time.perf_counter()
            if it >= args.warmup:
                n = len(pairs)
                res["device"].append(n / (t1 - t0))
                res["host"].append(n / (t3 - t2))
                for k, v in zip(("trunk", "search", "hypotheses"), st):
                    res[k].append(1e3 * v / n)
            angles, nH = [o["angle"] for o in outs], [len(o["H"]) for o in outs]
        # the graphed arms
        sync()
        r0 = torch.cuda.memory_reserved()
        ga = pipeline.GraphedYfccAligner(make(), net, maskRegionTh=th)
        for s, t in dev_pairs:
            ga.prepare(s, t)
        sync()
        graph_reserved = torch.cuda.memory_reserved() - r0
        kernels = {"x".join(map(str, k[1][:2])): {"search": r["n_kernels"], "loops": {str(c): L["n_kernels"] for c, L in r["loops"].items()}}
                   for k, r in ga.graphs.items()}
        ca = pipeline.ConcurrentAligner(lambda: (make(), networks(rf, S)), lanes=2, make_aligner=lambda c, n: pipeline.GraphedYfccAligner(c, n, maskRegionTh=th))
        for s, t in dev_pairs:
            ca.prepare(s, t)
        graph_model = make()
        for it in range(args.warmup + args.runs):
            sync()
            t0 = time.perf_counter()
            gouts = [pipeline.align_pair_yfcc_graph(graph_model, net, s, t, maskRegionTh=th) for s, t in dev_pairs]
            sync()
            t1 = time.perf_counter()
            routs = [ga(s, t) for s, t in dev_pairs]
            sync()
            t2 = time.perf_counter()
            louts = ca.run(dev_pairs)
            sync()
            t3 = time.perf_counter()
            if it >= args.warmup:
                n = len(pairs)
                res["graph_eager"].append(n / (t1 - t0))
                res["graphed"].append(n / (t2 - t1))
                res["lanes2"].append(n / (t3 - t2))
        g_angles, g_nH = [o["angle"] for o in routs], [len(o["H"]) for o in routs]
        l_nH = [len(o["H"]) for o in louts]
    name, power, clock = gpu_info()
    med = lambda v: round(float(np.median(v)), 3)
    print(json.dumps({"pairs_per_s": {"align_pair_yfcc": med(res["device"]), "drop_in_host_path": med(res["host"]),
                                      "align_pair_yfcc_graph": med(res["graph_eager"]), "GraphedYfccAligner": med(res["graphed"]),
                                      "ConcurrentAligner_2_lanes": med(res["lanes2"])},
                      "graph_kernels": kernels, "graph_reserved_mib": round(graph_reserved / 2 ** 20, 1),
                      "graph_angles": g_angles, "graph_hypotheses": g_nH, "lanes_hypotheses": l_nH,
                      "graph_loop_hypotheses_per_pair": 11,
                      "stage_ms_per_pair": {"trunk_11_images": med(res["trunk"]), "rotation_search": med(res["search"]),
                                            "hypothesis_loop": med(res["hypotheses"])},
                      "angles": angles, "hypotheses": nH, "engine": args.engine, "image": [480, 640], "pairs": len(pairs),
                      "runs": args.runs, "maskRegionTh": th, "trunk_11_images_peak_mib": round(trunk_peak / 2 ** 20, 1),
                      "gpu": name, "power_limit": power, "max_sm_clock": clock}))


if __name__ == "__main__":
    main()
