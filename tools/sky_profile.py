"""Time the drivers' sky mask on the GPU: the background-map resize, the graphed multi-hypothesis pair with and without segNet,
and evalYFCC's pair with a host versus a device background.

    python tools/sky_profile.py [--runs 20] [--warmup 3] [--pairs 16] [--yfcc-runs 5]

  * ``ops.imresize_mask`` (byte-scaling + PIL BILINEAR + ``< 128``) of a 480 x 640 map to 480 x 640 and of a 376 x 1241 map to
    376 x 1241, for each rotation: CUDA-event medians over --runs calls;
  * ``GraphedMultiAligner`` (maxCoarse = 10, evalCorr semantics) through a 2-lane ``ConcurrentAligner`` on 480 x 640 pairs, without
    and with ``segNet``: pairs/s over --pairs pairs (CUDA events around ``ConcurrentAligner.run``), median of --runs windows;
  * ``align_pair_yfcc`` (nbScale 7, coarseIter 10000, maxCoarse 10) on a 480 x 640 pair: segNet's map copied to the host and
    resized there (``getSky`` + the host ``It_bg``) versus kept on the device (``SegNet.run`` + the CUDA ``It_bg``); host-clock
    medians of --yfcc-runs synchronised calls.

Seeded synthetic weights and images (synthdata); the engine is f16x3, as bench.py's default.  The GPU's name and power limit
are read (read only) in the same run and printed with the numbers.
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


def cuda_ms(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return round(float(np.median(out)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--yfcc-runs", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sky_profile needs a CUDA device")
    import ransac_flow_b200 as rf
    import synthdata as S
    from segnet_profile import gpu_info
    name, power, clock = gpu_info()
    rf.model.set_engine("f16x3")
    rf.outil.corr_precision = 2
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock}

    # ---- the mask resize alone
    rs = np.random.RandomState(0)
    resize = {}
    for H, W in ((480, 640), (376, 1241)):
        m = torch.from_numpy((rs.rand(H, W) < 0.3).astype(np.float32)).cuda()
        for k in range(4):
            h, w = (H, W) if k % 2 == 0 else (W, H)
            resize["%dx%d rot %d" % (H, W, k)] = cuda_ms(lambda: rf.ops.imresize_mask(m, h, w, rot=k), args.runs * 5, args.warmup)
    res["imresize_mask_ms"] = resize

    # ---- the graphed multi-hypothesis pair through two lanes
    sds = (S.segnet_encoder_state(0), S.segnet_decoder_state(0))
    rsd = S.resnet50_conv4_state(0)

    def networks():
        net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7), "netFlowCoarse": rf.model.NetFlowCoarse(7),
               "netMatch": rf.model.NetMatchability(7)}
        net["netFeatCoarse"].load_state_dict(S.feature_extractor_state(0))
        net["netFlowCoarse"].load_state_dict(S.net_flow_coarse_state(1))
        net["netMatch"].load_state_dict(S.net_matchability_state(2))
        for mod in net.values():
            mod.cuda()
            mod.eval()
        return net

    def make_models(seg):
        c = rf.CoarseAlignA(7, 1000, 0.05, "Homography", 480, 2, False, 2, True, seg, resnet_state_dict=rsd, verbose=False,
                            segnet_state_dicts=sds if seg else None)
        return c, networks()

    pairs = [tuple(torch.from_numpy(a).cuda() for a in S.make_pair(i, 480, 640)[:2]) for i in range(4)]
    rate = {}
    for seg in (False, True):
        ca = rf.pipeline.ConcurrentAligner(lambda: make_models(seg), lanes=2, seed=1000,
                                           make_aligner=lambda c, n: rf.pipeline.GraphedMultiAligner(c, n, maxCoarse=10, segNet=seg))
        ca.prepare(*pairs[0])
        work = [pairs[i % len(pairs)] for i in range(args.pairs)]
        ms = cuda_ms(lambda: ca.run(work, copy=False), max(3, args.runs // 4), 1)
        rate["segNet" if seg else "plain"] = {"pairs_per_s": round(1e3 * args.pairs / ms, 2), "ms_per_pair": round(ms / args.pairs, 3),
                                              "graph_kernels": ca.lanes[0].graphs[next(iter(ca.lanes[0].graphs))]["n_kernels"]}
        del ca
        torch.cuda.synchronize()
    res["graphed_multi_2_lanes_480x640"] = rate

    # ---- evalYFCC's pair: host versus device background
    import PIL.Image as Image
    from ransac_flow_b200.segnet import SegNet
    src, tgt, _ = S.make_rotated_pair(70, 480, 640, 1)
    s_u8, t_u8 = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
    t_pil = Image.fromarray(tgt)
    net = networks()
    seg = SegNet(None, None, 2, False, state_dicts=sds)
    c = rf.CoarseAlignB(7, 10000, 0.05, "Homography", 480, 1, True, True, True, False, 2, resnet_state_dict=rsd, verbose=False)
    yfcc = {}
    for where in ("host", "device"):
        times = []
        for it in range(args.warmup + args.yfcc_runs):
            torch.manual_seed(1000)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            bg = seg.getSky(t_pil) if where == "host" else seg.run(t_u8)[0]
            out = rf.pipeline.align_pair_yfcc(c, net, s_u8, t_u8, maxCoarse=10, It_bg=bg)
            torch.cuda.synchronize()
            if it >= args.warmup:
                times.append(1e3 * (time.perf_counter() - t0))
        yfcc[where] = {"ms": round(float(np.median(times)), 2), "hypotheses": len(out["H"]), "angle": out["angle"]}
    res["align_pair_yfcc_480x640_ms"] = yfcc
    print(json.dumps(res))


if __name__ == "__main__":
    main()
