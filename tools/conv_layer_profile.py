#!/usr/bin/env python
"""Per-layer profile of the convolution programs of one config-2 pair on the split (`f16x3`) engine.

    python tools/conv_layer_profile.py [--reps N] [--out DIR]

One eager pair (bench.py's weights, synthdata pair 0, 480x640) records every layer program it runs and the input it runs
on: the ResNet-50 trunk on the 8-image ragged batch (7 pyramid scales + the target), the FeatureExtractor, NetFlowCoarse and
NetMatchability.  Each program is then warmed up and run N times under torch.profiler with CUDA activities; every op of a
program is exactly one kernel launch - the direct stems (`stem7`: the trunk's 7x7 / 2 and the FeatureExtractor's 3x3 / 1, the
fp32 image in, the stem output out) included - except a stem fused with the max-pool after it (RF_LAYER_STEM_POOL): one
kernel for the two ops, timed on the stem row, with the max-pool row marked fused and the pair's own floor (the image in, the
pooled output out) printed beside it.  The kernels zip with `program.ops` in launch order.

Per layer: kernel, shape, tiles x N tiles, K blocks (KI), median time, algorithmic GFLOP and the executed TFLOP/s (3 MMAs per
MAC on the split engine), algorithmic HBM bytes and GB/s, and which data-sheet floor bounds the layer and what share of it
the layer reaches.  The byte model counts 4 bytes per split activation element (2 fp16 planes) and every layer reading its
inputs and residual once and writing its output once; the weights are left out.  The floors are the H100 SXM data sheet's
(989 dense fp16 TFLOP/s, 3.35 TB/s), for a 700 W card: they are yardsticks, not rates this card reaches.

The flop / byte model (`layer_model`, `pair_sizes`) runs on the CPU; the timing needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0          # H100 SXM data sheet, dense fp16
PEAK_GBS = 3350.0            # H100 SXM data sheet, HBM3
MMAS_PER_MAC = 3             # split operands: hi*hi + lo*hi + hi*lo
ACT_BYTES = 4                # split activation: two fp16 planes

# program op codes (program.py)
OP_CONV, OP_MAXPOOL, OP_BLUR, OP_IM2COL, OP_POOLBLUR, OP_STEM7, OP_CONV_DUAL = 0, 1, 2, 3, 4, 5, 6
OP_NAMES = {OP_CONV: "conv", OP_MAXPOOL: "maxpool", OP_BLUR: "blur", OP_IM2COL: "im2col", OP_POOLBLUR: "poolblur",
            OP_STEM7: "stem7", OP_CONV_DUAL: "conv_dual"}


def pick_tw(Ho, Wo):
    """Tile width of wg_kernel for an image (pick_tw in csrc/gemm_tc.cu)."""
    best, best_area = 16, -1
    for tw in (16, 32, 8, 64, 128):
        th = 128 // tw
        area = ((Wo + tw - 1) // tw) * ((Ho + th - 1) // th)
        if best_area < 0 or area < best_area:
            best, best_area = tw, area
    return best


def pixel_tiles(ohw, flat):
    """Pixel tiles of wg_kernel on output images ``ohw`` (conv_impl in csrc/gemm_tc.cu): with ``flat`` (1x1 / stride-1 layers)
    tiles of 128 consecutive pixels of the whole batch, otherwise tw x (128 / tw) rectangles inside each image."""
    if flat:
        return (sum(h * w for h, w in ohw) + 127) // 128
    return sum(((w + pick_tw(h, w) - 1) // pick_tw(h, w)) * ((h + 128 // pick_tw(h, w) - 1) // (128 // pick_tw(h, w))) for h, w in ohw)


def _out(hw, k, s, p):
    return [((h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1) for h, w in hw]


def layer_model(ops, hw, dual=None, out_f32=()):
    """Shapes, flops and bytes of every op of a layer program (``program.ops``, ``program.dual``) run on the split engine
    on images ``hw`` [(H, W), ...].  Op indices in ``out_f32`` write fp32 (4 bytes per element as well).  Returns one dict
    per op; convolutions (stem, conv, conv_dual) carry the floor fields, other ops only their shapes."""
    dual = dual or {}
    hws = [list(hw)]
    rows = []
    for i, o in enumerate(ops):
        op, src, res, cin, cout, k, s, p = o[:8]
        if op == OP_POOLBLUR:
            k, s, p = 4, 2, 1
        elif op == OP_BLUR:
            k, p = 3, 1
        ohw = _out(hws[src], k, s, p)
        hws.append(ohw)
        pin = sum(h * w for h, w in hws[src])
        pout = sum(h * w for h, w in ohw)
        r = dict(index=i, op=OP_NAMES[op], cin=cin, cout=cout, k=k, stride=s, out_hw=ohw)
        if op in (OP_CONV, OP_CONV_DUAL, OP_STEM7):
            K = k * k * cin
            nbytes = (pin * cin * ACT_BYTES if op != OP_STEM7 else pin * 3 * 4) + pout * cout * ACT_BYTES
            if res is not None and res >= 0:
                nbytes += pout * cout * ACT_BYTES
            flat = op != OP_STEM7 and (k, s, p) == (1, 1, 0)
            if op == OP_CONV_DUAL:
                src2, cin2, s2 = dual[i]
                K += cin2
                nbytes += sum(h * w for h, w in hws[src2]) * cin2 * ACT_BYTES
                flat = flat and s2 == 1
            flop = 2.0 * pout * cout * K
            bn = 128 if cout > 64 else 64
            tiles = pixel_tiles(ohw, flat)
            t_flop = MMAS_PER_MAC * flop / (PEAK_TFLOPS * 1e12)
            t_byte = nbytes / (PEAK_GBS * 1e9)
            r.update(K=K, KI=(K + 63) // 64, tiles=tiles, ntiles=(cout + bn - 1) // bn, bn=bn, residual=res is not None and res >= 0,
                     gflop=flop / 1e9, bytes=nbytes, floor_ms=1e3 * max(t_flop, t_byte), bound="tensor" if t_flop >= t_byte else "hbm")
        rows.append(r)
    return rows


def pair_sizes(h=480, w=640, min_size=480, nb_scale=7, scale_r=2):
    """(H, W) of the trunk's ragged batch for one pair: the source pyramid (CoarseAlign.setPair) and the target."""
    from ransac_flow_b200.coarseAlignFeatMatch import _CoarseAlignBase, scale_list
    base = _CoarseAlignBase.__new__(_CoarseAlignBase)
    base.strideNet = 16
    sizes = [base._target_size(w, h, int(min_size * s)) for s in scale_list(nb_scale, scale_r)] + [base._target_size(w, h, min_size)]
    return [(hh, ww) for ww, hh in sizes]


def trunk_program(device="cpu"):
    """The split engine's ResNet-50 trunk program (conv3 and the down-sampling branch fused), built with bench.py's weights."""
    import synthdata
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4.__new__(ResNet50Conv4)
    import torch
    net.device = torch.device(device)
    net._sd = {k: v.detach().float() for k, v in synthdata.resnet50_conv4_state(0).items() if torch.is_tensor(v) and v.dtype.is_floating_point}
    return net._build(64, fuse_downsample=True)


def convs(rows):
    return [r for r in rows if "floor_ms" in r]


# ----------------------------------------------------------------------------- GPU part
def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, plim, mx = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": plim, "max_sm_clock": mx}
    except Exception as e:  # noqa: BLE001
        return {"error": "nvidia-smi query failed: %s" % e}


def record_programs():
    """Run pair 0 of the config-2 workload once, eagerly, recording every (program, input) that LayerProgram.run sees."""
    import torch
    import bench
    import ransac_flow_b200 as rf
    from ransac_flow_b200.program import LayerProgram
    rf.model.set_engine("f16x3")
    rf.outil.corr_precision = 2
    rsd, fe_sd, nf_sd, nm_sd = bench.states()
    net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7),
           "netFlowCoarse": rf.model.NetFlowCoarse(7), "netMatch": rf.model.NetMatchability(7)}
    for k, sd in (("netFeatCoarse", fe_sd), ("netFlowCoarse", nf_sd), ("netMatch", nm_sd)):
        net[k].load_state_dict(sd)
    for m in net.values():
        m.cuda()
        m.eval()
    coarse = rf.CoarseAlignA(7, 1000, 0.05, "Homography", 480, 2, False, 2, True, False, resnet_state_dict=rsd, verbose=False)
    coarse.device_preproc = True
    seen, order = {}, []
    run0 = LayerProgram.run

    def run(self, x, engine):
        key = (id(self), tuple(x.hw))
        if key not in seen:
            seen[key] = (self, type(x)(x.data.clone(), list(x.hw)), engine)
            order.append(key)
        return run0(self, x, engine)
    s, t = [torch.from_numpy(a).cuda() for a in bench.make_pairs(1, 2)[0]]
    LayerProgram.run = run
    try:
        torch.manual_seed(1000)
        coarse.setPair(s, t)
        Itw, Ith = coarse.target_size
        featt = rf.pipeline.fine_features(net["netFeatCoarse"], coarse.ItTensor)
        Hd = coarse.getCoarse_device(None)[0]
        fc = rf.ops.warp_grid(Hd.view(1, 3, 3), Ith, Itw)
        rf.pipeline.PredFlowMask_device(coarse.IsTensor, featt, fc, (Ith, Itw), net)
        torch.cuda.synchronize()
    finally:
        LayerProgram.run = run0
    names = {id(coarse.net._program_split): "trunk", id(net["netFeatCoarse"]._folded(4)): "feature_extractor",
             id(net["netFlowCoarse"]._folded(4)): "net_flow_coarse", id(net["netMatch"]._folded(4)): "net_matchability"}
    return [(names.get(k[0], "program%d" % i),) + seen[k] for i, k in enumerate(order)], (coarse, net)


def fused_pools(prog, x, engine):
    """Indices of the max-pool ops that run inside the stem kernel before them (the compiled program's RF_LAYER_STEM_POOL)."""
    from ransac_flow_b200.program import RF_LAYER_STEM_POOL
    key = (tuple(x.hw), str(x.data.device), int(engine) if int(engine) in (2, 4) else 0)
    layers = prog._compiled[key]["layers"]
    return {i + 1 for i in range(len(prog.ops)) if layers[i].flags & RF_LAYER_STEM_POOL}


def kernel_times(prog, x, engine, reps):
    """Median device time (us) and name of each op's kernel over ``reps`` runs of the program (None for a fused max-pool)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        prog.run(x, engine)
    torch.cuda.synchronize()
    fused = fused_pools(prog, x, engine)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            prog.run(x, engine)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    ev.sort(key=lambda e: e.time_range.start)
    ops = [i for i in range(len(prog.ops)) if i not in fused]       # the op each kernel of a run belongs to
    n = len(ops)
    if len(ev) != n * reps:
        raise SystemExit("conv_layer_profile: %d kernels for %d runs of a %d-kernel program: %s" % (len(ev), reps, n, sorted({e.name for e in ev})))
    med, names = [None] * len(prog.ops), ["(fused into op %d)" % (i - 1) for i in range(len(prog.ops))]
    for k, i in enumerate(ops):
        med[i] = statistics.median([ev[r * n + k].time_range.elapsed_us() for r in range(reps)])
        names[i] = ev[k].name
    return med, names


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for conv_layer_profile.json")
    args = ap.parse_args()
    import torch
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("conv_layer_profile: needs a CUDA device")
    info = gpu_info()
    progs, _keep = record_programs()
    sampler = bench.ClockSampler(0)
    sampler.start()
    report = {"gpu": info, "reps": args.reps, "peaks": {"tflops_f16": PEAK_TFLOPS, "hbm_gbs": PEAK_GBS, "source": "H100 SXM data sheet (700 W)"},
              "programs": []}
    for name, prog, x, engine in progs:
        med, knames = kernel_times(prog, x, engine, args.reps)
        rows = layer_model(prog.ops, x.hw, getattr(prog, "dual", {}))
        for r, us, kn in zip(rows, med, knames):
            r["kernel"], r["us"] = kn, us
            if us is None:                                         # a max-pool fused into the stem before it
                r["fused"] = True
                st = rows[r["index"] - 1]
                nbytes = st["bytes"] - st["cout"] * sum(h * w for h, w in st["out_hw"]) * ACT_BYTES + r["cout"] * sum(h * w for h, w in r["out_hw"]) * ACT_BYTES
                t_flop = MMAS_PER_MAC * st["gflop"] * 1e9 / (PEAK_TFLOPS * 1e12)
                st["pair_bytes"] = nbytes
                st["pair_floor_ms"] = 1e3 * max(t_flop, nbytes / (PEAK_GBS * 1e9))
                st["pair_floor_share"] = st["pair_floor_ms"] * 1e3 / st["us"]
                continue
            if "floor_ms" in r:
                r["tflops_executed"] = MMAS_PER_MAC * r["gflop"] * 1e9 / (us * 1e-6) / 1e12
                r["gbs"] = r["bytes"] / (us * 1e-6) / 1e9
                r["floor_share"] = r["floor_ms"] * 1e3 / us
        report["programs"].append({"name": name, "images": [list(v) for v in x.hw], "layers": rows,
                                   "total_us": sum(t for t in med if t is not None), "conv_us": sum(r["us"] for r in convs(rows)),
                                   "conv_floor_us": sum(1e3 * r["floor_ms"] for r in convs(rows))})
    report["clocks"] = sampler.stop()
    print("%s, power limit %s, max SM clock %s; SM clock during the runs: median %s MHz (%s)" % (
        info.get("name"), info.get("power_limit"), info.get("max_sm_clock"), report["clocks"].get("sm_mhz"), ", ".join(report["clocks"].get("reasons") or []) or "no throttle reason"))
    for P in report["programs"]:
        print("\n== %s on %s: %.1f us in all, convolutions %.1f us against a floor of %.1f us" % (
            P["name"], " ".join("%dx%d" % tuple(v) for v in P["images"]), P["total_us"], P["conv_us"], P["conv_floor_us"]))
        print("%3s %-9s %5s %5s %2s %1s %3s %3s %11s %3s %9s %8s %8s %8s %7s %6s %6s" % (
            "#", "op", "cin", "cout", "k", "s", "res", "BN", "tiles x nt", "KI", "us", "GFLOP", "TFLOP/s", "MB", "GB/s", "bound", "floor"))
        for r in P["layers"]:
            if "floor_ms" in r:
                print("%3d %-9s %5d %5d %2d %1d %3s %3d %6d x %2d %3d %9.1f %8.2f %8.1f %8.2f %7.0f %6s %5.0f%%" % (
                    r["index"], r["op"], r["cin"], r["cout"], r["k"], r["stride"], "yes" if r["residual"] else "", r["bn"], r["tiles"], r["ntiles"],
                    r["KI"], r["us"], r["gflop"], r["tflops_executed"], r["bytes"] / 1e6, r["gbs"], r["bound"], 100 * r["floor_share"]))
            elif r.get("fused"):
                st = P["layers"][r["index"] - 1]
                print("%3d %-9s %5d %5d %2d %1d %3s %3s %11s %3s %9s   fused into #%d: the pair's floor %.1f us (%.2f MB), reached %.0f%%" % (
                    r["index"], r["op"], r["cin"], r["cout"], r["k"], r["stride"], "", "", "", "", "-", st["index"], 1e3 * st["pair_floor_ms"],
                    st["pair_bytes"] / 1e6, 100 * st["pair_floor_share"]))
            else:
                print("%3d %-9s %5d %5d %2d %1d %3s %3s %11s %3s %9.1f   (%s)" % (r["index"], r["op"], r["cin"], r["cout"], r["k"], r["stride"], "", "", "", "",
                                                                               r["us"], r["kernel"][:40]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "conv_layer_profile.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
