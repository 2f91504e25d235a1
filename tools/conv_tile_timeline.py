#!/usr/bin/env python
"""Where a tile's time goes in the wgmma convolutions of the config-2 ResNet-50 trunk (split `f16x3` engine).

    python tools/conv_tile_timeline.py --out DIR [--reps N]

Builds the library once more with -DRF_TILE_TIMELINE into DIR (the normal build is left alone): in that variant thread 0 of
each consumer warpgroup and the producer lane of `wg_kernel` write %globaltimer stamps per tile into a buffer the caller
gives (csrc/gemm_tc.cu, TL_STAMP).  The trunk program of one config-2 pair (bench.py's weights, synthdata pair 0, the
8-image ragged batch) is recorded on the normal library, as tools/conv_layer_profile.py does, then run N times through the
timeline library.  Per convolution it prints the median over all tiles and runs, in microseconds, of (consumer warpgroup 0):

    wait K0   tile start -> the tile's first full barrier passed (the first K block's load, not hidden by the tile before)
    K loop    first full barrier -> last MMA retired (MMAs and the waits for the later K blocks)
    resid     last MMA retired -> the epilogue slot's barrier passed (its residual loaded)
    epi       residual barrier -> store committed (bias, residual, ReLU, split, shared-memory writes, TMA store issue)
    tile      tile start -> the same CTA's next tile start (the CTA's last tile: -> store committed)

and `lead`: how long before the last MMA retired the producer had issued the residual (negative: after).  The stamps cost
a few global stores per tile, so the timeline's layer times run somewhat above tools/conv_layer_profile.py's.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

TL_WORDS, TL_LAUNCH_WORDS = 16, 6                  # csrc/gemm_tc.cu


def build_timeline_lib(out_dir):
    """The library built with -DRF_TILE_TIMELINE into out_dir (build.py's sources and flags)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_rf_build", os.path.join(ROOT, "ransac-flow_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = os.path.join(out_dir, "timeline_build")
    os.makedirs(objdir, exist_ok=True)
    lib = os.path.join(objdir, "libransacflow_b200_timeline.so")
    procs = []
    for s in b.SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        procs.append((s, o, subprocess.Popen([nvcc] + b.NVCC_FLAGS + ["-DRF_TILE_TIMELINE", "-c", os.path.join(b.CSRC, s), "-o", o],
                                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for s, o, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise SystemExit("conv_tile_timeline: nvcc failed on %s:\n%s" % (s, out))
    subprocess.check_call([nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-o", lib] + [o for _, o, _ in procs] + ["-lcudart"])
    return lib


def load_timeline_lib(path):
    from ransac_flow_b200 import _lib
    lib = C.CDLL(path)
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.rf_tile_timeline_begin.restype, lib.rf_tile_timeline_begin.argtypes = C.c_int, [C.c_void_p, C.c_longlong]
    lib.rf_tile_timeline_launches.restype = C.c_longlong
    lib.rf_tile_timeline_launches.argtypes = [C.POINTER(C.c_longlong), C.c_longlong]
    return lib


def tile_phases(stamps, ntiles, grid):
    """Per tile (consumer warpgroup 0's stamps, the producer's for the lead): the phase durations in microseconds."""
    rows = []
    for t in range(ntiles):
        s = stamps[t]
        c = s[0:5]
        nxt = t + grid
        end = stamps[nxt][0] if nxt < ntiles else c[4]
        rows.append({"wait_k0": (c[1] - c[0]) / 1e3, "k_loop": (c[2] - c[1]) / 1e3, "resid": (c[3] - c[2]) / 1e3,
                     "epi": (c[4] - c[3]) / 1e3, "tile": (end - c[0]) / 1e3, "lead": (c[2] - s[14]) / 1e3})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", required=True, help="directory for the timeline build and conv_tile_timeline.json")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("conv_tile_timeline: needs a CUDA device")
    import conv_layer_profile as CLP
    import ransac_flow_b200 as rf
    os.makedirs(args.out, exist_ok=True)
    tl = load_timeline_lib(build_timeline_lib(args.out))
    info = CLP.gpu_info()
    progs, _keep = CLP.record_programs()
    name, prog, x, engine = [p for p in progs if p[0] == "trunk"][0]
    rows = CLP.layer_model(prog.ops, x.hw, getattr(prog, "dual", {}))
    conv_rows = [r for r in rows if r["op"] in ("conv", "conv_dual")]
    words = 2 * sum(r["tiles"] * r["ntiles"] for r in conv_rows) * TL_WORDS
    buf = torch.zeros(words, dtype=torch.int64, device="cuda")
    normal = rf.program.lib
    rf.program.lib = tl
    per_layer = [[] for _ in conv_rows]
    try:
        for _ in range(3):
            prog.run(x, engine)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            buf.zero_()
            tl.rf_tile_timeline_begin(C.c_void_p(buf.data_ptr()), words)
            prog.run(x, engine)
            torch.cuda.synchronize()
            n = tl.rf_tile_timeline_launches(None, 0)
            table = (C.c_longlong * n)()
            tl.rf_tile_timeline_launches(table, n)
            launches = np.array(table[:], dtype=np.int64).reshape(-1, TL_LAUNCH_WORDS)
            if len(launches) != len(conv_rows):
                raise SystemExit("conv_tile_timeline: %d wg_kernel launches for %d convolutions" % (len(launches), len(conv_rows)))
            stamps = buf.cpu().numpy()
            for k, (off, ntiles, grid, KI, cout, res) in enumerate(launches.tolist()):
                if off < 0:
                    raise SystemExit("conv_tile_timeline: timeline buffer too small")
                st = stamps[off:off + ntiles * TL_WORDS].reshape(ntiles, TL_WORDS)
                per_layer[k].append(dict(stamps=st, ntiles=ntiles, grid=grid, KI=KI, cout=cout, res=res))
    finally:
        rf.program.lib = normal
        tl.rf_tile_timeline_begin(None, 0)
    report = {"gpu": info, "reps": args.reps, "layers": []}
    print("%s, power limit %s, max SM clock %s; trunk on %s, median over tiles and %d runs (us per tile)" % (
        info.get("name"), info.get("power_limit"), info.get("max_sm_clock"), " ".join("%dx%d" % tuple(v) for v in x.hw), args.reps))
    print("%3s %-9s %5s %5s %2s %3s %3s %5s %4s %7s %7s %7s %7s %7s %7s %8s" % (
        "#", "op", "cin", "cout", "k", "res", "KI", "tiles", "CTAs", "wait K0", "K loop", "resid", "epi", "tile", "lead", "layer us"))
    for r, runs in zip(conv_rows, per_layer):
        ph = []
        layer_us = []
        for run in runs:
            ph += tile_phases(run["stamps"], run["ntiles"], run["grid"])
            layer_us.append((run["stamps"][:, 4].max() - run["stamps"][:, 0].min()) / 1e3)
        med = {k: statistics.median(p[k] for p in ph) for k in ph[0]}
        r0 = runs[0]
        rec = dict(index=r["index"], op=r["op"], cin=r["cin"], cout=r["cout"], k=r["k"], residual=bool(r0["res"]), KI=r0["KI"],
                   tiles=r0["ntiles"], ctas=r0["grid"], median_us=med, layer_us=statistics.median(layer_us))
        report["layers"].append(rec)
        print("%3d %-9s %5d %5d %2d %3s %3d %5d %4d %7.2f %7.2f %7.2f %7.2f %7.2f %7.2f %8.1f" % (
            r["index"], r["op"], r["cin"], r["cout"], r["k"], "yes" if r0["res"] else "", r0["KI"], r0["ntiles"], r0["grid"], med["wait_k0"], med["k_loop"], med["resid"], med["epi"], med["tile"], med["lead"], rec["layer_us"]))
    with open(os.path.join(args.out, "conv_tile_timeline.json"), "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
