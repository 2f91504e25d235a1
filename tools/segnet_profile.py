"""Time segNet's getSky on the GPU and break it into stages: resize (PIL BILINEAR + normalisation), encoder (one rf_run_layers
call over the distinct sizes), PPM (pooling, four 1x1 convs, concat), conv_last (3x3 + 150-class 1x1), vote.

    python tools/segnet_profile.py [--runs 20] [--warmup 5]

Seeded synthetic weights (synthdata) and images of 480 x 640 and 376 x 1241.  Times are CUDA-event medians over --runs calls
after --warmup calls.  Also printed: the GPU's name and power limit (read only) and the algorithmic FLOPs of the convolutions,
computed from the layer shapes (multiply-adds x 2 per distinct size; the split engine issues three fp16 MMAs per multiply-add).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def conv_flops(program, hw):
    """2 * MACs of every convolution of a LayerProgram for input sizes ``hw`` (from its compiled shapes)."""
    hws, total = [list(hw)], 0
    for i, o in enumerate(program.ops):
        op, src, _, cin, cout, k, s, p = o[:8]
        d = program.dil.get(i, 1)
        out = [((h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1) for h, w in hws[src]]
        hws.append(out)
        if op in (0, 6):
            kin = k * k * cin + (program.dual[i][1] if i in program.dual else 0)
            total += 2 * kin * cout * sum(h * w for h, w in out)
    return total, hws[-1]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in q.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("segnet_profile needs a CUDA device")
    import PIL.Image as Image
    import ransac_flow_b200  # noqa: F401
    import synthdata as S
    from ransac_flow_b200.segnet import POOL_SCALES, PPM_CHANNELS, SegNet
    net = SegNet(None, None, 2, False, state_dicts=(S.segnet_encoder_state(0), S.segnet_decoder_state(0)))
    name, power, clock = gpu_info()
    for H, W in ((480, 640), (376, 1241)):
        img = Image.fromarray(S.segnet_image(7, H, W))
        u8 = torch.from_numpy(np.array(img)).cuda()
        distinct, order = net.plan(H, W)
        stages = {k: [] for k in ("resize", "encoder", "ppm", "conv_last", "vote", "getSky")}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        with torch.no_grad():
            for it in range(args.warmup + args.runs):
                t0 = torch.cuda.Event(enable_timing=True)
                t0.record()
                net.getSky(img)                       # the whole call: host image -> host mask
                t1 = torch.cuda.Event(enable_timing=True)
                t1.record()
                ev[0].record()
                x = net.resize(u8, distinct)
                ev[1].record()
                c5 = net.encode(x)
                ev[2].record()
                cat = net.ppm(c5)
                ev[3].record()
                logits = net.conv_last(cat)
                ev[4].record()
                net.vote(logits, order, H, W)
                ev[5].record()
                torch.cuda.synchronize()
                if it >= args.warmup:
                    stages["getSky"].append(t0.elapsed_time(t1))
                    for k, name_ in enumerate(("resize", "encoder", "ppm", "conv_last", "vote")):
                        stages[name_].append(ev[k].elapsed_time(ev[k + 1]))
        enc_f, c5hw = conv_flops(net.encoder, distinct)
        P5 = sum(h * w for h, w in c5hw)
        dec_f = 2 * 2048 * PPM_CHANNELS * sum(b * b for b in POOL_SCALES) * len(distinct) + 2 * 9 * 4096 * 512 * P5 + 2 * 512 * 150 * P5
        print(json.dumps({"image": [H, W], "distinct_sizes": distinct, "pass_order": order,
                          "median_ms": {k: round(float(np.median(v)), 3) for k, v in stages.items()},
                          "algorithmic_tflop": round((enc_f + dec_f) / 1e12, 4), "gpu": name, "power_limit": power, "max_sm_clock": clock,
                          "runs": args.runs}))


if __name__ == "__main__":
    main()
