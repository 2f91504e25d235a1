"""Throughput of the MegaDepth validation (train/validation.py) on the device, and the time of its two kernels against the
torch compositions they replace.

    python tools/validation_profile.py [--pairs 24] [--kpts 400] [--engine f16x3] [--out result.json]

  pairs/s   : ``validation.validation`` over a synthetic dataset of PNG files (960 x 720 sources and targets, resized to
              640 x 480, ``--kpts`` keypoints per pair), against the reference's statements on this package's modules
              (PIL resize, ToTensor, ``F.affine_grid`` / ``F.grid_sample``, ``model.predFlowCoarse`` with its
              ``F.interpolate``, the full-resolution composition and ``alignmentError``'s per-keypoint ``.item()``); one
              warm-up pass each, then the timed pass, each ended by a device synchronise
  kernels   : CUDA events around 200 calls each, at 480 x 640 and 480 x 720: ``rf_affine_sample_u8`` against ToTensor +
              ``F.affine_grid`` + ``F.grid_sample``, and ``rf_val_keypoints`` against ``F.interpolate`` + grid + clamp +
              ``F.affine_grid`` + ``F.grid_sample`` + the estimate + the gather at the keypoints (on the device, no
              ``.item()``)

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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ransac_flow_b200 as rf  # noqa: E402
from oracle import synth  # noqa: E402

V = rf.validation


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def network(seed=1):
    net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7), "netFlowCoarse": rf.model.NetFlowCoarse(7)}
    net["netFeatCoarse"].load_state_dict(synth.feature_extractor_state(0))
    net["netFlowCoarse"].load_state_dict(synth.net_flow_coarse_state(seed))
    for m in net.values():
        m.cuda()
        m.eval()
    return net


def dataset(root, pairs, kpts, w0=960, h0=720):
    import pandas as pd
    rs = np.random.RandomState(0)
    rows, thetas = [], []
    for i in range(pairs):
        s, t, _ = synth.make_pair(100 + i, h0, w0)
        os.makedirs(os.path.join(root, "scene"), exist_ok=True)
        Image.fromarray(s).save(os.path.join(root, "scene", "s%d.png" % i))
        Image.fromarray(t).save(os.path.join(root, "scene", "t%d.png" % i))
        fmt = lambda a: ";".join("%.3f" % v for v in a)
        rows.append(dict(scene="scene", source_image="s%d.png" % i, target_image="t%d.png" % i,
                         XA=fmt(rs.uniform(0, w0 - 1, kpts)), YA=fmt(rs.uniform(0, h0 - 1, kpts)),
                         XB=fmt(rs.uniform(0, w0 - 1, kpts)), YB=fmt(rs.uniform(0, h0 - 1, kpts))))
        thetas.append(np.array([[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]], dtype=np.float32))
    return pd.DataFrame(rows, dtype=str), thetas


def reference_statements(df, valDir, inPklCoarse, network):
    """validation.py:56-110 as written, on this package's modules."""
    precAllAlign, totalAlign = np.zeros(8), 0
    with torch.no_grad():
        for i in range(len(df)):
            Is = Image.open(os.path.join(valDir, df["scene"][i], df["source_image"][i])).convert("RGB")
            Is, Xs, Ys = V.ResizeMinResolution(480, Is, df["XA"][i], df["YA"][i], 16)
            Isw, Ish = Is.size
            IsTensor = torch.from_numpy(np.array(Is)).permute(2, 0, 1)[None].float().div(255).cuda()
            It = Image.open(os.path.join(valDir, df["scene"][i], df["target_image"][i])).convert("RGB")
            It, Xt, Yt = V.ResizeMinResolution(480, It, df["XB"][i], df["YB"][i], 16)
            Itw, Ith = It.size
            ItTensor = torch.from_numpy(np.array(It)).permute(2, 0, 1)[None].float().div(255).cuda()
            gridY = torch.linspace(-1, 1, steps=Ith).view(1, -1, 1, 1).expand(1, Ith, Itw, 1)
            gridX = torch.linspace(-1, 1, steps=Itw).view(1, 1, -1, 1).expand(1, Ith, Itw, 1)
            grid = torch.cat((gridX, gridY), dim=3).cuda()
            flowGlobalT = F.affine_grid(torch.from_numpy(inPklCoarse[i]).unsqueeze(0).cuda(), ItTensor.size(), align_corners=False)
            IsSample = F.grid_sample(IsTensor, flowGlobalT, align_corners=False)
            featsSample = F.normalize(network["netFeatCoarse"](IsSample))
            featt = F.normalize(network["netFeatCoarse"](ItTensor))
            corr21 = network["netCorr"](featt, featsSample)
            _, flowCoarse = rf.model.predFlowCoarse(corr21, network["netFlowCoarse"], grid)
            flowFinal = F.grid_sample(flowGlobalT.permute(0, 3, 1, 2), flowCoarse, align_corners=False).permute(0, 2, 3, 1).contiguous()
            estimY = (flowFinal.narrow(3, 0, 1).view(1, 1, Ith, Itw) + 1) * 0.5 * (Isw - 1)
            estimX = (flowFinal.narrow(3, 1, 1).view(1, 1, Ith, Itw) + 1) * 0.5 * (Ish - 1)
            d = []
            for j in range(len(Xt)):
                xa, ya, xb, yb = int(Xs[j]), int(Ys[j]), int(Xt[j]), int(Yt[j])
                d.append(((estimY[0, 0, yb, xb].item() - xa) ** 2 + (estimX[0, 0, yb, xb].item() - ya) ** 2) ** 0.5)
            precAllAlign += np.sum(np.array(d).reshape(-1, 1) < V.PIXEL_GRID, axis=0)
            totalAlign += len(d)
    return precAllAlign / totalAlign


def pairs_per_s(fn, n):
    fn()                                              # warm-up: folded weights, layer programs, resampling tables
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0), out


def event_us(fn, calls=200):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return 1000.0 * a.elapsed_time(b) / calls


def kernel_times(H, W, kpts):
    rs = np.random.RandomState(1)
    src = torch.from_numpy(rs.randint(0, 256, (H, W, 3)).astype(np.uint8)).cuda()
    theta = torch.tensor([[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]], device="cuda")
    out = torch.empty((H * W, 3), device="cuda")
    fused_sample = event_us(lambda: V.affine_sample_u8(theta.reshape(-1), src, H, W, out=out))

    def torch_sample():
        t = src.permute(2, 0, 1)[None].float().div(255)
        return F.grid_sample(t, F.affine_grid(theta[None], (1, 3, H, W), align_corners=False), align_corners=False)
    torch_sample_us = event_us(torch_sample)
    flow8 = torch.from_numpy(rs.uniform(-0.05, 0.05, (1, 2, H // 8, W // 8)).astype(np.float32)).cuda()
    kp = torch.from_numpy(np.stack([rs.randint(0, W, kpts), rs.randint(0, H, kpts), rs.randint(0, W, kpts),
                                    rs.randint(0, H, kpts)], 1).astype(np.int32)).cuda()
    cnt = torch.tensor([kpts], dtype=torch.int32, device="cuda")
    acc = V.new_counts()
    fused_tail = event_us(lambda: V.val_keypoints(flow8, theta.reshape(-1), (H, W), (H, W), kp, cnt, acc))
    gy = torch.linspace(-1, 1, steps=H).view(1, -1, 1, 1).expand(1, H, W, 1)
    gx = torch.linspace(-1, 1, steps=W).view(1, 1, -1, 1).expand(1, H, W, 1)
    grid = torch.cat((gx, gy), dim=3).cuda()
    xb, yb = kp[:, 2].long(), kp[:, 3].long()

    def torch_tail():
        up = F.interpolate(flow8, scale_factor=8, mode="bilinear", align_corners=True)
        fc = torch.clamp(up.permute(0, 2, 3, 1) + grid, min=-1, max=1)
        g = F.affine_grid(theta[None], (1, 3, H, W), align_corners=False)
        ff = F.grid_sample(g.permute(0, 3, 1, 2), fc, align_corners=False).permute(0, 2, 3, 1)
        ex = (ff[0, yb, xb, 0] + 1) * 0.5 * (W - 1)
        ey = (ff[0, yb, xb, 1] + 1) * 0.5 * (H - 1)
        return ex, ey
    torch_tail_us = event_us(torch_tail)
    return dict(size="%dx%d" % (H, W), keypoints=kpts, affine_sample_us=fused_sample, torch_affine_sample_us=torch_sample_us,
                val_keypoints_us=fused_tail, torch_tail_us=torch_tail_us)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=24)
    ap.add_argument("--kpts", type=int, default=400)
    ap.add_argument("--engine", default="f16x3", choices=["f16x3", "fp32"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "validation_profile needs a GPU"
    rf.model.set_engine(args.engine)
    res = dict(gpu_info(), engine=args.engine, pairs=args.pairs, kpts_per_pair=args.kpts)
    with tempfile.TemporaryDirectory() as root:
        df, thetas = dataset(root, args.pairs, args.kpts)
        net = network()
        res["device_pairs_per_s"], p_dev = pairs_per_s(lambda: V.validation(df, root, thetas, net, None), args.pairs)
        res["reference_statements_pairs_per_s"], p_ref = pairs_per_s(lambda: reference_statements(df, root, thetas, net), args.pairs)
        res["prec_device"], res["prec_reference_statements"] = list(map(float, p_dev)), list(map(float, p_ref))
    res["kernels"] = [kernel_times(480, 640, args.kpts), kernel_times(480, 720, args.kpts)]
    res["gpu_after"] = gpu_info()["nvidia_smi"]
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
