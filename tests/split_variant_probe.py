"""Helper of tests/test_gpu_split_variants.py (not a test module): runs a fixed set of split-engine layers, the split trunk and
a correlation under whatever RF_FUSE_DOWNSAMPLE the environment holds (read when the trunk's split program is built) and saves
the outputs.
Usage: python tests/split_variant_probe.py OUT.npz"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ransac_flow_b200 as rf  # noqa: E402
from oracle import synth  # noqa: E402

dev = "cuda"
g = torch.Generator().manual_seed(12)


def sragged(sizes, c):
    xs = [torch.randn(h * w, c, generator=g) for h, w in sizes]
    return rf.ops.Ragged(rf.ops.to_split(torch.cat(xs).to(dev)), sizes)


out = {}
sizes = [(37, 53), (16, 24), (9, 5)]
# name: cin, cout, k, stride, residual
for name, cin, cout, k, stride, res in [("halo128", 128, 128, 3, 1, False), ("halo256res", 256, 256, 3, 1, True), ("halo64", 64, 64, 3, 1, False),
                                         ("shallow_ds", 64, 256, 1, 1, False), ("shallow_res", 64, 256, 1, 1, True), ("res_k256", 256, 1024, 1, 1, True),
                                         ("tap_deep", 512, 256, 1, 1, False), ("tap_s2", 128, 128, 3, 2, False)]:
    x = sragged(sizes, cin)
    w = rf.ops.to_split((torch.randn(cout, k * k * cin, generator=g) / np.sqrt(k * k * cin)).to(dev))
    b = torch.randn(cout, generator=g).to(dev)
    osz = [((h + 2 * (k // 2) - k) // stride + 1, (ww + 2 * (k // 2) - k) // stride + 1) for h, ww in sizes]
    r = sragged(osz, cout) if res else None
    y = rf.ops.conv2d(x, None, b, cout, k, stride, k // 2, True, r, rf.ops.ENGINE_SPLIT, w)
    out[name] = y.data.cpu().numpy().view(np.uint16)
# the trunk (fused or not, as the environment says) and the correlation on its features
from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4  # noqa: E402
rf.model.set_engine("f16x3")
net = ResNet50Conv4(synth.resnet50_conv4_state(0), device=dev)
img = rf.ops.Ragged(torch.rand(96 * 128 + 64 * 80, 3, generator=g).to(dev), [(96, 128), (64, 80)])
f = net(img)
out["trunk"] = rf.ops.from_split(f.data).cpu().numpy()
A = torch.nn.functional.normalize(torch.rand(700, 1024, generator=g), dim=1).to(dev)
B = torch.nn.functional.normalize(torch.rand(300, 1024, generator=g), dim=1).to(dev)
i1, i2, n = rf.ops.corr_mutual_nn(A, B, 2)
out["corr_i1"], out["corr_i2"] = i1[:int(n)].cpu().numpy(), i2[:int(n)].cpu().numpy()
torch.cuda.synchronize()
np.savez(sys.argv[1], **out)
print("saved", sorted(out))
