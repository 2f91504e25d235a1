"""Engine 4 ('f16x3'): fp16 hi / lo split operands on wgmma - three MMAs per MAC, 22 significand bits - against fp64
references of the same operands.  The bar is fp32-GRADE: every output element within 2^-22 of itself plus the accumulation
allowance of tests/wgmma_ref.py (far below what 11-bit arithmetic gives), i.e. what separates an fp32 convolution from another
fp32 convolution with a different accumulation order."""
import ctypes as C

import numpy as np
import pytest
import torch

import wgmma_ref as R
from oracle import synth
from test_gpu_ops import ragged

pytestmark = pytest.mark.gpu
TW_SWEEP_S1, TW_SWEEP_S2, ring_cases, _inputs = R.TW_SWEEP_S1, R.TW_SWEEP_S2, R.ring_cases, R.conv_inputs


def sragged(rf, xs):
    r = ragged(rf, xs)
    return rf.ops.Ragged(rf.ops.to_split(r.data), r.hw)


def test_split_roundtrip(rf):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(1000, 64, generator=g) * torch.logspace(-6, 4, 1000).view(-1, 1)).cuda()
    s = rf.ops.to_split(x)
    back = rf.ops.from_split(s)
    assert s.shape == (2, 1000, 64) and s.dtype == torch.float16
    # 22 significand bits for normal fp16 hi parts (|x| >= 2^-14); an absolute floor of 2^-35 below (fp16 subnormals)
    assert bool(((back - x).abs() <= torch.maximum(x.abs() * 2.0 ** -22, torch.tensor(2.0 ** -35, device="cuda"))).all())


SPLIT_CASES = [
    (64, 64, 3, [(24, 32), (9, 7)]), (64, 64, 3, [(120, 160), (60, 80), (33, 47)]), (64, 64, 1, [(16, 16)]),
    (64, 256, 1, [(13, 17), (6, 5), (1, 1)]), (128, 128, 3, [(16, 16), (16, 16)]), (256, 64, 1, [(30, 40)]),
    (1024, 256, 1, [(15, 20), (30, 40)]), (256, 256, 3, [(15, 20), (33, 25)]), (256, 1024, 1, [(20, 15), (40, 30)]),
    (512, 128, 1, [(60, 80)]), (192, 64, 1, [(37, 53)]), (64, 48, 3, [(12, 20)]), (128, 8, 3, [(6, 8)]), (512, 2048, 1, [(9, 5)]),
    (64, 512, 3, [(60, 80)]),
    # partial N tiles of BN = 128
    (64, 72, 3, [(9, 13)]), (64, 136, 1, [(11, 7)]), (128, 200, 3, [(6, 5), (1, 1)]),
    (64, 72, 3, TW_SWEEP_S1), (64, 136, 3, TW_SWEEP_S2)] + ring_cases("split")


@pytest.mark.parametrize("cin,cout,k,sizes", SPLIT_CASES)
@pytest.mark.parametrize("relu,res,stride", [(True, True, 1), (False, False, 1), (True, False, 2)])
def test_conv2d_split(rf, cin, cout, k, sizes, relu, res, stride):
    """Engine 4: the reference convolves the 22-bit split values (hi + lo * 2^-11) of input, weights and residual in fp64."""
    xs, w, bias, rs = _inputs(cin + cout * 3 + k, cin, cout, k, sizes, res, stride)
    _, y = R.check_conv(rf, 4, xs, w, bias, rs, stride, relu, "split %dx%d %d->%d stride %d" % (k, k, cin, cout, stride))
    assert y.dim() == 3 and y.dtype == torch.float16


DUAL_CASES = [
    (64, 64, 256, 1, [(60, 80), (13, 17), (1, 1)]), (128, 256, 512, 2, [(31, 41), (30, 40), (7, 5)]), (256, 512, 1024, 2, [(15, 20), (8, 11)]),
    (64, 128, 64, 2, [(9, 9)]),
    # Cin1 != Cin2: the switch from the first input's tensor map to the second's (kc1 = Cin1 / 64 K blocks) at different ring
    # phases (STAGES = 2 for BN 64, 3 for BN 128), partial N tiles
    (64, 128, 56, 1, [(7, 9)]), (128, 64, 56, 2, [(13, 11)]), (192, 128, 120, 1, [(6, 10), (3, 2)]), (128, 320, 120, 2, [(9, 7)]),
    (320, 64, 200, 1, [(5, 8)]), (256, 192, 136, 2, [(12, 17)]),
    # stride2 = 2 with tile width 128: the 256-pixel TMA box on the second input
    (64, 64, 64, 2, [(2, 256), (1, 255)])]


@pytest.mark.parametrize("c1,c2,cout,stride2,sizes", DUAL_CASES)
@pytest.mark.parametrize("relu", [True, False])
def test_conv1x1_dual_split(rf, c1, c2, cout, stride2, sizes, relu):
    """conv3 + down-sampling branch as one GEMM over two inputs == the two convolutions added, in fp64 on the split operands,
    element by element, into a NaN-filled output."""
    g = torch.Generator().manual_seed(c1 + 3 * c2 + cout + stride2)
    x2s = [torch.randn(1, c2, h, w, generator=g) for h, w in sizes]                                    # the block's input
    x1s = [torch.randn(1, c1, (h - 1) // stride2 + 1, (w - 1) // stride2 + 1, generator=g) for h, w in sizes]   # conv2's output
    w1 = torch.randn(cout, c1, generator=g) / np.sqrt(c1)
    w2 = torch.randn(cout, c2, generator=g) / np.sqrt(c2)
    bias = torch.randn(cout, generator=g)
    worst, y = dual_check(rf, x1s, x2s, w1, w2, bias, stride2, relu)
    print("dual 1x1 %d + %d -> %d stride2 %d: worst error / allowance %.3g" % (c1, c2, cout, stride2, worst))


def dual_call(rf, s1, s2, hw1, hw2, c1, c2, stride2, ws, bias, relu, y):
    """rf_conv1x1_dual_split into a caller-owned output."""
    lib, ptr = rf._lib.lib, rf._lib.ptr
    a = (C.c_int * (2 * len(hw1)))(*[v for p in hw1 for v in p])
    b = (C.c_int * (2 * len(hw2)))(*[v for p in hw2 for v in p])
    rf._lib.check(lib.rf_conv1x1_dual_split(ptr(s1), ptr(s2), len(hw1), a, b, c1, c2, int(stride2), ptr(ws), ptr(bias), ws.shape[1],
                                            int(relu), ptr(y), rf._lib.stream()))
    return y


def dual_check(rf, x1s, x2s, w1, w2, bias, stride2, relu):
    c1, c2, cout = x1s[0].shape[1], x2s[0].shape[1], w1.shape[0]
    hw1 = [(x.shape[2], x.shape[3]) for x in x1s]
    hw2 = [(x.shape[2], x.shape[3]) for x in x2s]
    s1, q1 = R.operand(R.nhwc(x1s), "split")
    s2, q2 = R.operand(R.nhwc(x2s), "split")
    ws, wq = R.operand(torch.cat([w1, w2], dim=1).contiguous(), "split")
    y = R.nan_output((2, sum(h * w for h, w in hw1), cout), torch.float16)
    dual_call(rf, s1.contiguous().cuda(), s2.contiguous().cuda(), hw1, hw2, c1, c2, stride2, ws.contiguous().cuda(), bias.cuda(), relu, y)
    torch.cuda.synchronize()
    got = R.images(R.from_split(y), hw1)
    wq, bq = wq.cuda(), bias.cuda()
    worst = 0.0
    for i, (a, b) in enumerate(zip(R.images(q1.cuda(), hw1), R.images(q2.cuda(), hw2))):
        b = b[:, :, ::stride2, ::stride2]
        ra, aa = R.conv_ref(a, wq[:, :c1, None, None], bq)
        rb, ab = R.conv_ref(b, wq[:, c1:, None, None])
        ref, absref = ra + rb, aa + ab
        if relu:
            ref = ref.clamp_min(0.0)
        worst = max(worst, R.check(got[i], ref, absref, R.R_SPLIT, R.ACC["split"], R.ATOL["split"], "dual image %d" % i))
    return worst, y


def test_dual_rejects_mismatched_sizes(rf):
    g = torch.Generator().manual_seed(0)
    s1 = sragged(rf, [torch.randn(1, 64, 8, 8, generator=g)])
    s2 = sragged(rf, [torch.randn(1, 64, 8, 8, generator=g)])
    ws = rf.ops.to_split(torch.randn(64, 128, generator=g).cuda())
    with pytest.raises(rf._lib.RFError):     # stride 2 on an 8 x 8 second input gives 4 x 4, not the first input's 8 x 8
        rf.ops.conv1x1_dual_split(s1, s2, 2, ws, None, True)


def test_resnet50_split_fused_downsample_matches_unfused(rf):
    """The trunk with conv3 + down-sampling fused == the plain topology to split precision (one fp32 accumulation instead of
    two rounded-to-22-bit halves added: differences of a few 1e-7 of the feature scale)."""
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4(synth.resnet50_conv4_state(0), device="cuda")
    g = torch.Generator().manual_seed(5)
    x = ragged(rf, [torch.rand(1, 3, 96, 128, generator=g), torch.rand(1, 3, 70, 50, generator=g)])
    outs = []
    for fuse in (True, False):
        P = net._build(64, fuse_downsample=fuse)
        out, ohw = P.run(x, rf.ops.ENGINE_SPLIT)
        outs.append(rf.ops.from_split(out.clone()))
        assert sum(1 for o in P.ops if o[0] == 6) == (3 if fuse else 0)
    torch.cuda.synchronize()
    scale = outs[1].abs().max().item()
    assert (outs[0] - outs[1]).abs().max().item() <= 2e-5 * max(1.0, scale), ((outs[0] - outs[1]).abs().max().item(), scale)


SPLIT_OUT32_CASES = [
    (128, 49, 3, [(60, 80)]), (128, 1, 3, [(6, 8), (6, 8)]), (64, 49, 3, [(12, 16)]),
    # partial N tiles of BN = 128; odd Cout switches the float2 store to the scalar one
    (64, 72, 3, [(9, 13)]), (64, 136, 1, [(11, 7)]), (128, 200, 3, [(6, 5), (1, 1)]), (64, 65, 3, [(7, 9)]), (64, 97, 1, [(12, 10)]),
    (128, 129, 3, [(5, 6)]),
    (64, 49, 3, TW_SWEEP_S1), (64, 97, 3, TW_SWEEP_S2)] + ring_cases("split", couts=(49, 129))


@pytest.mark.parametrize("cin,cout,k,sizes", SPLIT_OUT32_CASES)
@pytest.mark.parametrize("stride,bias", [(1, False), (1, True), (2, True)])
def test_conv2d_split_fp32_output(rf, cin, cout, k, sizes, stride, bias):
    """Engine 5: split operands, plain fp32 rows out (the 49- / 1-channel last layers of the heads), not rounded."""
    xs, w, b, _ = _inputs(cin + cout, cin, cout, k, sizes, False, stride)
    _, y = R.check_conv(rf, 5, xs, w, b if bias else None, None, stride, False, "split->fp32 %dx%d %d->%d stride %d" % (k, k, cin, cout, stride))
    assert y.dtype == torch.float32 and y.shape[1] == cout


def test_split_engine_rejects_unsupported_shapes(rf):
    x = torch.randn(1, 32, 4, 4)
    with pytest.raises(rf._lib.RFError):     # Cin % 64 != 0: no silent fallback
        rf.ops.conv2d(sragged(rf, [x]), None, None, 8, 1, 1, 0, False, None, rf.ops.ENGINE_SPLIT,
                      rf.ops.to_split(torch.randn(8, 32).cuda()))


def test_resnet50_conv4_split_engine_is_fp32_grade(rf):
    """The whole trunk (43 convolutions) on the split engine against the exact-FMA fp32 engine: the normalised features
    differ by fp32-rounding-level amounts, two orders of magnitude below the fp16 / TF32 engines."""
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4(synth.resnet50_conv4_state(0))
    g = torch.Generator().manual_seed(1)
    xs = [torch.randn(1, 3, 96, 128, generator=g), torch.randn(1, 3, 64, 48, generator=g)]
    x = ragged(rf, xs)
    try:
        rf.model.set_engine("fp32")
        f32 = net(x)
        ref = rf.ops.l2norm(f32.data).clone()
        scale = f32.data.abs().max().item()
        rf.model.set_engine("f16x3")
        fs = net(x)
        assert fs.split and fs.hw == f32.hw
        raw = (rf.ops.from_split(fs.data) - f32.data).abs().max().item() / scale
        got = rf.ops.l2norm(fs.data)
    finally:
        rf.model.set_engine("fp32")
    err = (got - ref).abs().max().item()
    print("split trunk vs fp32 engine: raw rel %.3g, normalised features max abs %.3g (max |f| %.3g)" % (raw, err, ref.abs().max().item()))
    assert raw < 3e-5 and err < 2e-6          # raw: 40-odd layers of two fp32-grade engines drifting apart (measured 1.6e-5 .. 2.1e-5)


def test_fine_networks_split_engine_is_fp32_grade(rf):
    """FeatureExtractor + CorrNeigh + both heads on the split engine vs the fp32 engine."""
    from test_gpu_pair import networks
    g = torch.Generator().manual_seed(2)
    It = torch.rand(1, 3, 96, 128, generator=g).cuda()
    Is = (It + 0.05 * torch.rand(1, 3, 96, 128, generator=g).cuda()).clamp(0, 1)
    outs = {}
    try:
        for eng in ("fp32", "f16x3"):
            rf.model.set_engine(eng)
            net = networks(rf)
            ft = rf.pipeline.fine_features(net["netFeatCoarse"], It)
            flowCoarse = rf.pipeline.base_grid(96, 128)
            f12, m, f8, mb = rf.pipeline.PredFlowMask_device(Is, ft, flowCoarse, (96, 128), net, with_match21=True)
            outs[eng] = (ft.data.clone(), f12.clone(), m.clone(), f8.clone(), mb.clone())
    finally:
        rf.model.set_engine("fp32")
    names = ("features", "flow12", "match", "flowDown8", "matchDown8")
    for n, a, b in zip(names, outs["fp32"], outs["f16x3"]):
        d = (a - b).abs().max().item()
        print("split fine nets vs fp32 engine: |%s| diff %.3g" % (n, d))
        assert d < (4e-6 if n == "features" else 1e-4), (n, d)
