"""Engine 4 ('f16x3'): fp16 hi / lo split operands on wgmma - three MMAs per MAC, 22 significand bits - against fp64
references of the same operands.  The bar is fp32-GRADE: errors a few 1e-7 of the output scale, i.e. what separates an fp32
convolution from another fp32 convolution with a different accumulation order."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import synth
from test_gpu_ops import ragged

pytestmark = pytest.mark.gpu
SPLIT_TOL = 4e-6          # relative to max(1, |y|max): 22-bit operands (2^-22 per product) + the tensor core's fp32 accumulation,
                          # which truncates and grows with K


def sragged(rf, xs):
    r = ragged(rf, xs)
    return rf.ops.Ragged(rf.ops.to_split(r.data), r.hw)


def simage(rf, y, i):
    o = y.offsets()
    h, w = y.hw[i]
    d = rf.ops.from_split(y.data[:, o[i]:o[i + 1]].contiguous())
    return d.view(1, h, w, y.C).permute(0, 3, 1, 2)


def test_split_roundtrip(rf):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(1000, 64, generator=g) * torch.logspace(-6, 4, 1000).view(-1, 1)).cuda()
    s = rf.ops.to_split(x)
    back = rf.ops.from_split(s)
    assert s.shape == (2, 1000, 64) and s.dtype == torch.float16
    # 22 significand bits for normal fp16 hi parts (|x| >= 2^-14); an absolute floor of 2^-35 below (fp16 subnormals)
    assert bool(((back - x).abs() <= torch.maximum(x.abs() * 2.0 ** -22, torch.tensor(2.0 ** -35, device="cuda"))).all())


@pytest.mark.parametrize("cin,cout,k,sizes", [
    (64, 64, 3, [(24, 32), (9, 7)]), (64, 64, 3, [(120, 160), (60, 80), (33, 47)]), (64, 64, 1, [(16, 16)]),
    (64, 256, 1, [(13, 17), (6, 5), (1, 1)]), (128, 128, 3, [(16, 16), (16, 16)]), (256, 64, 1, [(30, 40)]),
    (1024, 256, 1, [(15, 20), (30, 40)]), (256, 256, 3, [(15, 20), (33, 25)]), (256, 1024, 1, [(20, 15), (40, 30)]),
    (512, 128, 1, [(60, 80)]), (192, 64, 1, [(37, 53)]), (64, 48, 3, [(12, 20)]), (128, 8, 3, [(6, 8)]), (512, 2048, 1, [(9, 5)]),
    (64, 512, 3, [(60, 80)])])
@pytest.mark.parametrize("relu,res,stride", [(True, True, 1), (False, False, 1), (True, False, 2)])
def test_conv2d_split(rf, cin, cout, k, sizes, relu, res, stride):
    g = torch.Generator().manual_seed(cin + cout * 3 + k)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, k, k, generator=g) / np.sqrt(cin * k * k)
    bias = torch.randn(cout, generator=g)
    sx = sragged(rf, xs)
    wt = w.permute(0, 2, 3, 1).reshape(cout, k * k * cin).contiguous().cuda()
    ws = rf.ops.to_split(wt)
    # the reference sees the operands the kernel sees (22-bit split values), in fp64
    xq = [simage(rf, sx, i).double().cpu() for i in range(len(xs))]
    wq = rf.ops.from_split(ws).double().cpu().view(cout, k, k, cin).permute(0, 3, 1, 2)
    refs = [F.conv2d(x, wq, bias.double(), stride=stride, padding=k // 2) for x in xq]
    sr = None
    if res:
        rs = [torch.randn(r.shape, generator=g) for r in refs]
        sr = sragged(rf, rs)
        refs = [a + simage(rf, sr, i).double().cpu() for i, a in enumerate(refs)]
    if relu:
        refs = [F.relu(r) for r in refs]
    y = rf.ops.conv2d(sx, None, bias.cuda(), cout, k, stride, k // 2, relu, sr, rf.ops.ENGINE_SPLIT, ws)
    torch.cuda.synchronize()
    assert y.split and y.data.dtype == torch.float16
    worst = 0.0
    for i, r in enumerate(refs):
        got = simage(rf, y, i).double().cpu()
        assert tuple(got.shape) == tuple(r.shape)
        err = (got - r).abs().max().item() / max(1.0, r.abs().max().item())
        worst = max(worst, err)
    print("split conv %dx%d %d->%d stride %d: rel err %.3g" % (k, k, cin, cout, stride, worst))
    assert worst <= SPLIT_TOL, worst


@pytest.mark.parametrize("c1,c2,cout,stride2,sizes", [
    (64, 64, 256, 1, [(60, 80), (13, 17), (1, 1)]), (128, 256, 512, 2, [(31, 41), (30, 40), (7, 5)]), (256, 512, 1024, 2, [(15, 20), (8, 11)]),
    (64, 128, 64, 2, [(9, 9)])])
@pytest.mark.parametrize("relu", [True, False])
def test_conv1x1_dual_split(rf, c1, c2, cout, stride2, sizes, relu):
    """conv3 + down-sampling branch as one GEMM over two inputs == the two convolutions added, in fp64 on the split operands."""
    g = torch.Generator().manual_seed(c1 + 3 * c2 + cout + stride2)
    x2s = [torch.randn(1, c2, h, w, generator=g) for h, w in sizes]                                    # the block's input
    x1s = [torch.randn(1, c1, (h - 1) // stride2 + 1, (w - 1) // stride2 + 1, generator=g) for h, w in sizes]   # conv2's output
    w1 = torch.randn(cout, c1, generator=g) / np.sqrt(c1)
    w2 = torch.randn(cout, c2, generator=g) / np.sqrt(c2)
    bias = torch.randn(cout, generator=g)
    s1, s2 = sragged(rf, x1s), sragged(rf, x2s)
    ws = rf.ops.to_split(torch.cat([w1, w2], dim=1).contiguous().cuda())
    wq = rf.ops.from_split(ws).double().cpu()
    y = rf.ops.conv1x1_dual_split(s1, s2, stride2, ws, bias.cuda(), relu)
    torch.cuda.synchronize()
    assert y.split and y.hw == s1.hw
    worst = 0.0
    for i in range(len(sizes)):
        a = simage(rf, s1, i).double().cpu()
        b = simage(rf, s2, i).double().cpu()[:, :, ::stride2, ::stride2]
        ref = F.conv2d(a, wq[:, :c1, None, None]) + F.conv2d(b, wq[:, c1:, None, None]) + bias.double().view(1, -1, 1, 1)
        ref = F.relu(ref) if relu else ref
        got = simage(rf, y, i).double().cpu()
        assert tuple(got.shape) == tuple(ref.shape)
        worst = max(worst, (got - ref).abs().max().item() / max(1.0, ref.abs().max().item()))
    assert worst <= SPLIT_TOL, worst


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


@pytest.mark.parametrize("cin,cout,sizes", [(128, 49, [(60, 80)]), (128, 1, [(6, 8), (6, 8)]), (64, 49, [(12, 16)])])
def test_conv2d_split_fp32_output(rf, cin, cout, sizes):
    """Engine 5: split operands, plain fp32 rows out (the 49- / 1-channel last layers of the heads)."""
    g = torch.Generator().manual_seed(cin + cout)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, 3, 3, generator=g) / np.sqrt(cin * 9)
    sx = sragged(rf, xs)
    ws = rf.ops.to_split(w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous().cuda())
    wq = rf.ops.from_split(ws).double().cpu().view(cout, 3, 3, cin).permute(0, 3, 1, 2)
    y = rf.ops.conv2d(sx, None, None, cout, 3, 1, 1, False, None, rf.ops.ENGINE_SPLIT + 1, ws)
    torch.cuda.synchronize()
    assert not y.split and y.data.dtype == torch.float32 and y.data.shape[1] == cout
    for i in range(len(xs)):
        ref = F.conv2d(simage(rf, sx, i).double().cpu(), wq, padding=1)
        err = (y.image(i).double().cpu() - ref).abs().max().item() / max(1.0, ref.abs().max().item())
        assert err <= SPLIT_TOL, err


def test_split_engine_rejects_unsupported_shapes(rf):
    x = torch.randn(1, 32, 4, 4)
    with pytest.raises(rf._lib.RFError):     # Cin % 64 != 0: no silent fallback
        rf.ops.conv2d(sragged(rf, [x]), None, None, 8, 1, 1, 0, False, None, rf.ops.ENGINE_SPLIT,
                      rf.ops.to_split(torch.randn(8, 32).cuda()))


def _run_program(rf, P, x, engine):
    out, ohw = P.run(x, engine)
    return rf.ops.Ragged(out.clone(), ohw)


def test_split_pool_blur_ops_vs_fp32_engine(rf):
    """maxpool / blur / poolblur on split tensors == the fp32 kernels on the same values (to split precision)."""
    from ransac_flow_b200.program import LayerProgram
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(1, 64, 21, 30, generator=g), torch.randn(1, 64, 8, 9, generator=g)]
    for build in (lambda P: P.maxpool(0, 3, 2, 1), lambda P: P.blur(0, 2), lambda P: P.poolblur(0), lambda P: P.blur(0, 1)):
        P = LayerProgram(64)
        build(P)
        sx = sragged(rf, xs)
        xr = rf.ops.Ragged(rf.ops.from_split(sx.data), sx.hw)
        ref = _run_program(rf, P, xr, rf.ops.ENGINE_FP32)
        got = _run_program(rf, P, sx, rf.ops.ENGINE_SPLIT)
        assert got.split and got.hw == ref.hw
        err = (rf.ops.from_split(got.data) - ref.data).abs().max().item()
        assert err < 1e-6 * max(1.0, ref.data.abs().max().item()), err


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
