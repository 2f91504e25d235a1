"""Networks on the CUDA engine vs golden outputs of the reference modules (fp32 engine)."""
import numpy as np
import pytest
import torch

from conftest import golden
from oracle import model_oracle as MO
from oracle import synth

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(1e-12, np.abs(b).max())


def test_feature_extractor_vs_reference(rf):
    g = golden("feature_extractor")
    fe = rf.model.FeatureExtractor()
    fe.load_state_dict(synth.feature_extractor_state(int(g["seed"])))
    fe.cuda()
    fe.eval()
    y = fe(torch.from_numpy(g["x"]).cuda())
    assert tuple(y.shape) == g["y"].shape
    assert rel_err(y.cpu().numpy(), g["y"]) < 1e-4
    # reload other weights: the folded cache must follow
    fe.load_state_dict(synth.feature_extractor_state(5))
    y2 = fe(torch.from_numpy(g["x"]).cuda())
    ref2 = MO.feature_extractor(torch.from_numpy(g["x"]), synth.feature_extractor_state(5))
    assert rel_err(y2.cpu().numpy(), ref2.numpy()) < 1e-4
    fe.train()
    with pytest.raises(RuntimeError):
        fe(torch.from_numpy(g["x"]).cuda())


def test_fine_heads_vs_reference(rf):
    g = golden("fine_heads")
    corr = rf.model.CorrNeigh(7)(torch.from_numpy(g["a"]).cuda(), torch.from_numpy(g["b"]).cuda())
    assert np.abs(corr.cpu().numpy() - g["corr"]).max() < 1e-6
    nf = rf.model.NetFlowCoarse(7)
    nf.load_state_dict(synth.net_flow_coarse_state(1))
    assert nf.cuda() is not None
    nf.eval()
    flow = nf(torch.from_numpy(g["corr"]).cuda(), False)
    assert np.abs(flow.cpu().numpy() - g["flow"]).max() < 1e-6          # flow in [-1,1] units: << 1e-3
    nm = rf.model.NetMatchability(7)
    nm.load_state_dict(synth.net_matchability_state(2))
    nm.cuda()
    nm.eval()
    m = nm(torch.from_numpy(g["corr"]).cuda(), False)
    assert np.abs(m.cpu().numpy() - g["match"]).max() < 1e-6
    grid = torch.zeros(1, 6, 8, 2).cuda()
    _, fc = rf.model.predFlowCoarse(torch.from_numpy(g["corr"]).cuda(), nf, grid, up8X=False)
    assert tuple(fc.shape) == (1, 6, 8, 2)


def test_resnet50_conv4_vs_torchvision(rf):
    g = golden("resnet50_conv4")
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4(synth.resnet50_conv4_state(int(g["seed"])))
    x = rf.ops.Ragged.from_nchw(torch.from_numpy(g["x"]).cuda())
    y = net(x)
    assert rel_err(y.to_nchw().cpu().numpy(), g["y"]) < 1e-4
    # ragged batch: two different sizes in one pass == each alone
    x2 = torch.randn(1, 3, 48, 80)
    xs = rf.ops.Ragged(torch.cat([x.data, x2[0].permute(1, 2, 0).reshape(-1, 3).cuda()]), [(64, 96), (48, 80)])
    ys = net(xs)
    assert rel_err(ys.image(0).cpu().numpy(), g["y"]) < 1e-4
    ref2 = MO.resnet50_conv4(x2, synth.resnet50_conv4_state(int(g["seed"])))
    assert rel_err(ys.image(1).cpu().numpy(), ref2.numpy()) < 1e-4


@pytest.mark.parametrize("engine", ["tf32", "f16"])
def test_fine_networks_on_tensor_core_engines(rf, engine):
    """FeatureExtractor and the two heads through the nn.Module API on the wgmma engines.  'f16': fp16 activations
    (stem patches of 64 halves, fp16 pool+blur / blur, kind::f16 convs; conv3 of the heads hands fp32 to the TF32 conv4).
    10-bit operands either way: outputs close to the fp32 golden values, flow error far below 1e-3."""
    g = golden("feature_extractor")
    h = golden("fine_heads")
    fe = rf.model.FeatureExtractor()
    fe.load_state_dict(synth.feature_extractor_state(int(g["seed"])))
    nf = rf.model.NetFlowCoarse(7)
    nf.load_state_dict(synth.net_flow_coarse_state(1))
    nm = rf.model.NetMatchability(7)
    nm.load_state_dict(synth.net_matchability_state(2))
    for m in (fe, nf, nm):
        m.cuda()
        m.eval()
    rf.model.set_engine(engine)
    try:
        y = fe(torch.from_numpy(g["x"]).cuda())
        flow = nf(torch.from_numpy(h["corr"]).cuda(), False)
        match = nm(torch.from_numpy(h["corr"]).cuda(), False)
    finally:
        rf.model.set_engine("fp32")
    assert y.dtype == torch.float32 and flow.dtype == torch.float32 and match.dtype == torch.float32
    e_fe = rel_err(y.cpu().numpy(), g["y"])
    e_flow = np.abs(flow.cpu().numpy() - h["flow"]).max()
    e_match = np.abs(match.cpu().numpy() - h["match"]).max()
    print("[%s] FeatureExtractor rel err %.3g, flow err %.3g, matchability err %.3g" % (engine, e_fe, e_flow, e_match))
    assert e_fe < 1e-2 and e_flow < 2e-4 and e_match < 1e-3


def test_resnet50_conv4_f16_engine(rf):
    """Engine 'f16': the trunk with fp16 activations (stem im2col -> 192-half rows, fp16 max-pool, every bottleneck on
    wgmma fp16).  10-bit operands like TF32: close to the fp32 golden output, and ragged == alone."""
    g = golden("resnet50_conv4")
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4(synth.resnet50_conv4_state(int(g["seed"])))
    x = rf.ops.Ragged.from_nchw(torch.from_numpy(g["x"]).cuda())
    rf.model.set_engine("f16")
    try:
        y = net(x)
        assert y.data.dtype == torch.float16
        y1 = y.to_nchw().float().cpu().numpy()
        e1 = rel_err(y1, g["y"])
        x2 = torch.randn(1, 3, 48, 80)
        xs = rf.ops.Ragged(torch.cat([x.data, x2[0].permute(1, 2, 0).reshape(-1, 3).cuda()]), [(64, 96), (48, 80)])
        ys = net(xs)
        y2 = ys.image(0).float().cpu().numpy()
        ref2 = MO.resnet50_conv4(x2, synth.resnet50_conv4_state(int(g["seed"])))
        e2 = rel_err(ys.image(1).float().cpu().numpy(), ref2.numpy())
        # normalised rows (what the matcher sees)
        n = rf.ops.l2norm(ys.data)
        assert n.dtype == torch.float32
        ref_n = torch.nn.functional.normalize(ys.data.float(), dim=1)
        assert (n - ref_n).abs().max().item() < 1e-6
    finally:
        rf.model.set_engine("fp32")
    print("f16 trunk: rel err %.3g (alone), %.3g (ragged second image)" % (e1, e2))
    assert e1 < 1e-2 and e2 < 1e-2
    assert np.array_equal(y1, y2)                 # tiles never mix images: bit-identical alone vs in a ragged batch


def test_trunk_fused_stem_equals_explicit_im2col_stem(rf):
    """RF_OP_STEM7 (patches built in shared memory, what the fp16 trunk runs) against im2col + 1x1 conv on the same fp16
    weights, over a ragged batch with sizes that are not multiples of the 16 x 8 tile."""
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    sd = synth.resnet50_conv4_state(3)
    g = torch.Generator().manual_seed(5)
    imgs = [torch.randn(h * w, 3, generator=g) for h, w in [(64, 96), (48, 80), (34, 50)]]
    x = rf.ops.Ragged(torch.cat(imgs).cuda(), [(64, 96), (48, 80), (34, 50)])
    rf.model.set_engine("f16")
    try:
        net = ResNet50Conv4(sd)
        fused = net(x).data.float().cpu().numpy().copy()
        assert 5 in [o[0] for o in net._program_f16.ops[:2]]
        plain = net._build(64, fused_stem=False)
        assert 5 not in [o[0] for o in plain.ops[:2]]
        im2col = plain.run(x, rf.ops.ENGINE_F16)[0].float().cpu().numpy().copy()
    finally:
        rf.model.set_engine("fp32")
    d = np.abs(im2col - fused).max()
    print("fused vs im2col stem: max |diff| of the conv4 features = %.3g (max %.3g)" % (d, np.abs(im2col).max()))
    assert d <= 2e-3 * max(1.0, np.abs(im2col).max())


@pytest.mark.parametrize("k,cin,cout,stride,pad", [(5, 2, 16, 1, 2), (3, 4, 32, 2, 1), (7, 3, 64, 2, 3), (3, 3, 64, 1, 1)])
@pytest.mark.parametrize("engine", ["fp32", "tf32"])
def test_stem_as_im2col_plus_1x1(rf, k, cin, cout, stride, pad, engine):
    """LayerProgram.stem (im2col + 1x1 conv) == conv + BN + ReLU, on a ragged batch (generic and specialised kernels)."""
    import torch.nn.functional as F
    from ransac_flow_b200.program import LayerProgram
    from ransac_flow_b200.coarseAlignFeatMatch import _BN
    g = torch.Generator().manual_seed(k * 10 + cin)
    w = torch.randn(cout, cin, k, k, generator=g) / np.sqrt(cin * k * k)
    sd = {"bn.weight": torch.rand(cout, generator=g) + 0.5, "bn.bias": torch.randn(cout, generator=g) * 0.1,
          "bn.running_mean": torch.randn(cout, generator=g) * 0.1, "bn.running_var": torch.rand(cout, generator=g) + 0.5}
    xs = [torch.randn(1, cin, 37, 150, generator=g), torch.randn(1, cin, 9, 11, generator=g)]
    refs = [F.relu(F.batch_norm(F.conv2d(x, w, stride=stride, padding=pad), sd["bn.running_mean"], sd["bn.running_var"],
                                sd["bn.weight"], sd["bn.bias"], False, 0.0, 1e-5)) for x in xs]
    P = LayerProgram(cin)
    P.stem(0, w.cuda(), _BN({k_: v.cuda() for k_, v in sd.items()}, "bn"), stride, pad)
    data = torch.cat([x[0].permute(1, 2, 0).reshape(-1, cin) for x in xs]).contiguous().cuda()
    out, ohw = P.run(rf.ops.Ragged(data, [(37, 150), (9, 11)]), 1 if engine == "tf32" else 0)
    y = rf.ops.Ragged(out, ohw)
    tol = 4e-3 if engine == "tf32" else 2e-5
    for i, r in enumerate(refs):
        assert tuple(y.image(i).shape) == tuple(r.shape)
        assert (y.image(i).cpu() - r).abs().max().item() <= tol * max(1.0, r.abs().max().item())
