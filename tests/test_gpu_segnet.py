"""segNet on the split engine: dilated convolutions, the deep-stem im2col, the PPM kernels and the vote against fp64 references on
the operands the kernels consume; PIL BILINEAR resizes byte for byte; the whole network against the fp64 oracle and the
reference's golden masks up to proven ties; and a reference-style driver with --segNet through the drop-in."""
import ctypes as C
import os
import textwrap

import numpy as np
import PIL.Image as Image
import pytest
import torch
import torch.nn.functional as F

import wgmma_ref as R
from conftest import ROOT, golden
from oracle import seg_oracle as SO
from oracle import synth

pytestmark = pytest.mark.gpu


def _ints(v):
    return (C.c_int * len(v))(*[int(x) for x in v])


def _hw(sizes):
    return _ints([v for p in sizes for v in p])


# ------------------------------------------------------------------ dilated 3x3 convolutions (engine 4, rf_layer_t.dil)
def dilated_check(rf, sizes, cin, cout, d, res, relu, seed):
    from ransac_flow_b200.model import FoldedConv
    from ransac_flow_b200.program import LayerProgram
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, 3, 3, generator=g) / float(np.sqrt(9 * cin))
    bias = torch.randn(cout, generator=g)
    fc = FoldedConv(w, None, 1, pad=d, device="cuda")
    fc.bias = bias.cuda()
    P = LayerProgram(cin, device="cuda")
    P.conv(0, fc, relu=relu, res=0 if res else None, dil=d)
    xd, xq = R.operand(R.nhwc(xs), "split")
    out, ohw = P.run(rf.ops.Ragged(xd.contiguous().cuda(), sizes), 4)
    torch.cuda.synchronize()
    assert ohw == list(sizes)
    wq = R.from_split(fc.w_split).view(cout, 3, 3, cin).permute(0, 3, 1, 2).cuda()
    got = R.images(R.from_split(out), ohw)
    worst = 0.0
    for i, xi in enumerate(R.images(xq.cuda(), sizes)):
        ref = F.conv2d(xi, wq, bias.double().cuda(), padding=d, dilation=d)
        absref = F.conv2d(xi.abs(), wq.abs(), bias.double().abs().cuda(), padding=d, dilation=d)
        if res:
            ref, absref = ref + xi, absref + xi.abs()
        if relu:
            ref = ref.clamp_min(0.0)
        worst = max(worst, R.check(got[i], ref, absref, R.R_SPLIT, R.ACC["split"], R.ATOL["split"], "dil %d image %d" % (d, i)))
    print("dilation %d %s cout %d res %s relu %s: worst error / allowance %.3g" % (d, sizes, cout, res, relu, worst))


@pytest.mark.parametrize("d", [2, 4])
@pytest.mark.parametrize("res,relu", [(False, True), (True, True), (True, False), (False, False)])
def test_dilated_conv_ragged(rf, d, res, relu):
    sizes = [(19, 23), (3, 5), (47, 63), (1, 1)]          # the second and fourth are smaller than the dilation's reach
    dilated_check(rf, sizes, 128, 128, d, res, relu, 10 * d + 2 * res + relu)


@pytest.mark.parametrize("d", [2, 4])
def test_dilated_conv_partial_n_tile(rf, d):
    dilated_check(rf, [(3, 5), (17, 40)], 64, 200, d, False, True, 7 + d)


def test_dilation_refused_outside_engine_4(rf):
    from ransac_flow_b200.model import FoldedConv
    from ransac_flow_b200.program import LayerProgram
    fc = FoldedConv(torch.randn(64, 64, 3, 3) / 24, None, 1, pad=2, device="cuda")
    P = LayerProgram(64, device="cuda")
    P.conv(0, fc, relu=True, dil=2)
    with pytest.raises(AssertionError):
        P.run(rf.ops.Ragged(torch.zeros(16 * 16, 64, device="cuda"), [(16, 16)]), 0)
    # the library refuses it too, whatever the caller
    P.split_only = False
    with pytest.raises(rf._lib.RFError, match="dilation"):
        P.run(rf.ops.Ragged(torch.zeros(16 * 16, 64, device="cuda"), [(16, 16)]), 1)


def test_resnet50_program_with_explicit_dil_1_is_bit_identical(rf):
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4(synth.resnet50_conv4_state(0))
    P = net._build(64, fuse_downsample=True)
    Q = net._build(64, fuse_downsample=True)
    for i, o in enumerate(Q.ops):
        if o[0] == 0:
            Q.dil[i] = 1
    src, _, _ = synth.make_pair(5, 96, 128)
    x = rf.ops.Ragged(rf.ops.preproc_u8(torch.from_numpy(src).cuda().reshape(-1, 3), normalize=True), [(96, 128)])
    a = P.run(x, 4)[0].clone()
    b = Q.run(x, 4)[0].clone()
    for L in P._compiled[next(iter(P._compiled))]["layers"]:
        L.dil = 0          # a zero-filled field, as every program that predates the field passes: the same result
    c = P.run(x, 4)[0]
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(a.view(torch.int16), c.view(torch.int16))


# ------------------------------------------------------------------ deep-stem im2col, adaptive pooling, PPM concat
def test_deep_stem_conv(rf):
    """RF_OP_STEM3: segNet's 3x3 / stride 2 / pad 1, 3 -> 64 stem conv + BN + ReLU on the fp32 image, exact fp32 FMA, split output;
    ragged batch with images smaller than the kernel."""
    from ransac_flow_b200.program import LayerProgram
    sizes = [(304, 400), (33, 17), (1, 1), (2, 3)]
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]
    weight = torch.randn(64, 3, 3, 3, generator=g) / 5
    bn = torch.nn.BatchNorm2d(64).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(64, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(64, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(64, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(64, generator=g) + 0.5)
    P = LayerProgram(3, device="cuda")
    P.stem3(0, weight, bn)
    fc = P.ops[0][9]
    out, ohw = P.run(rf.ops.Ragged(R.nhwc(xs).cuda(), sizes), 4)
    torch.cuda.synchronize()
    assert ohw == [R.out_hw(h, w, 3, 2, 1) for h, w in sizes]
    wq = fc.w.double().view(3, 3, 3, 64).permute(3, 2, 0, 1).cpu()          # [27][64] (r, s, c) rows -> (64, 3, 3, 3)
    got = R.images(R.from_split(out).cpu(), ohw)
    for i, x in enumerate(xs):
        ref, absref = R.conv_ref(x, wq, fc.bias.cpu(), None, 2, 1, relu=True)
        R.check(got[i], ref, absref, R.R_SPLIT, 2.0 ** -18, R.ATOL["split"], "stem3 image %d" % i)
    with pytest.raises(AssertionError):                                      # split engine only
        P.run(rf.ops.Ragged(R.nhwc(xs).cuda(), sizes), 2)


def _split_in(rf, sizes, cch, seed):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(1, cch, h, w, generator=g) * 3 for h, w in sizes]
    xd, xq = R.operand(R.nhwc(xs), "split")
    return xd.contiguous().cuda(), R.images(xq, sizes)


@pytest.mark.parametrize("sizes", [[(1, 1)], [(2, 7)], [(5, 3)], [(47, 63)], [(5, 9), (1, 4), (47, 63), (6, 6), (13, 2)]],
                         ids=["h1", "h2", "h5", "47x63", "ragged"])
def test_adaptive_avgpool(rf, sizes):
    cch, bins = 64, (1, 2, 3, 6)
    xd, xq = _split_in(rf, sizes, cch, 4)
    n = len(sizes)
    ys = [torch.full((2, n * b * b, cch), float("nan"), device="cuda", dtype=torch.float16) for b in bins]
    ptrs = (C.c_void_p * 4)(*[y.data_ptr() for y in ys])
    rf._lib.check(rf._lib.lib.rf_adaptive_avgpool_split(xd.data_ptr(), n, _hw(sizes), cch, _ints(bins), 4, ptrs, rf._lib.stream()))
    torch.cuda.synchronize()
    for b, y in zip(bins, ys):
        got = R.images(R.from_split(y).cpu(), [(b, b)] * n)
        for i, xi in enumerate(xq):
            ref = F.adaptive_avg_pool2d(xi, b)
            absref = F.adaptive_avg_pool2d(xi.abs(), b)
            R.check(got[i], ref, absref, R.R_SPLIT, 2.0 ** -20, R.ATOL["split"], "bins %d image %d" % (b, i))


def test_ppm_concat(rf):
    sizes = [(5, 9), (1, 4), (47, 63), (13, 2)]
    n, c5, cb, bins = len(sizes), 64, 16, (1, 2, 3, 6)
    xd, xq = _split_in(rf, sizes, c5, 5)
    brs, brq = [], []
    for j, b in enumerate(bins):
        d, q = _split_in(rf, [(b, b)] * n, cb, 50 + j)
        brs.append(d)
        brq.append(q)
    P = sum(h * w for h, w in sizes)
    cy = c5 + 4 * cb
    y = torch.full((2, P, cy), float("nan"), device="cuda", dtype=torch.float16)
    ptrs = (C.c_void_p * 4)(*[t.data_ptr() for t in brs])
    rf._lib.check(rf._lib.lib.rf_ppm_concat_split(xd.data_ptr(), n, _hw(sizes), c5, ptrs, _ints(bins), 4, cb, y.data_ptr(), rf._lib.stream()))
    torch.cuda.synchronize()
    got = R.images(R.from_split(y).cpu(), sizes)
    for i, (h, w) in enumerate(sizes):
        assert torch.equal(got[i][:, :c5], xq[i])                      # conv5: copied bit for bit
        for j in range(4):
            # the source coordinates and weights are fp32 in ATen's fp32 kernel and in this one: the reference interpolates in fp32
            ref = F.interpolate(brq[j][i].float(), (h, w), mode="bilinear", align_corners=False).double()
            absref = F.interpolate(brq[j][i].abs(), (h, w), mode="bilinear", align_corners=False)
            R.check(got[i][:, c5 + j * cb:c5 + (j + 1) * cb], ref, absref, R.R_SPLIT, 2.0 ** -20, R.ATOL["split"], "branch %d image %d" % (j, i))


# ------------------------------------------------------------------ vote
def vote_call(rf, logits, sizes, order, H, W, segId, segFg):
    ncls = logits.shape[1]
    mask = torch.full((H, W), float("nan"), device="cuda")
    cls = torch.full((H, W), -1, device="cuda", dtype=torch.int32)
    scores = torch.full((H, W, ncls), float("nan"), device="cuda")
    rf._lib.check(rf._lib.lib.rf_seg_vote(logits.data_ptr(), len(sizes), _hw(sizes), ncls, _ints(order), len(order), H, W, segId, int(segFg),
                                          mask.data_ptr(), cls.data_ptr(), scores.data_ptr(), rf._lib.stream()))
    torch.cuda.synchronize()
    return mask.cpu().numpy(), cls.cpu().numpy(), scores.cpu().double()


def test_vote_against_fp64_with_repeats_and_ties(rf):
    sizes, order, H, W, ncls = [(4, 6), (7, 5), (1, 1)], [0, 1, 1, 1, 2], 13, 17, 150
    g = torch.Generator().manual_seed(9)
    logits = torch.randn(sum(h * w for h, w in sizes), ncls, generator=g) * 3
    logits[:, 7] = logits[:, 11] = -40.0
    logits[24:34, 7] = logits[24:34, 11] = 40.0     # the top two rows of the repeated scale: classes 7 and 11 tie exactly, 7 must win
    imgs = R.images(logits.double(), sizes)
    scores = torch.zeros(1, ncls, H, W, dtype=torch.float64)
    for k in order:
        up = F.interpolate(imgs[k].float(), (H, W), mode="bilinear", align_corners=False).double()     # fp32 coordinates, like ATen's
        scores = scores + torch.softmax(up, 1) / 5
    ref = scores[0].permute(1, 2, 0)
    for segId, segFg in ((2, False), (7, True), (7, False)):
        mask, cls, got = vote_call(rf, logits.cuda(), sizes, order, H, W, segId, segFg)
        assert float((got - ref).abs().max()) <= 1e-6
        s = np.sort(ref.numpy(), -1)
        decided = (s[..., -1] - s[..., -2]) > 2e-6
        assert np.array_equal(cls[decided], ref.numpy().argmax(-1)[decided])
        hit = (cls == segId).astype(np.float32)
        assert np.array_equal(mask, 1 - hit if segFg else hit)
        tie = got.numpy()[..., 7] == got.numpy()[..., 11]
        assert tie.any() and not (cls[tie] == 11).any()
    assert (cls == 7).any()


# ------------------------------------------------------------------ PIL BILINEAR
@pytest.mark.parametrize("src,dst", [((37, 53), (20, 11)), ((37, 53), (96, 81)), ((480, 640), (304, 400)), ((376, 1241), (152, 504)),
                                     ((29, 31), (376, 504))])
def test_bilinear_resize_is_pil(rf, src, dst):
    img = np.random.RandomState(src[0]).randint(0, 256, src + (3,)).astype(np.uint8)
    got = rf.ops.resize_bilinear_u8(torch.from_numpy(img).cuda(), dst[1], dst[0]).cpu().numpy()
    assert np.array_equal(got, np.asarray(Image.fromarray(img).resize((dst[1], dst[0]), Image.BILINEAR)))


# ------------------------------------------------------------------ whole network
@pytest.fixture(scope="module")
def segnets(rf):
    from ransac_flow_b200.segnet import SegNet
    sds = (synth.segnet_encoder_state(0), synth.segnet_decoder_state(0))
    return {v: SegNet(None, None, v[0], v[1], state_dicts=sds) for v in ((2, False), (1, True))}, sds


@pytest.mark.parametrize("seed,h,w", [(0, 96, 128), (1, 20, 400), (2, 64, 80)])
def test_getsky_against_fp64_oracle(rf, segnets, seed, h, w):
    nets, sds = segnets
    img = Image.fromarray(synth.segnet_image(seed, h, w))
    mask64, pred64, sc64, _ = SO.get_sky(sds[0], sds[1], img, 2, False, torch.float64)
    mask, cls, scores = nets[(2, False)].run(img, want_class=True, want_scores=True)
    dev = float((scores.double().cpu() - torch.from_numpy(sc64).permute(1, 2, 0)).abs().max())
    print("getSky %dx%d: max |score - fp64| = %.3g" % (h, w, dev))
    assert dev <= 1e-4
    top12, top1_seg = SO.margins(sc64, 2)
    diff = mask.cpu().numpy() != mask64
    assert (top1_seg[diff] <= 2 * dev).all(), int(diff.sum())
    assert (top12[cls.cpu().numpy() != pred64] <= 2 * dev).all()
    assert np.array_equal(nets[(2, False)].getSky(img), mask.cpu().numpy())


@pytest.mark.parametrize("seed,h,w", [(0, 96, 128), (1, 20, 400)])
@pytest.mark.parametrize("segId,segFg", [(2, False), (1, True)])
def test_getsky_against_reference_golden(rf, segnets, tmp_path, seed, h, w, segId, segFg):
    g = golden("segnet")
    tag = "%d_%d_%d" % (seed, segId, int(segFg))
    p = str(tmp_path / "img.png")
    Image.fromarray(synth.segnet_image(seed, h, w)).save(p)
    mask = segnets[0][(segId, segFg)].getSky(p)                 # a path, as the drivers pass it
    assert mask.dtype == np.float32 and mask.shape == (h, w)
    diff = mask != g["mask_" + tag]
    assert (g["margin_seg_" + tag][diff] <= 2e-4).all() and (g["margin12_" + tag][diff] <= 2e-4).all(), int(diff.sum())


def test_encoder_runs_once_on_a_ragged_batch(rf, segnets):
    net = segnets[0][(2, False)]
    img = Image.fromarray(synth.segnet_image(3, 480, 640))
    net.run(img)
    distinct, order = net.plan(480, 640)
    assert distinct == [(304, 400), (376, 504)] and order == [0, 1, 1, 1, 1]
    calls = []
    real = net.encoder.run
    net.encoder.run = lambda x, e: calls.append((list(x.hw), rf._lib.launch_count())) or real(x, e)
    try:
        before = rf._lib.launch_count()
        net.run(img)
        torch.cuda.synchronize()
        total = rf._lib.launch_count() - before
    finally:
        del net.encoder.run
    assert len(calls) == 1 and calls[0][0] == [(304, 400), (376, 504)]
    n_enc = len(net.encoder.ops)              # one launch per layer
    # 2 resizes x 2 passes, 1 preproc, the encoder, 1 pooling, 4 PPM convs, 1 concat, 2 conv_last, 1 vote
    assert total == 4 + 1 + n_enc + 1 + 4 + 1 + 2 + 1, total


# ------------------------------------------------------------------ a driver with --segNet through the drop-in
DRIVER = textwrap.dedent('''
    import sys
    sys.path.append('../../utils')
    import numpy as np, torch
    from PIL import Image
    from scipy.misc import imresize
    from coarseAlignFeatMatch import CoarseAlign
    import outil
    I1 = Image.open(sys.argv[1]).convert('RGB')
    I2 = Image.open(sys.argv[2]).convert('RGB')
    coarseModel = CoarseAlign(3, 500, 0.05, 'Homography', 96, 2, False, 1.5, True, True)
    coarseModel.setPair(I1, I2)
    Ith, Itw = coarseModel.It.size[1], coarseModel.It.size[0]
    It_bg = coarseModel.skyFromSeg(sys.argv[2])
    It_bg = (imresize(It_bg, (Ith, Itw)) < 128).astype(np.float32)
    fgMask = ((np.zeros((Ith, Itw)) + (1 - It_bg)) > 0.5).astype(np.float32)
    torch.manual_seed(7)
    bestPara = coarseModel.getCoarse(fgMask)
    np.save(sys.argv[3] + '/maskBG.npy', It_bg.astype(bool))
    np.save(sys.argv[3] + '/H.npy', np.zeros(1) if bestPara is None else bestPara)
''')


def test_dropin_driver_with_segnet(rf, tmp_path, monkeypatch):
    from ransac_flow_b200 import dropin
    from ransac_flow_b200.segnet import SegNet
    drv = tmp_path / "evaluation" / "evalHpatch"
    drv.mkdir(parents=True)
    (drv / "evaluation.py").write_text(DRIVER)
    src, tgt, _ = synth.make_pair(31, 96, 128)
    p1, p2 = str(tmp_path / "a.png"), str(tmp_path / "b.png")
    Image.fromarray(src).save(p1)
    Image.fromarray(tgt).save(p2)
    sds = (synth.segnet_encoder_state(0), synth.segnet_decoder_state(0))
    enc, dec, rsd = str(tmp_path / "enc.pth"), str(tmp_path / "dec.pth"), str(tmp_path / "r50.pth")
    torch.save(sds[0], enc)
    torch.save(sds[1], dec)
    torch.save(synth.resnet50_conv4_state(0), rsd)
    monkeypatch.setenv("RF_SEGNET_ENCODER", enc)
    monkeypatch.setenv("RF_SEGNET_DECODER", dec)
    monkeypatch.setenv("RF_RESNET50_WEIGHTS", rsd)
    monkeypatch.setattr("sys.argv", list(__import__("sys").argv))
    monkeypatch.chdir(tmp_path)
    saved = {k: __import__("sys").modules.get(k) for k in ("coarseAlignFeatMatch", "outil", "model", "kornia", "kornia.geometry")}
    try:
        dropin.main([str(drv / "evaluation.py"), p1, p2, str(tmp_path)])
    finally:
        for k, v in saved.items():
            if v is None:
                __import__("sys").modules.pop(k, None)
            else:
                __import__("sys").modules[k] = v
    maskBG = np.load(str(tmp_path / "maskBG.npy"))
    sky = SegNet(None, None, 2, False, state_dicts=sds).getSky(p2)
    ca = rf.CoarseAlignA(3, 500, 0.05, "Homography", 96, 2, False, 1.5, True, False, resnet_state_dict=synth.resnet50_conv4_state(0),
                         verbose=False)
    ca.setPair(Image.open(p1).convert("RGB"), Image.open(p2).convert("RGB"))
    Ith, Itw = ca.It.size[1], ca.It.size[0]
    expect = dropin.imresize(sky, (Ith, Itw)) < 128
    assert np.array_equal(maskBG, expect)
    torch.manual_seed(7)
    H = ca.getCoarse(((1 - expect.astype(np.float32)) > 0.5).astype(np.float32))
    Hd = np.load(str(tmp_path / "H.npy"))
    assert (H is None and Hd.shape == (1,)) or np.array_equal(Hd, H)
