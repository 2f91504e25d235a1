"""The drivers' sky mask on the device: ``ops.imresize_mask`` (SciPy 1.2's ``imresize(np.rot90(It_bg, k), (h, w)) < 128``) bit for
bit against ``dropin.imresize``; segNet and the background-masked hypothesis loop inside ``GraphedMultiAligner`` /
``ConcurrentAligner`` against the eager, host-steered loop; the device background in ``align_pair_yfcc``; and
``align_pair_kitti(It_bg=...)`` against the oracle's KITTI loop given the same background."""
import numpy as np
import PIL.Image as Image
import pytest
import torch

from oracle import pair_oracle as PO
from oracle import synth
from oracle import warp_oracle as WO
from test_gpu_pair import FLOW_TOL, fixed_randint, networks, oracle_net

pytestmark = pytest.mark.gpu


def expected_keep(m, h, w, k):
    from ransac_flow_b200.dropin import imresize
    return imresize(np.rot90(m, k), (h, w)) < 128


# ------------------------------------------------------------------ ops.imresize_mask
# (map H, W) -> (h, w): down- and up-scaling, one side unchanged (a skipped PIL pass), 1-pixel sides, KITTI's full size to itself
SIZES = [((96, 128), (48, 64)), ((37, 53), (96, 81)), ((60, 80), (30, 80)), ((60, 80), (60, 41)), ((1, 50), (7, 3)),
         ((40, 1), (1, 1)), ((5, 7), (1, 9)), ((376, 1241), (376, 1241)), ((31, 17), (17, 31))]


def maps(kind, H, W, seed):
    rs = np.random.RandomState(seed)
    if kind == "binary":
        return (rs.rand(H, W) < 0.3).astype(np.float32)
    if kind == "float":
        return rs.rand(H, W).astype(np.float32)
    return np.full((H, W), 1.0 if kind == "ones" else 0.0, dtype=np.float32)


@pytest.mark.parametrize("kind", ["binary", "float", "zeros", "ones"])
@pytest.mark.parametrize("k", [0, 1, 2, 3])
@pytest.mark.parametrize("src,dst", SIZES, ids=["%dx%d-%dx%d" % (s + d) for s, d in SIZES])
def test_imresize_mask_is_scipy_imresize(rf, kind, k, src, dst):
    m = maps(kind, src[0], src[1], 7 * k + src[0])
    h, w = dst
    got = rf.ops.imresize_mask(torch.from_numpy(m).cuda(), h, w, rot=k)
    assert got.dtype == torch.float32 and tuple(got.shape) == (h, w) and got.is_cuda
    ref = expected_keep(m, h, w, k)
    assert np.array_equal(got.cpu().numpy(), ref.astype(np.float32)), int((got.cpu().numpy() != ref).sum())
    if kind in ("zeros", "ones"):
        assert ref.all()                   # a constant map byte-scales to 0: every pixel is kept
    assert np.array_equal(rf.ops.imresize_mask(m, h, w, rot=k).cpu().numpy(), ref.astype(np.float32))     # a host map


@pytest.mark.parametrize("k", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["binary", "float"])
def test_imresize_mask_yfcc_rotated_targets(rf, k, kind):
    """The resized sizes of a 480x640 YFCC pair's four rotated targets at minSize 480 (no PIL pass) and at 96."""
    m = maps(kind, 480, 640, 11 + k)
    for h, w in ((480, 640), (96, 128)):
        h, w = (h, w) if k % 2 == 0 else (w, h)
        got = rf.ops.imresize_mask(torch.from_numpy(m).cuda(), h, w, rot=k).cpu().numpy()
        assert np.array_equal(got, expected_keep(m, h, w, k).astype(np.float32))


def test_bytescale_is_scipy_bytescale(rf):
    """The byte-scaled map itself, with a wide value range and negative values (fp32 arithmetic, as numpy on a float32 map)."""
    from ransac_flow_b200.dropin import imresize
    rs = np.random.RandomState(3)
    for m in (rs.randn(77, 131).astype(np.float32) * 1000, (rs.rand(300, 200) * 1e-3 - 5).astype(np.float32)):
        for k in range(4):
            got = rf.ops.bytescale_mask_u8(torch.from_numpy(m).cuda(), k).cpu().numpy()
            r = np.rot90(m, k)
            assert np.array_equal(got, imresize(r, r.shape))         # same size: PIL's resize copies


def test_imresize_mask_graph_replay(rf):
    H, W, h, w = 120, 160, 96, 128
    static = torch.from_numpy(maps("binary", H, W, 1)).cuda()
    for k in range(4):
        hh, ww = (h, w) if k % 2 == 0 else (w, h)
        rf.ops.imresize_mask(static, hh, ww, rot=k)                   # warm-up: the resampling tables
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = rf.ops.imresize_mask(static, hh, ww, rot=k)
        for seed in (2, 3):
            m = maps("float", H, W, seed + 10 * k)
            static.copy_(torch.from_numpy(m))
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy(), expected_keep(m, hh, ww, k).astype(np.float32))
            assert torch.equal(out, rf.ops.imresize_mask(static, hh, ww, rot=k))


# ------------------------------------------------------------------ segNet inside the graphed aligners
SDS = {}


def segnet_sds():
    if not SDS:
        SDS["sds"] = (synth.segnet_encoder_state(0), synth.segnet_decoder_state(0))
    return SDS["sds"]


def coarse_seg(rf, segId, nbScale=3, minSize=96):
    return rf.CoarseAlignA(nbScale, 1000, 0.05, "Homography", minSize, segId, False, 2, True, True, resnet_state_dict=synth.resnet50_conv4_state(0),
                           verbose=False, segnet_state_dicts=segnet_sds())


@pytest.fixture(scope="module")
def sky_pair(rf, tmp_path_factory):
    """A KITTI-shaped synthetic pair and the segNet class whose pixels cover the least of the target above 10 %: the background."""
    from ransac_flow_b200.segnet import SegNet
    src, tgt, _ = synth.make_pair(41, 96, 256)
    probe = SegNet(None, None, 2, False, state_dicts=segnet_sds())
    _, cls, _ = probe.run(torch.from_numpy(tgt).cuda(), want_class=True)
    ids, counts = np.unique(cls.cpu().numpy(), return_counts=True)
    frac = counts / counts.sum()
    ok = [(f, int(i)) for f, i in zip(frac, ids) if 0.1 <= f <= 0.9]
    assert ok, list(zip(ids.tolist(), frac.tolist()))
    path = str(tmp_path_factory.mktemp("sky") / "target.png")
    Image.fromarray(tgt).save(path)
    return dict(src=src, tgt=tgt, segId=min(ok)[1], path=path)


def test_graphed_segnet_pair_equals_the_steered_loop(rf, sky_pair):
    from ransac_flow_b200.dropin import imresize
    net = networks(rf)
    c = coarse_seg(rf, sky_pair["segId"])
    c.device_preproc = True
    s, t = torch.from_numpy(sky_pair["src"]).cuda(), torch.from_numpy(sky_pair["tgt"]).cuda()
    c.setPair(s, t)
    w, h = c.target_size
    bg = (imresize(c.skyFromSeg(sky_pair["path"]), (h, w)) < 128).astype(np.float32)
    print("background: %.1f %% of the %dx%d target (segId %d)" % (100 * (1 - bg.mean()), h, w, sky_pair["segId"]))
    assert 0.1 <= 1 - bg.mean() <= 0.9
    torch.manual_seed(5)
    a = rf.pipeline.align_pair_device(c, net, s, t, maxCoarse=3, with_match21=True, It_bg=bg)
    torch.manual_seed(5)
    b = rf.pipeline.align_pair_multi(c, net, s, t, maxCoarse=3, with_match21=True, segNet=True)
    torch.manual_seed(5)
    plain = rf.pipeline.align_pair_multi(c, net, s, t, maxCoarse=3, with_match21=True)
    assert len(a["H"]) >= 1 and len(b["H"]) == len(a["H"]) and np.array_equal(a["H"], b["H"])
    assert np.array_equal(a["flowDown8"], b["flowDown8"]) and np.array_equal(a["matchDown8"], b["matchDown8"]) and a["nbMatch"] == b["nbMatch"]
    assert b["It_bg"].dtype == bool and np.array_equal(b["It_bg"], bg.astype(bool))
    assert "It_bg" not in plain and not np.array_equal(plain["H"][0], b["H"][0]), "the background does not change the first hypothesis"
    ga = rf.pipeline.GraphedMultiAligner(c, net, maxCoarse=3, with_match21=True, segNet=True)
    ga.prepare(s, t)
    for _ in range(2):
        torch.manual_seed(5)
        g = ga(s, t)
        assert np.array_equal(g["H"], b["H"]) and np.array_equal(g["flowDown8"], b["flowDown8"]) and np.array_equal(g["matchDown8"], b["matchDown8"])
        assert g["nbMatch"] == b["nbMatch"] and np.array_equal(g["It_bg"], b["It_bg"])


def test_segnet_needs_a_segnet_model(rf):
    c = rf.CoarseAlignA(3, 1000, 0.05, "Homography", 96, 2, False, 2, True, False, resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False)
    with pytest.raises(NotImplementedError, match="segNet=True"):
        rf.pipeline.GraphedMultiAligner(c, networks(rf), segNet=True)
    src, tgt, _ = synth.make_pair(41, 96, 256)
    with pytest.raises(NotImplementedError, match="segNet=True"):
        rf.pipeline.align_pair_multi(c, networks(rf), Image.fromarray(src), Image.fromarray(tgt), maxCoarse=1, segNet=True)


def test_segnet_graph_launches_and_eviction(rf, sky_pair):
    net = networks(rf)
    c = coarse_seg(rf, sky_pair["segId"])
    seg = c.segNet
    s, t = torch.from_numpy(sky_pair["src"]).cuda(), torch.from_numpy(sky_pair["tgt"]).cuda()
    plain = rf.pipeline.GraphedMultiAligner(c, net, maxCoarse=2, with_match21=True)
    withseg = rf.pipeline.GraphedMultiAligner(c, net, maxCoarse=2, with_match21=True, segNet=True, max_graphs=1)
    n_plain = plain.prepare(s, t)["n_kernels"]
    rec = withseg.prepare(s, t)
    H, W = sky_pair["tgt"].shape[:2]
    distinct, _ = seg.plan(H, W)
    n0 = rf._lib.launch_count()
    seg.run(t)
    torch.cuda.synchronize()
    n_seg = rf._lib.launch_count() - n0
    # resize passes, 1 preproc, the encoder, 1 pooling, 4 PPM convs, 1 concat, 2 conv_last, 1 vote
    assert n_seg == sum((h != H) + (w != W) for h, w in distinct) + 1 + len(seg.encoder.ops) + 1 + 4 + 1 + 2 + 1
    w, h = c.target_size
    n_mask = 2 + (w != W) + (h != H)              # min / max + byte-scaling, then the PIL passes that run
    # + 1: the first hypothesis' RANSAC is masked too (the mask's bilinear reduction to the feature grid)
    print("graph kernels: %d without segNet, %d with (segNet %d, mask %d)" % (n_plain, rec["n_kernels"], n_seg, n_mask))
    assert rec["n_kernels"] == n_plain + n_seg + n_mask + 1
    mine = {(id(p), k) for p in (seg.encoder, seg.head) for k in p._compiled}
    assert mine and mine <= rec["prog_keys"]
    # a second input size evicts the first graph (max_graphs = 1) and the segNet buffers only it used
    src2, tgt2, _ = synth.make_pair(13, 120, 160)
    withseg.prepare(torch.from_numpy(src2).cuda(), torch.from_numpy(tgt2).cuda())
    left = {(id(p), k) for p in (seg.encoder, seg.head) for k in p._compiled}
    assert len(withseg.graphs) == 1 and not (mine & left) and left
    assert left <= withseg.graphs[next(iter(withseg.graphs))]["prog_keys"]


def test_eviction_keeps_what_another_aligner_graph_uses(rf, sky_pair):
    """Two aligners on one model: their graphs point into the same layer-program entries (the key is the image-set signature).
    B's eviction leaves every entry A's live graph uses, and A's next replay equals the eager pair bit for bit."""
    net = networks(rf)
    c = coarse_seg(rf, sky_pair["segId"])
    s, t = torch.from_numpy(sky_pair["src"]).cuda(), torch.from_numpy(sky_pair["tgt"]).cuda()
    A = rf.pipeline.GraphedMultiAligner(c, net, maxCoarse=2, with_match21=True)
    B = rf.pipeline.GraphedMultiAligner(c, net, maxCoarse=2, with_match21=True, segNet=True, max_graphs=1)
    a = A.prepare(s, t)
    b = B.prepare(s, t)
    shared = a["prog_keys"] & b["prog_keys"]
    assert shared and {(id(p), k) for p, k in a["pins"]} == a["prog_keys"]
    src2, tgt2, _ = synth.make_pair(13, 120, 160)
    B.prepare(torch.from_numpy(src2).cuda(), torch.from_numpy(tgt2).cuda())           # evicts B's first graph
    assert len(B.graphs) == 1 and all(r is not b for r in B.graphs.values())
    assert all(k in p._compiled for p, k in a["pins"]), "an entry A's live graph points into was freed"
    torch.manual_seed(5)
    got = A(s, t)
    torch.manual_seed(5)
    want = rf.pipeline.align_pair_multi(c, net, s, t, maxCoarse=2, with_match21=True)
    assert len(got["H"]) == len(want["H"]) >= 1
    for key in ("H", "flowDown8", "matchDown8"):
        assert np.array_equal(got[key], want[key]), key
    assert got["nbMatch"] == want["nbMatch"] and got["nbInlier"] == want["nbInlier"]


def test_two_lanes_with_segnet_equal_each_lane_alone(rf, sky_pair):
    segId = sky_pair["segId"]
    ca = rf.pipeline.ConcurrentAligner(lambda: (coarse_seg(rf, segId), networks(rf)), lanes=2, seed=3,
                                       make_aligner=lambda c, n: rf.pipeline.GraphedMultiAligner(c, n, maxCoarse=2, segNet=True))
    a, b = ca.lanes
    assert a.coarse.segNet is not b.coarse.segNet and a.coarse.segNet.encoder is not b.coarse.segNet.encoder
    srcB, tgtB, _ = synth.make_pair(42, 96, 256)
    P = [(torch.from_numpy(sky_pair["src"]).cuda(), torch.from_numpy(sky_pair["tgt"]).cuda()),
         (torch.from_numpy(srcB).cuda(), torch.from_numpy(tgtB).cuda())]
    pairs = [P[0], P[1], P[1], P[0]]
    ca.prepare(*P[0])
    ca.seed(3)                                    # the warm-up runs of the capture drew from the lanes' generators
    together = ca.run(pairs)
    ca.seed(3)
    for k in range(2):
        for i in range(k, len(pairs), 2):
            alone = ca.lanes[k](*pairs[i])
            for key in ("H", "flowDown8", "matchDown8", "It_bg"):
                assert np.array_equal(alone[key], together[i][key]), (k, i, key)
            assert alone["nbMatch"] == together[i]["nbMatch"]
    assert not together[0]["It_bg"].all()


# ------------------------------------------------------------------ the eager pair paths
def test_yfcc_device_background_equals_host_background(rf):
    from ransac_flow_b200.segnet import SegNet
    src, tgt, _ = synth.make_rotated_pair(81, 96, 128, 2)
    t = torch.from_numpy(tgt).cuda()
    _, cls, _ = SegNet(None, None, 2, False, state_dicts=segnet_sds()).run(t, want_class=True)
    ids, counts = np.unique(cls.cpu().numpy(), return_counts=True)
    small = [(f, int(i)) for f, i in zip(counts / counts.sum(), ids) if 0.05 <= f <= 0.5]     # the sky: a minority class
    sky_dev = SegNet(None, None, min(small)[1] if small else 0, False, state_dicts=segnet_sds()).run(t)[0]
    sky_host = sky_dev.cpu().numpy()
    if sky_host.all() or not sky_host.any():           # no such class: use a band of sky instead
        sky_dev = torch.zeros_like(sky_dev)
        sky_dev[:20] = 1
        sky_host = sky_dev.cpu().numpy()
    rs = np.random.RandomState(4)
    samples = [rs.randint(0, 2 ** 31, (1000, 4)).astype(np.int64) for _ in range(12)]
    net = networks(rf)
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    h_out = rf.pipeline.align_pair_yfcc(rf.CoarseAlignB(3, 1000, 0.05, "Homography", 96, 1, True, True, True, False, 2,
                                                        resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False),
                                        net, Is, It, maxCoarse=3, It_bg=sky_host, samples=samples)
    d_out = rf.pipeline.align_pair_yfcc(rf.CoarseAlignB(3, 1000, 0.05, "Homography", 96, 1, True, True, True, False, 2,
                                                        resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False),
                                        net, Is, It, maxCoarse=3, It_bg=sky_dev, samples=samples)
    print("YFCC: angle %d, scores %s, %d hypotheses" % (h_out["angle"], h_out["nbInlierRot"], len(h_out["H"])))
    assert d_out["angle"] == h_out["angle"] and d_out["nbInlierRot"] == h_out["nbInlierRot"]
    assert len(h_out["H"]) >= 1 and np.array_equal(d_out["H"], h_out["H"]) and d_out["nbMatch"] == h_out["nbMatch"]
    assert np.array_equal(d_out["flowDown8"], h_out["flowDown8"]) and np.array_equal(d_out["matchDown8"], h_out["matchDown8"])
    assert d_out["It_bg"].dtype == bool and np.array_equal(d_out["It_bg"], h_out["It_bg"]) and not h_out["It_bg"].all()


def oracle_kitti(coarse, net, Is, It, It_bg, fineSize, cc_th, maskRegionTh, maxH):
    """``pair_oracle.align_pair_kitti`` (evaluation/evalKITTI/evaluation.py:216-336) with the background of :245-250 given: the
    same statements on the oracle's own helpers, ``It_bg`` in place of its ones."""
    strideNet = 8
    It_resize = PO.resize_img(It, strideNet, fineSize)
    It_d2 = PO.resize_img(It, strideNet, fineSize // 2)
    w_org, h_org = It.size
    tensor_s = PO.to_tensor(Is).unsqueeze(0)
    grid_org = WO.base_grid(h_org, w_org)
    w_r, h_r = It_resize.size
    tensor_resize, grid_resize = PO.to_tensor(It_resize).unsqueeze(0), WO.base_grid(h_r, w_r)
    w_d2, h_d2 = It_d2.size
    tensor_d2, grid_d2 = PO.to_tensor(It_d2).unsqueeze(0), WO.base_grid(h_d2, w_d2)
    coarse.setPair(Is, It)
    Mask = np.zeros((h_org, w_org), dtype=np.float32)
    Hs, D2, Msk, Fin = [], [], [], []
    nbCoarse = 0
    while nbCoarse < maxH:
        fgMask = ((Mask + (1 - It_bg)) > 0.5).astype(np.float32)
        bestPara = coarse.getCoarse(fgMask)
        if bestPara is None:
            break
        bp = torch.from_numpy(bestPara).unsqueeze(0)
        homography_d2 = WO.warp_grid(bp, h_d2, w_d2)
        homography_resize = WO.warp_grid(bp, h_r, w_r)
        IsSample_d2 = WO.grid_sample(tensor_s, homography_d2)
        _, _, flowFine_d2, _ = PO.pred_flow_mask_kitti(IsSample_d2, tensor_d2, homography_d2, grid_d2, net)
        flowCoarse, _ = WO.compose_fine(flowFine_d2, homography_resize, grid_resize, clamp=True)
        IsSample = WO.grid_sample(tensor_s, flowCoarse)
        _, matchFine_org, f8, m8 = PO.pred_flow_mask_kitti(IsSample, tensor_resize, flowCoarse, grid_org, net)
        matchFine = WO.remove_small_cc(matchFine_org, 0.99, cc_th)
        if ((matchFine > 0.9999) * (1 - fgMask)).mean() > maskRegionTh or nbCoarse == 0:
            Hs.append(bp.numpy())
            D2.append(flowFine_d2.numpy())
            Msk.append(m8.numpy())
            Fin.append(f8.numpy())
            nbCoarse += 1
            Mask = ((Mask + matchFine * (1 - fgMask)) > 0.9999).astype(np.float32)
        else:
            break
    cat = lambda l: np.concatenate(l, axis=0) if l else np.zeros((0,))
    return dict(H=cat(Hs), flow_d2=cat(D2), mask=cat(Msk), flow=cat(Fin))


@pytest.mark.parametrize("where", ["host", "device"])
def test_kitti_background_vs_oracle(rf, where):
    from ransac_flow_b200.dropin import imresize
    src, tgt, _ = synth.make_pair(41, 96, 256)
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    sky = np.zeros((96, 256), dtype=np.float32)
    sky[:30] = 1                                         # a raw skyFromSeg-like map: the sky band on top
    sky[30:40, :60] = 1
    bg = (imresize(sky, (96, 256)) < 128).astype(np.float32)
    rsd = synth.resnet50_conv4_state(0)
    oc = PO.CoarseAlignOracle(rsd, nbScale=3, nbIter=1000, tolerance=0.05, minSize=96, scaleR=1.2, variant="A", seed=1000)
    log, inner = [], oc._ransac

    def recording(m1, m2):
        r = inner(m1, m2)
        log.append(oc.last_samples)
        return r
    oc._ransac = recording
    ref = oracle_kitti(oc, oracle_net(), Is, It, bg, 96, 0.01, 0.005, 2)
    c = rf.CoarseAlignA(3, 1000, 0.05, "Homography", 96, 2, False, 1.2, True, False, resnet_state_dict=rsd, verbose=False)
    with fixed_randint(log + log[-1:]):
        out = rf.pipeline.align_pair_kitti(c, networks(rf), Is, It, fineSize=96, cc_th=0.01, maskRegionTh=0.005, maxH=2,
                                           It_bg=sky if where == "host" else torch.from_numpy(sky).cuda())
    nH = len(ref["H"])
    print("KITTI with background: %d hypothesis(es) in the oracle, %d here" % (nH, len(out["H"])))
    assert out["It_bg"].dtype == bool and np.array_equal(out["It_bg"], bg.astype(bool))
    assert nH >= 1 and len(out["H"]) == nH
    np.testing.assert_allclose(out["H"], ref["H"], atol=1e-5)
    assert np.abs(out["flow_d2"] - ref["flow_d2"]).max() < FLOW_TOL and np.abs(out["flow"] - ref["flow"]).max() < FLOW_TOL
    assert np.abs(out["mask"] - ref["mask"]).max() < FLOW_TOL
    # the background changes the first hypothesis' matches: the unmasked run draws from another match list
    with fixed_randint(log + log[-1:]):
        none = rf.pipeline.align_pair_kitti(c, networks(rf), Is, It, fineSize=96, cc_th=0.01, maskRegionTh=0.005, maxH=2)
    assert "It_bg" not in none and not np.array_equal(none["H"][0], out["H"][0])
