"""evalKITTI's pair with no host control (``pipeline.align_pair_kitti_graph``, ``GraphedKittiAligner``): the fused acceptance / mask
step ``ops.kitti_region_step`` bit for bit against a numpy restatement of evaluation/evalKITTI/evaluation.py:316-326, the device
pair against the host-steered ``align_pair_kitti`` for every way the loop ends, the cached target features, graph replays with
eviction, and ``ConcurrentAligner`` lanes."""
import numpy as np
import PIL.Image as Image
import pytest
import torch

from oracle import synth
from test_gpu_pair import networks
from test_gpu_sky import segnet_sds

pytestmark = pytest.mark.gpu

TH = 0.9999


# ------------------------------------------------------------------ ops.kitti_region_step
def numpy_step(match, Mask, bg, fgMask, status, alive, first, maskRegionTh):
    """evaluation.py:316-326 for one hypothesis, as the reference's numpy statements, plus the gate of a dead flag."""
    count = int(np.count_nonzero((match > TH) & (fgMask == 0)))
    ok = status == 0 and (first or bool(((match > TH) * (1 - fgMask)).mean() > maskRegionTh))
    alive = bool(alive) and ok
    if alive:
        matchFine = match * (1 - fgMask)
        Mask = ((Mask + matchFine) > TH).astype(np.float32)
        fgMask = ((Mask + (1 - bg)) > 0.5).astype(np.float32)
    return Mask, fgMask, alive, count


def near_threshold(rs, n):
    """Matchabilities on both sides of 0.9999f and 1 - 0.9999f (Mask + match rounds there), a few negatives and 0 / 1."""
    t = np.float32(TH)
    specials = np.array([t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(2)), 1.0, 0.0, np.float32(1e-4),
                         np.float32(-1e-4), np.nextafter(np.float32(1e-4), np.float32(0)), np.nextafter(np.float32(-1e-4), np.float32(0)),
                         np.float32(0.99), np.float32(0.5)], dtype=np.float32)
    v = rs.rand(n).astype(np.float32) * np.float32(0.9999)
    pick = rs.rand(n) < 0.3
    v[pick] = specials[rs.randint(0, len(specials), int(pick.sum()))]
    return v


def step_case(rs, H, W, count, nan=False):
    """Maps with exactly ``count`` pixels where match > 0.9999 and fgMask == 0 (capped at the number of free pixels)."""
    n = H * W
    bg = (rs.rand(n) > 0.15).astype(np.float32)
    Mask = (rs.rand(n) < 0.3).astype(np.float32)
    fg = ((Mask + (1 - bg)) > 0.5).astype(np.float32)
    match = near_threshold(rs, n)
    free = np.flatnonzero(fg == 0)
    match[free] = np.minimum(match[free], np.float32(TH))                      # nothing counted yet
    on = rs.choice(free, min(count, len(free)), replace=False)
    match[on] = np.where(rs.rand(len(on)) < 0.5, np.float32(1.0), np.nextafter(np.float32(TH), np.float32(2)))
    busy = np.flatnonzero(fg == 1)
    if len(busy):
        match[busy[: len(busy) // 2]] = 1.0                                   # matched, but under the mask: not counted
    if nan:
        match[rs.rand(n) < 0.05] = np.nan
    return [a.reshape(H, W) for a in (match, Mask, bg, fg)]


def run_step(rf, match, Mask, bg, fg, status, alive, first, cmin):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dm, dM, db, df = d(match), d(Mask), d(bg), d(fg)
    st = torch.tensor([status], dtype=torch.int32, device="cuda")
    al = torch.tensor([int(alive)], dtype=torch.int32, device="cuda")
    rec = rf.ops.kitti_region_step(dm, dM, db, df, st, al, first, cmin)
    return dM.cpu().numpy(), df.cpu().numpy(), int(al.item()), rec.cpu().numpy()


@pytest.mark.parametrize("H,W", [(376, 1241), (1, 1), (5, 7), (33, 257), (1000, 3)])
@pytest.mark.parametrize("th", [0.005, 0.01])
def test_region_step_is_the_numpy_loop(rf, H, W, th):
    rs = np.random.RandomState(H * 7 + W)
    n = H * W
    cmin = rf.pipeline.kitti_region_cmin(n, th)
    cases = 0
    for count in sorted({max(0, cmin - 1), cmin, cmin + 1, 0}):
        for status, alive, first, nan in ((0, 1, False, False), (0, 1, True, False), (1, 1, False, False), (3, 1, True, True),
                                          (2, 1, True, False), (0, 0, False, False), (0, 0, True, False), (0, 1, False, True)):
            match, Mask, bg, fg = step_case(rs, H, W, count, nan)
            want = numpy_step(match, Mask, bg, fg, status, alive, first, th)
            gM, gf, ga, rec = run_step(rf, match, Mask, bg, fg, status, alive, first, cmin)
            tag = (count, status, alive, first, nan)
            assert np.array_equal(gM, want[0]) and gM.dtype == np.float32, tag
            assert np.array_equal(gf, want[1]), tag
            assert ga == int(want[2]) and rec[0] == ga and rec[1] == want[3], (tag, ga, rec, want[2:])
            if not want[2]:
                assert np.array_equal(gM, Mask) and np.array_equal(gf, fg), tag        # a dead hypothesis touches nothing
            cases += 1
    assert cases >= 16


def test_region_step_counts_at_the_threshold(rf):
    """376 x 1241: cmin - 1 new pixels are rejected, cmin accepted, and the maps follow the verdict."""
    H, W, th = 376, 1241, 0.005
    cmin = rf.pipeline.kitti_region_cmin(H * W, th)
    rs = np.random.RandomState(9)
    seen = set()
    for count in (cmin - 1, cmin, cmin + 1):
        match, Mask, bg, fg = step_case(rs, H, W, count)
        assert int(np.count_nonzero((match > TH) & (fg == 0))) == count
        want = numpy_step(match, Mask, bg, fg, 0, 1, False, th)
        gM, gf, ga, rec = run_step(rf, match, Mask, bg, fg, 0, 1, False, cmin)
        assert ga == int(want[2]) == int(count >= cmin) and rec[1] == count
        assert np.array_equal(gM, want[0]) and np.array_equal(gf, want[1])
        seen.add(ga)
    assert seen == {0, 1}


def test_region_step_in_a_graph(rf):
    """Captured once, replayed over changing maps and flags: the same bits as the eager call on fresh buffers."""
    H, W, th = 61, 97, 0.01
    cmin = rf.pipeline.kitti_region_cmin(H * W, th)
    z = lambda: torch.zeros((H, W), device="cuda")
    sm, sM, sb, sf = z(), z(), z(), z()
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    al = torch.ones(1, dtype=torch.int32, device="cuda")
    rec = torch.zeros(2, dtype=torch.int32, device="cuda")
    rf.ops.kitti_region_step(sm, sM, sb, sf, st, al, False, cmin, rec)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        rf.ops.kitti_region_step(sm, sM, sb, sf, st, al, False, cmin, rec)
    rs = np.random.RandomState(2)
    for count, status, alive in ((cmin, 0, 1), (cmin - 1, 0, 1), (cmin + 5, 1, 1), (cmin + 5, 0, 0), (cmin + 9, 0, 1)):
        match, Mask, bg, fg = step_case(rs, H, W, count)
        for dst, src in ((sm, match), (sM, Mask), (sb, bg), (sf, fg)):
            dst.copy_(torch.from_numpy(src))
        st.fill_(status)
        al.fill_(alive)
        g.replay()
        torch.cuda.synchronize()
        want = run_step(rf, match, Mask, bg, fg, status, alive, False, cmin)
        assert np.array_equal(sM.cpu().numpy(), want[0]) and np.array_equal(sf.cpu().numpy(), want[1])
        assert int(al.item()) == want[2] and np.array_equal(rec.cpu().numpy(), want[3])


# ------------------------------------------------------------------ the pair against align_pair_kitti
def coarse(rf, minSize=96, segNet=False, segId=2, tolerance=0.05):
    return rf.CoarseAlignA(3, 1000, tolerance, "Homography", minSize, segId, False, 1.2, True, segNet, resnet_state_dict=synth.resnet50_conv4_state(0),
                           verbose=False, segnet_state_dicts=segnet_sds() if segNet else None)


def flat_target(h, w):
    return np.full((h, w, 3), 128, dtype=np.uint8)


def assert_same_pair(eager, dev, size):
    n = len(eager["H"])
    assert len(dev["H"]) == n and len(dev["maps"]) == n and dev["size"] == size == eager["size"]
    for key in ("H", "flow_d2", "mask", "flow"):
        assert dev[key].dtype == eager[key].dtype and np.array_equal(dev[key], eager[key]), key
    for (fe, me), (fd, md) in zip(eager["maps"], dev["maps"]):
        assert torch.equal(fe, fd) and np.array_equal(me, md.cpu().numpy())
    assert len(dev["nbMatch"]) == len(dev["nbInlier"]) == n and all(m >= i for m, i in zip(dev["nbMatch"], dev["nbInlier"]))


def device_pair(rf, c, net, src, tgt, fineSize, th, maxH):
    """``align_pair_kitti_graph``'s own steps, keeping the raw records: (its dict, how the loop ended)."""
    P = rf.pipeline
    packed, maps, size, shapes, _ = P._kitti_device(c, net, torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), fineSize, 0.01, th, maxH)
    host = P._to_host(packed).copy()
    out = P._unpack_kitti(host.copy(), maps, size, shapes, maxH)
    n = len(out["H"])
    end = "cap" if n == maxH else ("region" if host.reshape(maxH, -1)[n, 1] == 0 else "ransac")
    return out, end


# (pair seed, h, w, fineSize, maskRegionTh, maxH, kind).  The region threshold ends the pairs at 0.005 - 0.2 (the untextured
# target too: its border features still give RANSAC a model), the cap the ones that accept everything (maskRegionTh = -1), and a
# failed RANSAC the model whose tolerance admits no inlier (the reference's `nbInlier[best] == 0: return None`)
PAIRS = [(41, 96, 256, 96, 0.005, 5, "pair"), (7, 120, 160, 64, 0.005, 5, "pair"), (13, 96, 256, 96, 0.05, 5, "pair"),
         (42, 96, 256, 96, 0.2, 4, "pair"), (41, 96, 256, 96, -1.0, 1, "pair"), (41, 96, 256, 96, -1.0, 2, "pair"),
         (7, 120, 160, 64, -1.0, 6, "pair"), (3, 96, 256, 96, 0.005, 4, "flat"), (41, 96, 256, 96, 0.005, 3, "no inlier")]


def test_graph_pair_is_align_pair_kitti(rf):
    """Small KITTI-shaped pairs: the same hypotheses as the host-steered loop, bit for bit, and every way the loop ends."""
    net = networks(rf)
    seen = set()
    for seed, h, w, fineSize, th, maxH, kind in PAIRS:
        src, tgt, _ = synth.make_pair(seed, h, w)
        if kind == "flat":
            tgt = flat_target(h, w)
        c = coarse(rf, tolerance=0.0 if kind == "no inlier" else 0.05)
        torch.manual_seed(11)
        try:
            eager = rf.pipeline.align_pair_kitti(c, net, Image.fromarray(src), Image.fromarray(tgt), fineSize=fineSize, cc_th=0.01,
                                                 maskRegionTh=th, maxH=maxH)
        except TypeError:                               # RANSAC without a model (utils/outil.py:162): the device path raises too
            torch.manual_seed(11)
            with pytest.raises(TypeError):
                device_pair(rf, c, net, src, tgt, fineSize, th, maxH)
            seen.add("raise")
            continue
        torch.manual_seed(11)
        dev, end = device_pair(rf, c, net, src, tgt, fineSize, th, maxH)
        n = len(eager["H"])
        print("KITTI %s seed %d maskRegionTh %g maxH %d: %d hypothesis(es), ended by %s, nbMatch %s" % (kind, seed, th, maxH, n, end, dev["nbMatch"]))
        assert_same_pair(eager, dev, (h, w))
        assert dev["capped"] == (end == "cap")
        seen.add(end)
    assert {"cap", "region", "ransac"} <= seen, seen


def test_graph_pair_is_align_pair_kitti_full_size(rf):
    """376 x 1241 at the driver's fineSize 650 (both fine levels at their real sizes), through the public entry point."""
    src, tgt, _ = synth.make_pair(2, 376, 1241)
    c = coarse(rf, 400)
    net = networks(rf)
    torch.manual_seed(11)
    eager = rf.pipeline.align_pair_kitti(c, net, Image.fromarray(src), Image.fromarray(tgt), maxH=5)
    torch.manual_seed(11)
    dev = rf.pipeline.align_pair_kitti_graph(c, net, torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), maxH=5)
    print("KITTI 376x1241: %d hypothesis(es), capped %s" % (len(eager["H"]), dev["capped"]))
    assert len(eager["H"]) >= 1
    assert_same_pair(eager, dev, (376, 1241))
    assert dev["capped"] == (len(eager["H"]) == 5)


def test_graph_pair_with_segnet(rf):
    """``segNet=True``: segNet's map of the target, byte-scaled to the original size, masks every hypothesis; the pair equals
    ``align_pair_kitti`` given that map, and ``It_bg`` matches."""
    from ransac_flow_b200.segnet import SegNet
    src, tgt, _ = synth.make_pair(41, 96, 256)
    t = torch.from_numpy(tgt).cuda()
    _, cls, _ = SegNet(None, None, 2, False, state_dicts=segnet_sds()).run(t, want_class=True)
    ids, counts = np.unique(cls.cpu().numpy(), return_counts=True)
    ok = [(f, int(i)) for f, i in zip(counts / counts.sum(), ids) if 0.1 <= f <= 0.9]
    assert ok
    c = coarse(rf, segNet=True, segId=min(ok)[1])
    net = networks(rf)
    sky = c.segNet.run(t)[0]
    torch.manual_seed(4)
    eager = rf.pipeline.align_pair_kitti(c, net, Image.fromarray(src), Image.fromarray(tgt), fineSize=96, maskRegionTh=0.005, maxH=4, It_bg=sky)
    torch.manual_seed(4)
    dev = rf.pipeline.align_pair_kitti_graph(c, net, src, tgt, fineSize=96, maskRegionTh=0.005, maxH=4, segNet=True)
    torch.manual_seed(4)
    plain = rf.pipeline.align_pair_kitti_graph(c, net, src, tgt, fineSize=96, maskRegionTh=0.005, maxH=4)
    assert len(eager["H"]) >= 1
    assert_same_pair(eager, dev, (96, 256))
    assert dev["It_bg"].dtype == bool and np.array_equal(dev["It_bg"], eager["It_bg"]) and not dev["It_bg"].all()
    assert "It_bg" not in plain and not np.array_equal(plain["H"][0], dev["H"][0]), "the background does not change the first hypothesis"


@pytest.mark.parametrize("engine", ["fp32", "f16x3"])
def test_cached_target_features_are_the_batched_ones(rf, engine):
    """Both fine levels of a 376 x 1241 pair: the target's features computed in the first hypothesis' two-image batch equal
    the per-hypothesis batch's bit for bit, and so does everything PredFlowMask_kitti_device derives from them."""
    rf.model.set_engine(engine)
    try:
        net = networks(rf)
        src, tgt, _ = synth.make_pair(2, 376, 1241)
        c = coarse(rf, 400)
        s, t = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
        tensor_s = c._to_tensor01(s)
        for fineSize in (650, 325):
            w, h = rf.pipeline.fine_sizes(1241, 376, 8, fineSize)
            It = c._to_tensor01(rf.ops.resize_lanczos_u8(t, w, h))
            box = {}
            outs = []
            for k, Hm in enumerate(([[1.0, 0.02, 0.01], [0.0, 1.0, -0.03], [0.0, 0.0, 1.0]], [[0.97, 0.0, 0.05], [0.01, 1.02, 0.0], [0.0, 0.001, 1.0]])):
                grid = rf.ops.warp_grid(torch.tensor(Hm, device="cuda").view(1, 3, 3), h, w)
                IsSample = rf.ops.grid_sample(tensor_s, grid)
                batched = rf.pipeline.PredFlowMask_kitti_device(IsSample, It, grid, (h, w), net)
                cached = rf.pipeline.PredFlowMask_kitti_device(IsSample, It, grid, (h, w), net, featt=box.get("featt"), feat_box=box)
                f = rf.pipeline.fine_features(net["netFeatCoarse"], torch.cat([IsSample, It], dim=0))
                half = f.data.shape[0] // 2
                assert torch.equal(box["featt"].data, f.data[half:]), (fineSize, k)
                for a, b in zip(batched, cached):
                    assert torch.equal(a, b), (fineSize, k)
                outs.append(cached)
            assert not torch.equal(outs[0][0], outs[1][0])
    finally:
        rf.model.set_engine("fp32")


# ------------------------------------------------------------------ graphs and lanes
def test_graphed_aligner_replays_and_evicts(rf):
    """Two input sizes, interleaved, with room for one graph: every replay equals the eager device pair under the same seed."""
    c = coarse(rf)
    net = networks(rf)
    ga = rf.pipeline.GraphedKittiAligner(c, net, fineSize=96, maskRegionTh=0.005, maxH=3, max_graphs=1)
    P = [tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(41, 96, 256)[:2]),
         tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(7, 120, 160)[:2])]
    for i, (s, t) in enumerate([P[0], P[1], P[0], P[0], P[1]]):
        rec = ga.prepare(s, t)
        assert len(ga.graphs) == 1 and rec["n_kernels"] > 0
        torch.manual_seed(20 + i)
        got = ga(s, t)
        torch.manual_seed(20 + i)
        want = rf.pipeline.align_pair_kitti_graph(c, net, s, t, fineSize=96, maskRegionTh=0.005, maxH=3)
        assert len(got["H"]) == len(want["H"]) >= 1 and got["capped"] == want["capped"], i
        for key in ("H", "flow_d2", "mask", "flow"):
            assert np.array_equal(got[key], want[key]), (i, key)
        assert got["nbMatch"] == want["nbMatch"] and got["nbInlier"] == want["nbInlier"]
        for (fg, mg), (fw, mw) in zip(got["maps"], want["maps"]):
            assert torch.equal(fg, fw) and torch.equal(mg, mw)
        live = ga.fetch(ga.enqueue(s, t), copy=False)["maps"]
        assert all(f.data_ptr() == rec["flow12"][k][0].data_ptr() for k, (f, _) in enumerate(live))
    print("KITTI graph: %d kernels per pair" % rec["n_kernels"])


def test_concurrent_lanes_do_not_depend_on_interleaving(rf):
    ca = rf.pipeline.ConcurrentAligner(lambda: (coarse(rf), networks(rf)), lanes=2, seed=3,
                                       make_aligner=lambda c, n: rf.pipeline.GraphedKittiAligner(c, n, fineSize=96, maxH=3))
    P = [tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(41, 96, 256)[:2]),
         tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(42, 96, 256)[:2])]
    pairs = [P[0], P[1], P[1], P[0]]
    ca.prepare(*P[0])
    ca.seed(3)
    together = ca.run(pairs)
    ca.seed(3)
    for k in range(2):
        for i in range(k, len(pairs), 2):
            alone = ca.lanes[k](*pairs[i])
            for key in ("H", "flow_d2", "mask", "flow"):
                assert np.array_equal(alone[key], together[i][key]), (k, i, key)
            assert alone["nbMatch"] == together[i]["nbMatch"] and len(alone["H"]) >= 1
            for (fa, ma), (ft, mt) in zip(alone["maps"], together[i]["maps"]):
                assert torch.equal(fa, ft) and torch.equal(ma, mt)
