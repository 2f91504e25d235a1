"""evalYFCC's pair from CUDA graphs (``pipeline.align_pair_yfcc_graph``, ``GraphedYfccAligner``): the rotation-select and
select-copy kernels against numpy restatements, the slot chain against the eager draw-and-rewind sequence, whole pairs bit
for bit against ``align_pair_yfcc`` under ``torch.manual_seed`` (every rotation, a square target, skipped draws, every way the
loop ends, the TypeError, segNet, the driver's defaults), the oracle's samples, graph replays with eviction and lanes.
The kernel entries of ``yfcc_graph`` are assigned to these tests in tests/test_kernel_replay_inventory.py."""
import numpy as np
import PIL.Image as Image
import pytest
import torch

from oracle import synth
from test_gpu_pair import networks
from test_gpu_sky import segnet_sds

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ kernels
def numpy_select(status, counts, masks, nbPoint=4):
    """evaluation.py:195-212 after the RANSAC calls, as rotation_scores / np.argmax state it."""
    scores, drawn, err = [], 0, False
    for s, m, mk in zip(status, counts, masks):
        M = min(m, len(mk))
        drew = M >= nbPoint
        drawn += drew
        err |= drew and s == 2
        scores.append(int(np.count_nonzero(mk[:M])) if drew and s == 0 else 0)
    w = int(np.argmax(scores))
    return [w] + scores + [drawn, int(err), w & 1]


@gpu
def test_rotation_select_is_the_numpy_restatement(rf):
    rs = np.random.RandomState(0)
    cases = 0
    for trial in range(300):
        caps = rs.choice([0, 3, 4, 5, 37, 300, 2000], size=4)
        status = rs.choice([0, 0, 0, 1, 2, 3], size=4).tolist()
        counts = [int(min(c, rs.choice([0, 2, 3, 4, 5, 40, 5000]))) if trial % 3 else int(c) for c in caps]
        if trial % 5 == 0:                                 # ties: equal popcounts on several rotations
            base = (rs.rand(int(max(caps))) < 0.4).astype(np.uint8)
            masks = [base[:c].copy() for c in caps]
        else:
            masks = [(rs.rand(c) < rs.rand()).astype(np.uint8) for c in caps]
        for k in range(4):                                  # a count above the buffer is bounded by it; garbage past M ignored
            if trial % 7 == k:
                counts[k] = int(caps[k]) + 3
        d = lambda v: torch.tensor([v], dtype=torch.int32, device="cuda")
        rec = rf.yfcc_graph.rotation_select([d(s) for s in status], [d(c) for c in counts],
                                            [torch.from_numpy(m).cuda() if len(m) else torch.zeros(0, dtype=torch.uint8, device="cuda")
                                             for m in masks])
        want = numpy_select(status, counts, masks)
        assert rec.cpu().numpy().tolist() == want, (trial, status, counts, caps, want, rec)
        cases += 1
    assert cases == 300


@gpu
def test_select_copy(rf):
    srcs = [torch.full((37, 3), k, dtype=torch.uint8, device="cuda") for k in range(4)]
    for sel in range(-1, 5):
        for use in ([0, 1, 2, 3], [0, 2], [1, 3]):
            dst = torch.full((37, 3), 99, dtype=torch.uint8, device="cuda")
            rf.yfcc_graph.select_copy([srcs[k] if k in use else None for k in range(4)], torch.tensor([sel], dtype=torch.int32,
                                                                                                  device="cuda"), dst)
            want = sel if sel in use else 99
            assert (dst == want).all(), (sel, use)
    big = [torch.randn(1200, 1024, device="cuda") for _ in range(4)]
    dst = torch.empty_like(big[0])
    rf.yfcc_graph.select_copy(big, torch.tensor([2], dtype=torch.int32, device="cuda"), dst)
    assert torch.equal(dst, big[2])


@gpu
def test_slot_chain_reads_the_eager_tables(rf):
    """RANSAC calls with fewer than 4 matches at chosen positions: under one seed, the chained calls over T tables drawn up
    front return bit for bit what the eager draw-and-rewind sequence returns, and the slots count the draws."""
    rs = np.random.RandomState(3)
    M, nbIter = 120, 1000
    m1 = torch.from_numpy(np.c_[rs.rand(M, 2).astype(np.float32) * 2 - 1, np.ones(M, np.float32)]).cuda()
    H = np.array([[1.0, 0.05, 0.02], [-0.03, 0.98, 0.01], [0.0, 0.01, 1.0]])
    p = m1.cpu().numpy().astype(np.float64) @ H.T
    m2 = torch.from_numpy((p / p[:, 2:]).astype(np.float32)).cuda()
    m2[:40, :2] += torch.from_numpy(rs.rand(40, 2).astype(np.float32)).cuda()       # outliers
    counts = [120, 3, 0, 50, 4, 2, 120, 3, 7, 120, 90]
    T = len(counts)
    for seed in (1, 2):
        torch.manual_seed(seed)
        eager = []
        for m in counts:
            cnt = torch.tensor([m], dtype=torch.int32, device="cuda")
            gen = torch.cuda.default_generators[torch.cuda.current_device()]
            state = gen.get_state()
            raw = rf.ops.philox_words(nbIter, 4, "cuda")
            r = rf.ops.ransac_homography(m1, m2, raw, 0.05, 100, cnt, rf.ops.SAMPLES_PHILOX64)
            if int(r[3].item()) == 3:
                gen.set_state(state)                       # no draw: the reference returns None before torch.randint
            eager.append(r)
        after_eager = torch.cuda.get_rng_state()
        torch.manual_seed(seed)
        draws = rf.yfcc_graph.DrawnTables(nbIter, 4, T, torch.device("cuda"))
        chained = [draws.call(i).ransac(m1, m2, torch.tensor([m], dtype=torch.int32, device="cuda"), 0.05, 100) for i, m in enumerate(counts)]
        assert draws.slots.cpu().tolist() == [0] + list(np.cumsum([m >= 4 for m in counts]))
        assert draws.slots.cpu().tolist()[:-1] == rf.yfcc_graph.slot_chain(counts)
        for i, (a, b) in enumerate(zip(eager, chained)):
            assert torch.equal(a[3], b[3]), i
            if int(a[3].item()) == 0:
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), i
        ndraw = sum(m >= 4 for m in counts)
        torch.manual_seed(seed)
        for _ in range(ndraw):
            rf.ops.philox_words(nbIter, 4, "cuda")
        assert torch.equal(after_eager, torch.cuda.get_rng_state())
    # injected tables go through the same slots (SAMPLES_MOD)
    tabs = [synth.draw_samples(50 + j, 2 ** 31 - 1, nbIter) for j in range(T)]
    draws = rf.yfcc_graph.DrawnTables(nbIter, 4, T, torch.device("cuda"), samples=tabs)
    j = 0
    for i, m in enumerate(counts):
        cnt = torch.tensor([m], dtype=torch.int32, device="cuda")
        b = draws.call(i).ransac(m1, m2, cnt, 0.05, 100)
        if m >= 4:
            a = rf.ops.ransac_homography(m1, m2, torch.from_numpy(tabs[j]).cuda(), 0.05, 100, cnt, rf.ops.SAMPLES_MOD)
            assert all(torch.equal(x, y) for x, y in zip(a, b)), i
            j += 1


# ------------------------------------------------------------------ whole pairs against align_pair_yfcc
def coarse_b(rf, nbScale=3, nbIter=1000, minSize=96, tolerance=0.05, segNet=False, segId=1, segFg=True):
    return rf.CoarseAlignB(nbScale, nbIter, tolerance, "Homography", minSize, segId, segFg, True, True, segNet, 2,
                           resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False,
                           segnet_state_dicts=segnet_sds() if segNet else None)


def assert_same_pair(eager, got, tag=""):
    n = len(eager["H"])
    assert got["angle"] == eager["angle"] and got["nbInlierRot"] == eager["nbInlierRot"], (tag, got["nbInlierRot"], eager["nbInlierRot"])
    assert len(got["H"]) == n, (tag, len(got["H"]), n)
    for key in ("H", "flowDown8", "matchDown8"):
        assert got[key].dtype == eager[key].dtype and np.array_equal(got[key], eager[key]), (tag, key)
    assert list(got["nbMatch"]) == list(eager["nbMatch"]), tag
    assert got["It_bg"].dtype == bool and np.array_equal(got["It_bg"], eager["It_bg"]), tag


def graph_pair(rf, c, net, Is, It, maxCoarse, th, It_bg=None, samples=None):
    """``align_pair_yfcc_graph``'s own steps keeping the raw records: (its dict, the search record, how the loop ended)."""
    Y, P = rf.yfcc_graph, rf.pipeline
    with torch.no_grad():
        S = Y._search_device(c, P._as_device_u8(c, Is), P._as_device_u8(c, It), maxCoarse, It_bg, False, samples)
        rec = P._to_host(S["rec"]).copy()
        Y._raise_on_error(rec)
        L = Y._loop_device(c, net, S, Y.unpack_record(rec)[4], maxCoarse, th)
        host = P._to_host(L["packed"]).copy()
        bg = P._to_host(L["bg"]).copy() if L["bg"] is not None else None
    out = Y._result(rec, host.copy(), bg, L["size"], L["f8shape"], maxCoarse)
    n = len(out["H"])
    st = host.reshape(maxCoarse + 1, -1)[min(n, maxCoarse), 1]
    end = "cap" if n == maxCoarse + 1 else {0: "region", 1: "ransac", 3: "too_few"}[int(st)]
    return out, rec, end


def run_both(rf, c, net, Is, It, maxCoarse, th, seed, It_bg=None):
    torch.manual_seed(seed)
    eager = rf.pipeline.align_pair_yfcc(c, net, Is, It, maxCoarse=maxCoarse, maskRegionTh=th, It_bg=It_bg)
    torch.manual_seed(seed)
    got, rec, end = graph_pair(rf, c, net, Is, It, maxCoarse, th, It_bg)
    return eager, got, rec, end


@gpu
def test_rotations_and_loop_ends_equal_align_pair_yfcc(rf):
    """Targets rotated by 0 / 90 / 180 / 270 degrees (winners in both classes), a square target, and the loop ended by the
    region threshold (maskRegionTh 1.0 rejects every later hypothesis) and by the cap (-1 accepts all)."""
    net = networks(rf)
    seen_class, seen_end = set(), set()
    cases = [(60 + k, 96, 128, k, 3, 0.01) for k in range(4)] + [(64, 96, 96, 1, 3, 0.01), (65, 96, 96, 2, 2, 0.01),
                                                                  (61, 96, 128, 1, 3, 1.0), (62, 96, 128, 2, 2, -1.0)]
    for seed, h, w, k, maxCoarse, th in cases:
        src, tgt, _ = synth.make_rotated_pair(seed, h, w, k)
        c = coarse_b(rf)
        eager, got, rec, end = run_both(rf, c, net, Image.fromarray(src), torch.from_numpy(tgt).cuda(), maxCoarse, th, 7)
        print("seed %d %dx%d k %d: angle %d scores %s, %d hypotheses, ended by %s, class %d" % (
            seed, h, w, k, got["angle"], got["nbInlierRot"], len(got["H"]), end, rec[7]))
        assert_same_pair(eager, got, (seed, k))
        seen_class.add(int(rec[7]))
        seen_end.add(end)
    assert seen_class == {0, 1} and {"cap", "region"} <= seen_end, (seen_class, seen_end)


def keep_box(shape, s, y0, x0):
    """A skyFromSeg-like map of the unrotated target: 1 (sky) everywhere but an s x s box at (y0, x0)."""
    m = np.ones(shape, dtype=np.float32)
    m[y0:y0 + s, x0:x0 + s] = 0
    return m


def rotation_counts(rf, c, bgmap):
    counts = []
    for k in range(4):
        c._select_target(k)
        bg = rf.pipeline.yfcc_background(bgmap, k, c.rotated_target_size(k))
        counts.append(int(c._match_device(((1 - bg) > 0.5).float())[3].item()))
    return counts


def find_masks(rf, c):
    """Over pairs and keep boxes: one map under which some rotations but not all have 4 matches, and one under which none has."""
    mixed, none = None, None
    for seed, k in ((66, 1), (67, 0), (68, 2), (69, 3), (76, 1), (77, 0)):
        src, tgt, _ = synth.make_rotated_pair(seed, 96, 128, k)
        Is, It = Image.fromarray(src), torch.from_numpy(tgt).cuda()
        c._set_rotated_pair(Is, It)
        for y0, x0 in ((8, 8), (30, 40), (50, 70), (8, 60)):
            for s in range(2, 60, 2):
                bgmap = torch.from_numpy(keep_box(tgt.shape[:2], s, y0, x0)).cuda()
                counts = rotation_counts(rf, c, bgmap)
                drew = len(rf.pipeline.rotation_draws(counts))
                if drew == 0 and none is None:
                    none = (Is, It, bgmap, counts)
                if 0 < drew < 4 and mixed is None:
                    mixed = (Is, It, bgmap, counts)
                if mixed is not None and none is not None:
                    return mixed, none
    return mixed, none


@gpu
def test_skipped_draws_and_too_few_matches(rf):
    """Background maps that leave some rotations fewer than 4 matches (the eager path skips their draws, asserted from its
    counts) and one that leaves every rotation and the first hypothesis too few (the loop ends by too few matches): bit for
    bit, and the generator advances by T tables."""
    net = networks(rf)
    c = coarse_b(rf)
    mixed, none = find_masks(rf, c)
    print("masks: mixed %s, none drew %s" % (mixed and mixed[3], none and none[3]))
    assert mixed is not None and none is not None
    ends = set()
    for Is, It, bgmap, counts in (mixed, none):
        T = 4 + 3 + 1
        c._set_rotated_pair(Is, It)
        assert rotation_counts(rf, c, bgmap) == counts                # the eager path's own counts: these draws are skipped
        eager, got, rec, end = run_both(rf, c, net, Is, It, 3, 0.01, 9, It_bg=bgmap)
        after_graph = torch.cuda.get_rng_state()
        torch.manual_seed(9)
        for _ in range(T):
            rf.ops.philox_words(c.nbIter, 4, "cuda")
        assert torch.equal(after_graph, torch.cuda.get_rng_state()), "the graph path advances the generator by T tables"
        print("counts %s, drew %d, scores %s, %d hypotheses, ended by %s" % (counts, rec[5], got["nbInlierRot"], len(got["H"]), end))
        assert rec[5] == len(rf.pipeline.rotation_draws(counts)) < 4
        assert_same_pair(eager, got, counts)
        assert not got["It_bg"].all()
        ends.add(end)
    assert "too_few" in ends


@gpu
def test_no_model_raises(rf):
    """RANSAC without a model in the rotation search (tolerance 0 and fewer than 100 hypotheses: utils/outil.py:162): both
    paths raise TypeError, the graph aligner too."""
    net = networks(rf)
    src, tgt, _ = synth.make_rotated_pair(67, 96, 128, 0)
    Is, It = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
    c = coarse_b(rf, nbIter=50, tolerance=0.0)
    with pytest.raises(TypeError):
        rf.pipeline.align_pair_yfcc(c, net, Is, It, maxCoarse=2)
    with pytest.raises(TypeError):
        rf.pipeline.align_pair_yfcc_graph(c, net, Is, It, maxCoarse=2)
    ga = rf.pipeline.GraphedYfccAligner(c, net, maxCoarse=2)
    with pytest.raises(TypeError):
        ga(Is, It)


@gpu
def test_segnet_equals_align_pair_yfcc_given_its_map(rf):
    from ransac_flow_b200.segnet import SegNet
    src, tgt, _ = synth.make_rotated_pair(68, 96, 128, 1)
    t = torch.from_numpy(tgt).cuda()
    _, cls, _ = SegNet(None, None, 2, False, state_dicts=segnet_sds()).run(t, want_class=True)
    ids, counts = np.unique(cls.cpu().numpy(), return_counts=True)
    ok = [(f, int(i)) for f, i in zip(counts / counts.sum(), ids) if 0.1 <= f <= 0.9]
    assert ok
    c = coarse_b(rf, segNet=True, segId=min(ok)[1], segFg=False)
    net = networks(rf)
    Is = Image.fromarray(src)
    sky = c.segNet.run(t)[0]
    torch.manual_seed(4)
    eager = rf.pipeline.align_pair_yfcc(c, net, Is, t, maxCoarse=3, It_bg=sky)
    torch.manual_seed(4)
    got = rf.pipeline.align_pair_yfcc_graph(c, net, Is, t, maxCoarse=3, segNet=True)
    assert_same_pair(eager, got, "segNet")
    assert not got["It_bg"].all() and len(got["H"]) >= 1
    ga = rf.pipeline.GraphedYfccAligner(c, net, maxCoarse=3, segNet=True)
    ga.prepare(src, tgt)
    torch.manual_seed(4)
    assert_same_pair(eager, ga(src, tgt), "segNet graph")
    # the same map given as an input
    gb = rf.pipeline.GraphedYfccAligner(c, net, maxCoarse=3)
    gb.prepare(src, tgt, It_bg=sky)
    torch.manual_seed(4)
    assert_same_pair(eager, gb(src, tgt, It_bg=sky), "It_bg graph")


@gpu
def test_driver_defaults_480x640(rf):
    """nbScale 7, coarseIter 10000, minSize 480, maxCoarse 10: align_pair_yfcc, align_pair_yfcc_graph and a GraphedYfccAligner
    replay under one seed."""
    net = networks(rf)
    src, tgt, _ = synth.make_rotated_pair(70, 480, 640, 3)
    c = coarse_b(rf, 7, 10000, 480)
    eager, got, rec, end = run_both(rf, c, net, Image.fromarray(src), Image.fromarray(tgt), 10, 0.01, 5)
    print("480x640: angle %d scores %s, %d hypotheses, ended by %s" % (got["angle"], got["nbInlierRot"], len(got["H"]), end))
    assert_same_pair(eager, got, "480x640")
    ga = rf.pipeline.GraphedYfccAligner(coarse_b(rf, 7, 10000, 480), net, maxCoarse=10)
    r = ga.prepare(src, tgt)
    print("480x640 graphs: search %d kernels, loops %s" % (r["n_kernels"], {k: L["n_kernels"] for k, L in r["loops"].items()}))
    torch.manual_seed(5)
    assert_same_pair(eager, ga(src, tgt), "480x640 graph")


@gpu
def test_oracle_samples(rf):
    """One oracle case of tests/test_gpu_yfcc.py driven by the oracle's samples: the graph path gives what align_pair_yfcc gives."""
    from test_gpu_yfcc import oracle_yfcc
    Is, It, oc, ref, log = oracle_yfcc(61, 96, 128, 1, 3, 96, 1000, maxCoarse=2)
    net = networks(rf)
    c = coarse_b(rf)
    t = torch.from_numpy(np.array(It)).cuda()
    eager = rf.pipeline.align_pair_yfcc(c, net, Is, t, maxCoarse=2, samples=oc.all_samples)
    got = rf.pipeline.align_pair_yfcc_graph(c, net, Is, t, maxCoarse=2, samples=oc.all_samples)
    assert_same_pair(eager, got, "oracle samples")
    assert got["angle"] == ref["angle"]


# ------------------------------------------------------------------ graphs and lanes
def dev_pair(seed, h, w, k):
    return tuple(torch.from_numpy(a).cuda() for a in synth.make_rotated_pair(seed, h, w, k)[:2])


@gpu
def test_graphed_aligner_replays_and_evicts(rf):
    """Three input sizes, interleaved, with room for one record: every replay equals the eager staged call and align_pair_yfcc
    under the same seed."""
    c = coarse_b(rf)
    net = networks(rf)
    ga = rf.pipeline.GraphedYfccAligner(c, net, maxCoarse=2, max_graphs=1)
    P = [dev_pair(71, 96, 128, 1), dev_pair(72, 96, 96, 2), dev_pair(73, 120, 160, 3)]
    for i, (s, t) in enumerate([P[0], P[1], P[0], P[2], P[2], P[1]]):
        rec = ga.prepare(s, t)
        assert len(ga.graphs) == 1 and rec["n_kernels"] > 0 and len(rec["loops"]) == (1 if s.shape[1] == t.shape[1] == 96 else 2)
        torch.manual_seed(30 + i)
        got = ga(s, t)
        torch.manual_seed(30 + i)
        staged = rf.pipeline.align_pair_yfcc_graph(c, net, s, t, maxCoarse=2)
        torch.manual_seed(30 + i)
        eager = rf.pipeline.align_pair_yfcc(c, net, s, t, maxCoarse=2)
        assert_same_pair(staged, got, i)
        assert_same_pair(eager, got, i)
    print("YFCC graphs: search %d kernels, loops %s" % (rec["n_kernels"], {k: L["n_kernels"] for k, L in rec["loops"].items()}))


@gpu
def test_concurrent_lanes_do_not_depend_on_interleaving(rf):
    ca = rf.pipeline.ConcurrentAligner(lambda: (coarse_b(rf), networks(rf)), lanes=2, seed=3,
                                       make_aligner=lambda c, n: rf.pipeline.GraphedYfccAligner(c, n, maxCoarse=2))
    P = [dev_pair(74, 96, 128, 1), dev_pair(75, 96, 128, 0)]
    pairs = [P[0], P[1], P[1], P[0]]
    ca.prepare(*P[0])
    ca.prepare(*P[1])                                     # a capture's warm-up draws from the lane's generator: none inside run
    ca.seed(3)
    together = ca.run(pairs)
    ca.seed(3)
    for k in range(2):
        for i in range(k, len(pairs), 2):
            alone = ca.lanes[k](*pairs[i])
            assert_same_pair(alone, together[i], (k, i))
            assert len(alone["H"]) >= 1
