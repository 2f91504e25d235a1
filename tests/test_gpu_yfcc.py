"""evalYFCC's pair loop on the device (``pipeline.align_pair_yfcc``) against the CPU oracle (tests/yfcc_oracle.py), the
host-steered drop-in path (``pipeline.align_pair_yfcc_host``: the ``CoarseAlignB`` mirror plus the driver's statements)
and the mirror's own ``setTarget`` / ``getCoarse``."""
import json

import numpy as np
import PIL.Image as Image
import pytest
import torch

import geometry_ref as G
import ransac_ref as R
import yfcc_oracle as YO
from oracle import outil_oracle as OO
from oracle import synth
from test_gpu_pair import FLOW_TOL, fixed_randint, networks, oracle_net
from test_gpu_parity import tie_report
from test_gpu_ransac_exact import exact_and_certified

pytestmark = pytest.mark.gpu
PREC = {"fp32": 0, "f16x3": 2}


@pytest.fixture
def engine(request, rf):
    rf.model.set_engine(request.param)
    rf.outil.corr_precision = PREC[request.param]
    yield request.param
    rf.model.set_engine("fp32")
    rf.outil.corr_precision = 0


def coarse_b(rf, nbScale=3, nbIter=1000, minSize=96):
    return rf.CoarseAlignB(nbScale, nbIter, 0.05, "Homography", minSize, 1, True, True, True, False, 2,
                           resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False)


def inlier_grid(c, kept, mask, n):
    """The InlierMask of coarseAlignFeatMatch.py (B) :188-195 from the device path's kept target cells and inlier mask."""
    idx = kept[:n].cpu().numpy()[mask[:n].cpu().numpy().astype(bool)]
    h16, w16 = c.featt.shape[2], c.featt.shape[3]
    Wt, Ht = c.Wt.cpu().numpy(), c.Ht.cpu().numpy()
    m = np.zeros((h16, w16), dtype=np.float32)
    m[((Wt[idx] / 2 + 0.5) * h16).astype(np.int64), ((Ht[idx] / 2 + 0.5) * w16).astype(np.int64)] = 1
    return m


@pytest.mark.parametrize("engine", ["fp32", "f16x3"], indirect=True)
def test_rotated_batch_equals_separate_set_target(rf, engine):
    """The 3 + 4 image batch of ``_set_rotated_pair``: each rotated, resized target is PIL's rotate(expand=True) + LANCZOS
    bit for bit, and its features (raw and normalised) and the source's are what setSource / setTarget compute alone."""
    src, tgt, _ = synth.make_rotated_pair(3, 120, 160, 1)
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    c = coarse_b(rf)
    c._set_rotated_pair(Is, torch.from_numpy(tgt).cuda())
    ref = coarse_b(rf)
    ref.setSource(Is)
    assert np.array_equal(np.asarray(c.Is), np.asarray(ref.Is)) and torch.equal(c.IsTensor, ref.IsTensor)
    assert torch.equal(c.featsMultiScale, ref.featsMultiScale)
    assert torch.equal(c.WMultiScale, ref.WMultiScale) and torch.equal(c.HMultiScale, ref.HMultiScale)
    for k in range(4):
        c._select_target(k)
        ref.setTarget(It.rotate(90 * k, expand=True))
        assert np.array_equal(np.asarray(c.It), np.asarray(ref.It)), k
        assert c.rotated_target_size(k) == ref.It.size and c.target_size == ref.It.size
        assert torch.equal(c.ItTensor, ref.ItTensor)
        assert torch.equal(c._featt_raw.data, ref._featt_raw.data) and c._featt_raw.hw == ref._featt_raw.hw
        assert torch.equal(c.featt, ref.featt) and (c.W2, c.H2) == (ref.W2, ref.H2)
        for name in ("Wt", "Ht", "WtInt", "HtInt"):
            assert torch.equal(getattr(c, name), getattr(ref, name)), name


def test_get_coarse_device_equals_get_coarse(rf):
    """Variant B's getCoarse_device == getCoarse with the same samples, unmasked and masked: identical match lists, H bit
    for bit, identical inlier mask."""
    src, tgt, _ = synth.make_pair(8, 96, 128)
    c = coarse_b(rf)
    c.setSource(Image.fromarray(src))
    c.setTarget(Image.fromarray(tgt))
    Mt = np.zeros((96, 128), dtype=np.float32)
    Mt[:, 80:] = 1                                      # mask the right third of the target
    for mt, seed in ((None, 40), (np.zeros((96, 128), np.float32), 41), (Mt, 42), (torch.from_numpy(Mt).cuda(), 43)):
        raw = synth.draw_samples(seed, 2 ** 31 - 1, 1000)
        Hd, nb, mask, status, cnt = c.getCoarse_device(mt, raw)
        n = int(cnt.item())
        m1, m2 = c.match1[:n].cpu().numpy(), c.match2[:n].cpu().numpy()
        _, _, kept, _ = c._match_device(mt)
        assert int(status.item()) == 0 and n >= 4
        grid = inlier_grid(c, kept, mask, n)
        with fixed_randint([raw % n]):
            H, InlierMask = c.getCoarse(np.zeros((96, 128)) if mt is None else (mt.cpu().numpy() if torch.is_tensor(mt) else mt))
        assert len(c.match1) == n and np.array_equal(c.match1.cpu().numpy(), m1) and np.array_equal(c.match2.cpu().numpy(), m2)
        assert np.array_equal(H, Hd.cpu().numpy().reshape(3, 3))
        assert np.array_equal(InlierMask, grid) and int(InlierMask.sum()) == int(mask[:n].sum())
    assert InlierMask[:, 5:].sum() == 0                 # the masked cells hold no inlier


def oracle_yfcc(seed, h, w, k, nbScale, minSize, nbIter, maxCoarse, It_bg=None):
    """The oracle's run of ``make_rotated_pair(seed, h, w, k)``; ``log``: per getCoarse call, the oracle's unmasked fp32 score
    matrix and mutual pairs (index1, index2) of the current target."""
    src, tgt, _ = synth.make_rotated_pair(seed, h, w, k)
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    oc = YO.CoarseAlignYFCC(synth.resnet50_conv4_state(0), nbScale=nbScale, nbIter=nbIter, tolerance=0.05, minSize=minSize,
                            scaleR=2, seed=1000)
    log = []
    get = oc.getCoarse

    def logged(Mt):
        if len(log) < 4:                                # the rotation search: the (masked) target of each rotation
            featt = oc.featt * oc._mask16(Mt).float()[None, None]
            i1, i2, score = OO.mutualMatching(oc.featsMultiScale.numpy(), featt.contiguous().view(featt.shape[1], -1).numpy(),
                                              return_score=True)
            log.append((score, set(zip(i1.tolist(), i2.tolist()))))
            r = get(Mt)
            log[-1] += (oc.match1, oc.match2, oc.last_samples)
            return r
        return get(Mt)
    oc.getCoarse = logged
    ref = YO.align_pair_yfcc(oc, oracle_net(), Is, It, maxCoarse=maxCoarse, It_bg=It_bg)
    return Is, It, oc, ref, log


def check_rotation_matches(c, log, masks=(None,) * 4):
    """Per rotation: the device's mutual pairs are the oracle's up to PROVEN arg-max ties - a differing pair's margin in the
    oracle's fp32 scores is below twice the score deviation the engine's features cause plus the correlation's own error
    (tests/test_gpu_parity.py).  Returns, per rotation, whether the two lists are identical."""
    from ransac_flow_b200 import ops
    same = []
    for k in range(4):
        score, ref_pairs = log[k][:2]
        c._select_target(k)
        c._match_device(masks[k])
        n = int(c._count.item())
        got_pairs = set(zip(c._idx1[:n].cpu().tolist(), c._idx2[:n].cpu().tolist()))
        ft = c._featt_rows if masks[k] is None else ops.l2norm(c._featt_raw.data, c._valid16(masks[k]))    # the masked target
        dev = float((c._feats_rows.double() @ ft.double().t() - torch.from_numpy(score).cuda().double()).abs().max())
        same.append(got_pairs == ref_pairs)
        ties = tie_report(score, ref_pairs, got_pairs)
        print("rotation %d: pairs %d (oracle %d), sym-diff %d, score deviation %.3g" % (k, len(got_pairs), len(ref_pairs), len(ties), dev))
        assert dev < 2e-5
        for pair, margin in ties:
            assert margin <= 2 * dev + 1e-6, "rotation %d: pair %s differs and is not an arg-max tie (margin %.3g)" % (k, pair, margin)
    return same


@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_rotation_search_vs_oracle(rf, k):
    """Targets rotated by 0 / 90 / 180 / 270 degrees: the device's chosen angle and per-rotation scores are the oracle's
    with the oracle's samples (one table per RANSAC call, in the reference's order)."""
    Is, It, oc, ref, log = oracle_yfcc(60 + k, 96, 128, k, 3, 96, 1000, maxCoarse=0)
    c = coarse_b(rf)
    out = rf.pipeline.align_pair_yfcc(c, networks(rf), Is, torch.from_numpy(np.array(It)).cuda(), maxCoarse=0,
                                      samples=oc.all_samples)
    print("k=%d: angle %d (oracle %d), scores %s (oracle %s)" % (k, out["angle"], ref["angle"], out["nbInlierRot"], ref["nbInlierRot"]))
    assert np.array_equal(np.asarray(c.It), np.asarray(oc.It))           # the winning rotation is the current target
    check_rotation_matches(c, log)
    assert out["angle"] == ref["angle"] and out["nbInlierRot"] == ref["nbInlierRot"]
    assert len(out["H"]) == len(ref["H"]) == 1
    np.testing.assert_allclose(out["H"], ref["H"], atol=1e-5)


def test_whole_480x640_pair_vs_oracle_and_host_path(rf):
    """A 480x640 pair at the driver's defaults (nbScale 7, scaleR 2, minSize 480, coarseIter 10000, maxCoarse 10) with the
    oracle's samples: same angle, scores and number of hypotheses, H and flows within the pair tests' tolerances.  Then,
    under torch.manual_seed, the device path's own draws against the host-steered drop-in path (torch.randint on CUDA)."""
    Is, It, oc, ref, log = oracle_yfcc(70, 480, 640, 3, 7, 480, 10000, maxCoarse=10)
    net = networks(rf)
    c = coarse_b(rf, 7, 10000, 480)
    out = rf.pipeline.align_pair_yfcc(c, net, Is, It, maxCoarse=10, samples=oc.all_samples)
    nH = len(out["H"])
    print("480x640: angle %d, scores %s, %d hypotheses (oracle %d)" % (out["angle"], out["nbInlierRot"], nH, len(ref["H"])))
    check_rotation_matches(c, log)
    assert out["angle"] == ref["angle"] and out["nbInlierRot"] == ref["nbInlierRot"] and nH == len(ref["H"]) >= 1
    np.testing.assert_allclose(out["H"], ref["H"], atol=1e-5)
    assert np.abs(out["flowDown8"] - ref["flowDown8"]).max() < FLOW_TOL
    assert np.abs(out["matchDown8"] - ref["matchDown8"]).max() < FLOW_TOL
    for a, b in zip(out["flow12"], ref["flow12"]):
        assert np.abs(a.cpu().numpy() - b.numpy()).max() < FLOW_TOL
    assert out["It_bg"].shape == (480, 640) and out["It_bg"].all()

    for s in (5, 6):
        torch.manual_seed(s)
        a = rf.pipeline.align_pair_yfcc(coarse_b(rf, 7, 10000, 480), net, Is, It, maxCoarse=10)
        after_a = torch.cuda.get_rng_state()
        torch.manual_seed(s)
        b = rf.pipeline.align_pair_yfcc_host(coarse_b(rf, 7, 10000, 480), net, Is, It, maxCoarse=10)
        assert torch.equal(after_a, torch.cuda.get_rng_state()), "the device path consumed another number of generator words"
        assert a["angle"] == b["angle"] and a["nbInlierRot"] == b["nbInlierRot"] and len(a["H"]) == len(b["H"])
        assert np.array_equal(a["H"], b["H"])
        np.testing.assert_allclose(a["flowDown8"], b["flowDown8"], atol=1e-6)
        np.testing.assert_allclose(a["matchDown8"], b["matchDown8"], atol=1e-6)
        assert np.array_equal(a["It_bg"], b["It_bg"])


def sigma_ratio(m1, m2, samples, best):
    """sigma_8 / ||A||_F of the DLT matrix of unique hypothesis ``best``."""
    us = np.asarray(samples)[R.unique_rows(samples)][best:best + 1]
    return float(G.dlt_ref(m1[us], m2[us])[2][0])


def test_sky_mask_vs_oracle(rf):
    """``It_bg`` (a synthetic skyFromSeg map of the unrotated target, the sky band on top) rotated with each target,
    imresized and thresholded as the driver does: same angle, hypotheses and background map as the oracle, the masked match
    lists the oracle's up to proven ties.

    Per rotation, on the oracle's match list and samples, the RANSAC kernel returns bit for bit what the restatement
    ransac_given_H returns on the kernel's DLT, the oracle's score is the restatement on LAPACK's DLT, and every
    per-hypothesis count of both lies in certify's bounds.  A score may differ from the oracle's only through uncertified
    hypotheses.  Rotation 3 does (kernel 9, oracle 10), and the cause is a degenerate winning sample: its matches sit on
    the 16-pixel feature grid, and LAPACK's winner is a sample with sigma_8 / ||A||_F = 2.2e-17, whose null space is
    numerically two-dimensional (dlt_ref gives no bound).  The kernel's Householder DLT returns another vector of it and
    counts fewer than 10 there.  The largest certified lower bound is 9, so a score of 9 and a score of 10 are both
    admissible."""
    src, tgt, _ = synth.make_rotated_pair(81, 96, 128, 2)
    sky = np.zeros(tgt.shape[:2], dtype=np.float32)
    sky[:20] = 1
    Is, It, oc, ref, log = oracle_yfcc(81, 96, 128, 2, 3, 96, 1000, maxCoarse=3, It_bg=sky)
    c = coarse_b(rf)
    out = rf.pipeline.align_pair_yfcc(c, networks(rf), Is, It, maxCoarse=3, It_bg=sky, samples=oc.all_samples)
    print("sky: angle %d, scores %s (oracle %s), %d hypotheses (oracle %d)" % (out["angle"], out["nbInlierRot"], ref["nbInlierRot"],
                                                                              len(out["H"]), len(ref["H"])))
    assert np.array_equal(out["It_bg"], ref["It_bg"]) and not out["It_bg"].all()
    masks = [((1 - rf.pipeline.yfcc_background(sky, k, c.rotated_target_size(k))) > 0.5).astype(np.float32) for k in range(4)]
    same = check_rotation_matches(c, log, masks)

    def score(r):
        return int(r["mask"].sum()) if r["status"] == R.OK else 0
    for k in range(4):
        _, _, om1, om2, osmp = log[k]
        exp, lap, _, _ = exact_and_certified(rf, om1, om2, osmp, 0.05, "sky rotation %d" % k)
        assert score(lap) == ref["nbInlierRot"][k]                       # the oracle's score is LAPACK's restatement
        if same[k]:
            assert out["nbInlierRot"][k] == score(exp)                   # the device path's is the kernel's restatement
        if out["nbInlierRot"][k] != ref["nbInlierRot"][k]:
            assert same[k], "rotation %d: match lists differ" % k
            cert = R.certify(om1, om2, osmp, 0.05)
            lo, hi = R.outcome_bounds(cert)
            assert exp["status"] == lap["status"] == R.OK
            assert lo <= score(exp) <= hi and lo <= score(lap) <= hi
            # the higher score's winner counts less under the other DLT (whose best is lower), so it must be uncertified
            top = exp if score(exp) > score(lap) else lap
            assert cert["lo"][top["best"]] < cert["hi"][top["best"]]
            print("rotation %d: device %d, oracle %d, certified range [%d, %d]; winners %d (kernel, sigma_8 / ||A|| %.2g) "
                  "and %d (LAPACK, %.2g)" % (k, score(exp), score(lap), lo, hi, exp["best"], sigma_ratio(om1, om2, osmp, exp["best"]),
                                            lap["best"], sigma_ratio(om1, om2, osmp, lap["best"])))
    assert out["angle"] == ref["angle"] and len(out["H"]) == len(ref["H"]) >= 1
    np.testing.assert_allclose(out["H"], ref["H"], atol=1e-5)
    assert np.abs(out["flowDown8"] - ref["flowDown8"]).max() < FLOW_TOL
    assert np.abs(out["matchDown8"] - ref["matchDown8"]).max() < FLOW_TOL


def test_saved_files_read_back(rf, tmp_path):
    """save_pair + save_rotation write evalYFCC's per-scene tree; getResults' reader gives back the in-memory results."""
    src, tgt, _ = synth.make_rotated_pair(90, 96, 128, 1)
    c = coarse_b(rf)
    torch.manual_seed(3)
    out = rf.pipeline.align_pair_yfcc(c, networks(rf), Image.fromarray(src), Image.fromarray(tgt), maxCoarse=3)
    fine, coarse = tmp_path / "fine" / "scene", tmp_path / "coarse" / "scene"
    fine.mkdir(parents=True)
    coarse.mkdir(parents=True)
    nH = rf.results.save_pair(str(coarse), str(fine), 4, out, It_bg=out["It_bg"])
    rf.results.save_rotation(str(fine), {4: out["angle"]})
    assert nH == len(out["H"]) >= 1
    assert json.load(open(fine / "rotation.json"))["4"] == out["angle"]
    assert np.array_equal(np.load(fine / ("maskBG_4_%dH.npy" % nH)), out["It_bg"])
    fg, mg = rf.results.getFlow_from_files(4, str(fine), sorted(p.name for p in fine.iterdir()), str(coarse), str(fine), True, 0.95)
    fg2, mg2 = rf.pipeline.getFlow_corr(out["flowDown8"], out["H"], out["matchDown8"], th=0.95, multiH=True)
    assert torch.equal(fg, fg2) and torch.equal(mg, mg2)
