"""evalYFCC's pair loop on the CPU: the oracle against the unmodified reference's golden run (tests/yfcc_oracle.py), the
rotation.json format getResults.py reads, and the rotation search's draw schedule and scores."""
import json

import numpy as np
import PIL.Image as Image
import pytest
import torch

import yfcc_oracle as YO
from conftest import golden
from oracle import synth


def oracle_net():
    return {"netFeatCoarse": synth.feature_extractor_state(0), "netFlowCoarse": synth.net_flow_coarse_state(1),
            "netMatch": synth.net_matchability_state(2)}


def test_oracle_reproduces_reference_rotation_search_and_hypotheses():
    g = golden("yfcc_rotation_search")
    a = YO.GOLDEN_ARGS
    oc = YO.CoarseAlignYFCC(synth.resnet50_conv4_state(0), inject=list(g["samples"]), nbScale=a["nbScale"], nbIter=a["nbIter"],
                            tolerance=0.05, minSize=a["minSize"], scaleR=a["scaleR"])
    out = YO.align_pair_yfcc(oc, oracle_net(), Image.fromarray(g["src"]), Image.fromarray(g["tgt"]), maxCoarse=a["maxCoarse"])
    assert len(oc.all_samples) == len(g["samples"]) and not oc.inject          # one table per RANSAC call, in the same order
    assert out["angle"] == int(g["angle"]) and out["nbInlierRot"] == g["nbInlierRot"].tolist()
    assert np.array_equal(np.asarray(oc.It), g["It"])
    np.testing.assert_allclose(out["Hrot"], g["Hrot"], atol=1e-5)
    assert out["H"].shape == g["H"].shape
    np.testing.assert_allclose(out["H"], g["H"], atol=1e-5)
    np.testing.assert_allclose(out["flowDown8"], g["flowDown8"], atol=1e-6)
    np.testing.assert_allclose(out["matchDown8"], g["matchDown8"], atol=1e-6)


def test_golden_fixture_bites():
    """The golden run exercises the tie rule (two rotations with the same score: the first wins) and several hypotheses."""
    g = golden("yfcc_rotation_search")
    s = g["nbInlierRot"]
    assert int(np.argmax(s)) * 90 == int(g["angle"]) and (s == s.max()).sum() >= 2
    assert len(g["H"]) >= 2 and len(g["samples"]) >= int(g["calls_rot"].sum()) + len(g["H"])


def test_save_rotation_round_trips_as_get_results_reads_it(rf, tmp_path):
    angles = {0: 90, 1: 0, 7: 270, 12: 180}
    path = rf.results.save_rotation(str(tmp_path), angles)
    assert path == str(tmp_path / "rotation.json")
    with open(path, "r") as f:                           # evalYFCC/getResults.py:255-257
        rotation = json.load(f)
    assert all(rotation[str(i)] == a for i, a in angles.items()) and len(rotation) == len(angles)
    assert json.loads(open(path).read()) == {str(k): v for k, v in angles.items()}


@pytest.mark.parametrize("counts,expect", [([3, 50, 0, 7], [1, 3]), ([4, 4, 4, 4], [0, 1, 2, 3]), ([0, 1, 2, 3], []),
                                           ([100, 3, 3, 9], [0, 3])])
def test_draw_schedule_consumes_nothing_for_rotations_with_too_few_matches(rf, counts, expect):
    """The reference draws torch.randint(M, (nbIter, 4)) inside RANSAC only, after getCoarse's ``len(match1) < 4`` return:
    a seeded generator must end where the reference's sequence of draws leaves it."""
    assert rf.pipeline.rotation_draws(counts) == expect
    nbIter = 50
    ref, ours = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    ref_tables = []
    for M in counts:                                     # evaluation.py:198-206 with coarseAlignFeatMatch.py (B) :179-183
        if M >= 4:
            ref_tables.append(torch.randint(M, (nbIter, 4), generator=ref))
    our_tables = [torch.randint(counts[k], (nbIter, 4), generator=ours) for k in rf.pipeline.rotation_draws(counts)]
    assert len(ref_tables) == len(our_tables) and all(torch.equal(a, b) for a, b in zip(ref_tables, our_tables))
    assert torch.equal(ref.get_state(), ours.get_state())


def test_rotation_scores(rf):
    # RANSAC ran on rotations 1 and 3; 1 returned None (status 1): scores 0, the first maximum wins
    s = rf.pipeline.rotation_scores([1, 3], np.array([1, 0]), np.array([17, 12]))
    assert s == [0, 0, 0, 12] and int(np.argmax(s)) == 3
    s = rf.pipeline.rotation_scores([0, 1, 2, 3], np.zeros(4), np.array([5, 9, 9, 2]))
    assert int(np.argmax(s)) == 1
    with pytest.raises(TypeError):                      # RF_RANSAC_NO_MODEL: utils/outil.py:162
        rf.pipeline.rotation_scores([2], np.array([2]), np.array([0]))


def test_yfcc_background_is_the_drivers_imresize(rf):
    """pipeline.yfcc_background (dropin.imresize) == the oracle's restatement of :193 / :212, with and without a sky map."""
    rs = np.random.RandomState(4)
    sky = (rs.rand(37, 53) > 0.7).astype(np.float32)
    for k in range(4):
        size = (64, 48) if k % 2 == 0 else (48, 64)
        assert np.array_equal(rf.pipeline.yfcc_background(sky, k, size), YO.background(sky, k, size))
        assert np.array_equal(rf.pipeline.yfcc_background(None, k, size), YO.background(np.ones((37, 53), np.float32), k, size))
    assert rf.pipeline.yfcc_background(None, 0, (64, 48)).all()


def test_make_rotated_pair():
    for k in range(4):
        s, t, H = synth.make_rotated_pair(2, 24, 40, k)
        s0, t0, H0 = synth.make_pair(2, 24, 40)
        assert np.array_equal(s, s0) and np.array_equal(H, H0) and t.flags["C_CONTIGUOUS"]
        assert np.array_equal(np.asarray(Image.fromarray(t0).rotate(90 * k, expand=True)), t)
