"""RANSAC kernel vs the oracle and the reference's golden vectors (bit-exact inlier masks)."""
import numpy as np
import pytest
import torch

import geometry_ref as G
from conftest import golden
from oracle import outil_oracle as OO
from oracle import synth

pytestmark = pytest.mark.gpu
CASES = ["ransac_m120", "ransac_m636", "ransac_grid", "ransac_remainder_only", "ransac_none", "ransac_lowinlier"]


def run_kernel(rf, m1, m2, samples, tol, M_dev=None):
    H, nb, mask, st = rf.ops.ransac_homography(torch.from_numpy(m1).cuda(), torch.from_numpy(m2).cuda(),
                                               torch.from_numpy(samples).cuda(), tol, 100, M_dev)
    torch.cuda.synchronize()
    return H.cpu().numpy().reshape(3, 3), int(nb.item()), mask.cpu().numpy().astype(bool), int(st.item())


@pytest.mark.parametrize("name", CASES)
def test_golden_cases(rf, name):
    g = golden(name)
    H, nb, mask, st = run_kernel(rf, g["match1"], g["match2"], g["samples"], float(g["tol"]))
    if bool(g["is_none"]):
        assert st == 1
        return
    assert st == 0
    assert nb == int(g["nbInlier"])
    assert np.array_equal(mask, g["isInlier"])                     # bit-exact mask vs the reference
    np.testing.assert_allclose(H, g["H"], rtol=0, atol=2e-7)       # Householder DLT vs LAPACK dgesdd
    # per-hypothesis: chunk-0 homographies and reprojection errors
    us = OO.unique_samples(g["samples"])[: len(g["chunk0_H"])]
    Hd = rf.ops.homography_dlt(torch.from_numpy(g["match1"][us]).cuda(), torch.from_numpy(g["match2"][us]).cuda()).cpu().numpy()
    G.dlt_check(Hd.reshape(len(us), 9), g["match1"][us], g["match2"][us])     # sign included wherever the bound is below 1
    err = rf.ops.prediction(torch.from_numpy(g["match1"]).cuda(), torch.from_numpy(g["match2"]).cuda(),
                            torch.from_numpy(g["chunk0_H"][:8]).cuda()).cpu().numpy()
    assert np.array_equal(err, OO.Prediction(g["match1"], g["match2"], g["chunk0_H"][:8]))   # same fp32 op order


@pytest.mark.parametrize("seed,M,nbIter,frac", [(101, 636, 1000, 0.6), (102, 256, 1000, 0.6), (103, 1200, 1000, 0.6),
                                                (104, 50, 1000, 0.5), (105, 636, 50000, 0.6), (106, 4, 200, 1.0),
                                                (107, 300, 99, 0.6), (108, 300, 100, 0.6), (109, 300, 101, 0.6),
                                                (110, 636, 4097, 0.3)])
def test_seeded_vs_oracle(rf, seed, M, nbIter, frac):
    m1, m2, _ = synth.make_matches(seed, M, frac, grid=(30, 40) if seed % 2 else None)
    samples = synth.draw_samples(seed, M, nbIter)
    try:
        Ho, nbo, inlo, _ = OO.RANSAC_from_samples(m1, m2, samples, 0.05)
        expect = 0 if Ho is not None else 1
    except TypeError:
        expect = 2
    H, nb, mask, st = run_kernel(rf, m1, m2, samples, 0.05)
    assert st == expect
    if expect == 0:
        assert nb == int(nbo)
        assert np.array_equal(mask, inlo)
        np.testing.assert_allclose(H, Ho, rtol=0, atol=2e-7)


def test_status_none_and_no_model(rf):
    m1, m2, _ = synth.make_matches(3, 40, 0.0)
    H, nb, mask, st = run_kernel(rf, m1, m2, synth.draw_samples(3, 40, 50), 0.0)      # remainder only, nothing scores
    assert st == 2 and nb == 0 and not mask.any()
    H, nb, mask, st = run_kernel(rf, m1, m2, synth.draw_samples(3, 40, 400), 0.0)     # a full zero chunk
    assert st == 1
    # the Python mirror turns these into the reference's behaviours
    t1, t2 = torch.from_numpy(m1).cuda(), torch.from_numpy(m2).cuda()
    assert rf.outil.RANSAC(400, t1, t2, 0.0, 4, rf.outil.Homography) == (None, 0, [], [])
    with pytest.raises(TypeError):
        rf.outil.RANSAC(50, t1, t2, 0.0, 4, rf.outil.Homography)


def test_device_side_match_count(rf):
    """M_dev: matches beyond the device count are ignored and samples are taken modulo the count."""
    m1, m2, _ = synth.make_matches(7, 400, 0.6)
    Mtrue = 300
    raw = synth.draw_samples(7, 2 ** 31 - 1, 1000)
    Ho, nbo, inlo, _ = OO.RANSAC_from_samples(m1[:Mtrue], m2[:Mtrue], raw % Mtrue, 0.05)
    Md = torch.tensor([Mtrue], dtype=torch.int32).cuda()
    H, nb, mask, st = run_kernel(rf, m1, m2, raw, 0.05, Md)
    assert st == 0 and nb == int(nbo)
    assert np.array_equal(mask[:Mtrue], inlo) and not mask[Mtrue:].any()


def test_mirror_api_matches_reference_types(rf):
    g = golden("ransac_m636")
    real = torch.randint
    torch.randint = lambda high, size, **k: torch.from_numpy(g["samples"]).cuda()
    try:
        H, nb, inl, m2in = rf.outil.RANSAC(1000, torch.from_numpy(g["match1"]).cuda(), torch.from_numpy(g["match2"]).cuda(),
                                           0.05, 4, rf.outil.Homography)
    finally:
        torch.randint = real
    assert H.dtype == np.float32 and H.shape == (3, 3) and inl.dtype == bool and int(nb) == int(g["nbInlier"])
    assert np.array_equal(inl, g["isInlier"]) and np.array_equal(m2in, g["match2"][g["isInlier"]])
    # ScoreRANSAC / Homography / Prediction mirrors
    us = torch.from_numpy(OO.unique_samples(g["samples"])[:100]).cuda()
    H21, cnt = rf.outil.ScoreRANSAC(torch.from_numpy(g["match1"]).cuda(), torch.from_numpy(g["match2"]).cuda(), 0.05, us, rf.outil.Homography)
    assert np.array_equal(cnt.cpu().numpy(), g["chunk0_counts"])


def test_fuzz_many_seeds_bit_exact(rf):
    """40 random configurations (M 4..1500, nbIter 1..3000, inlier fraction 0..1, grid / continuous coordinates,
    tolerance 0.005..0.1): status, inlier count and inlier mask bit-exact against the oracle, H within 2e-7."""
    rs = np.random.RandomState(2024)
    n_ok = n_none = n_nomodel = 0
    for case in range(40):
        M = int(rs.choice([4, 5, 8, 37, 100, 333, 636, 1200, 1500]))
        nbIter = int(rs.choice([1, 7, 99, 100, 101, 250, 1000, 3000]))
        frac = float(rs.choice([0.0, 0.1, 0.3, 0.6, 0.9, 1.0]))
        tol = float(rs.choice([0.005, 0.02, 0.05, 0.1]))
        seed = 5000 + case
        m1, m2, _ = synth.make_matches(seed, M, frac, grid=(30, 40) if case % 3 == 0 else None)
        samples = synth.draw_samples(seed, M, nbIter)
        try:
            Ho, nbo, inlo, _ = OO.RANSAC_from_samples(m1, m2, samples, tol)
            expect = 0 if Ho is not None else 1
        except TypeError:
            expect = 2
        H, nb, mask, st = run_kernel(rf, m1, m2, samples, tol)
        assert st == expect, (case, M, nbIter, frac, tol, st, expect)
        if expect == 0:
            n_ok += 1
            assert nb == int(nbo) and np.array_equal(mask, inlo), (case, M, nbIter, frac, tol)
            np.testing.assert_allclose(H, Ho, rtol=0, atol=2e-7)
        elif expect == 1:
            n_none += 1
        else:
            n_nomodel += 1
    print("fuzz: %d ok, %d None, %d no-model" % (n_ok, n_none, n_nomodel))
    assert n_ok >= 20
