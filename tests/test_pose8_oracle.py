"""The numpy restatement of cv2.findFundamentalMat(FM_8POINT) (tests/fundamental_oracle.py) against cv2's results stored by
tests/gen_pose8_golden.py from the reference's own opencv_decompose(p1, p2, False, threshold): F, the candidate count and order
for N = 7, the None cases, and the driver's recoverPose counts and (R, t)."""
import numpy as np
import pytest
from conftest import golden

import fundamental_oracle as FO
import pose_oracle as PO

G = golden("yfcc_pose_8point")
EPS = np.finfo(np.float64).eps


def points(s):
    p1, p2 = FO.golden_points(G["scenes"][s])
    np.testing.assert_array_equal(np.array([p1.sum(), p2.sum()]), G["s%d_checksum" % s])
    return p1, p2


def conditioning(p1, p2):
    """The relative gap that bounds how far two backward-stable solvers' F may differ: (lambda_7 - lambda_8) / lambda_0 of A for
    N >= 8, sigma_6 / sigma_0 of the 7 x 9 system for N = 7 (its null space), 0 when there is no model."""
    m1, m2 = FO.as_f32(p1), FO.as_f32(p2)
    norm = FO.normalisation(m1, m2)
    if norm is None:
        return 0.0
    if len(p1) == 7:
        S = np.linalg.svd(FO.rows(m1, m2, norm), compute_uv=False)
        return float(S[6] / S[0])
    w = np.linalg.eigvalsh(FO.moments(m1, m2)[4])[::-1]
    return float((w[7] - w[8]) / w[0])


def f_tolerance(gap, dA=0.0):
    """Relative max-abs distance allowed between two F (F22 = 1) from the same moments (up to a relative perturbation dA of A):
    1e-11 where the problem is well conditioned, else the first-order perturbation bound of the null vector, 64 (eps + dA) / gap."""
    return max(1e-11, 64 * (EPS + dA) / max(gap, 1e-300))


def f_close(F_a, F_b, gap, dA=0.0):
    F_a, F_b = np.asarray(F_a).reshape(-1, 9), np.asarray(F_b).reshape(-1, 9)
    d = np.abs(F_a - F_b).max() / np.abs(F_b).max()
    return len(F_a) == len(F_b) and d <= f_tolerance(gap, dA), d


def counts_certified(F_a, F_b, p1, p2, counts_a, counts_b):
    """recoverPose counts from two F agree, or every point whose chosen-pose cheirality decision differs is within the pose
    difference of flipping: its fp64 margin (tests/pose_oracle.py: cheirality_margin) scaled by 64 eps / |pose_a - pose_b|
    is below 1."""
    if list(counts_a) == list(counts_b):
        return True
    for Ea, Eb in zip(np.asarray(F_a).reshape(-1, 9), np.asarray(F_b).reshape(-1, 9)):
        Pa, Pb = PO.decompose(Ea), PO.decompose(Eb)
        for P, Q in zip(Pa, Pb):
            delta = np.abs(P - Q).max() + 64 * EPS
            diff = np.nonzero(PO.cheirality(P, p1, p2)[0] != PO.cheirality(Q, p1, p2)[0])[0]
            if len(diff) and not np.all(PO.cheirality_margin(Q, p1[diff], p2[diff]) * (64 * EPS / delta) < 1.0):
                return False
    return len(counts_a) == len(counts_b)


def unpack(bits, n):
    return np.unpackbits(bits)[:n].astype(np.uint8)


def test_golden_covers_the_issue_cases():
    sc = G["scenes"]
    n7 = [len(G["s%d_F" % s]) // 3 for s in range(len(sc)) if sc[s][0] == 7 and sc[s][4] == 0]
    assert 1 in n7 and 3 in n7
    assert {0, 4, 5, 6, 8, 9, 50, 2000, 100000, 300000} <= set(int(n) for n in sc[:, 0])
    assert str(G["cv2_version"]).startswith("4.")


@pytest.mark.parametrize("s", range(len(G["scenes"])))
def test_fundamental_matches_cv2(s):
    p1, p2 = points(s)
    N = len(p1)
    F, mask, _ = FO.fundamental(p1, p2)
    if not bool(G["s%d_has_F" % s]):
        assert F is None
        assert bool(G["s%d_has_mask" % s]) == (mask is not None)
        if mask is not None:
            np.testing.assert_array_equal(mask, unpack(G["s%d_mask" % s], N))
        assert not bool(G["s%d_has_pose" % s])
        return
    F_cv = G["s%d_F" % s]
    gap = conditioning(p1, p2)
    ok, d = f_close(F, F_cv, gap)
    assert ok, (d, gap, f_tolerance(gap))
    np.testing.assert_array_equal(mask, unpack(G["s%d_mask" % s], N))
    # the driver's loop on the oracle's F: per-candidate chained counts, then its (R, t)
    est, mfinal, _, rp = FO.opencv_decompose(p1, p2)
    counts = [g[k] for _, g, k in rp[4]]
    assert counts_certified(F, F_cv, p1, p2, counts, G["s%d_cand_counts" % s]), (counts, G["s%d_cand_counts" % s])
    assert (est is not None) == bool(G["s%d_has_pose" % s])
    if list(counts) == list(G["s%d_cand_counts" % s]) and d <= 1e-9:
        # the driver's num_inlier (its mask_final aliases the array cv2 writes in place: the last candidate's mask)
        assert rp[0] == max(G["s%d_cand_counts" % s])
        if len(counts) == 1:
            assert rp[0] == int(G["s%d_pose_count" % s])
        np.testing.assert_allclose(est[0], G["s%d_R" % s], atol=1e-8, rtol=0)
        np.testing.assert_allclose(est[1], G["s%d_t" % s], atol=1e-8, rtol=0)
        if "s%d_err" % s in G:
            R_gt, t_gt = PO.scene(N, G["scenes"][s][1], int(G["scenes"][s][2]), planar=bool(G["scenes"][s][3]))[2:]
            assert abs(max(PO.evaluate_R_t(R_gt, t_gt, est[0], est[1])) - float(G["s%d_err" % s])) < 1e-6


def test_fp32_cast_is_visible():
    """Without findFundamentalMat's fp32 cast the eight-point F moves far beyond the tolerance: the comparison can tell."""
    s = next(s for s in range(len(G["scenes"])) if G["scenes"][s][0] == 2000 and G["scenes"][s][4] == 0)
    p1, p2 = points(s)
    F_raw, _ = FO.run8point(p1, p2)
    assert not f_close(F_raw, G["s%d_F" % s], conditioning(p1, p2))[0]


def test_seven_point_normalises():
    """cv2 4.13's seven-point solver normalises the points: the unnormalised statement gives other candidates."""
    s = next(s for s in range(len(G["scenes"])) if G["scenes"][s][0] == 7 and len(G["s%d_F" % s]) == 9)
    p1, p2 = points(s)
    raw = FO.run7point(FO.as_f32(p1), FO.as_f32(p2), normalise=False)
    assert len(raw) != 3 or np.abs(raw.reshape(-1, 3) - G["s%d_F" % s]).max() > 1e-6 * np.abs(G["s%d_F" % s]).max()
