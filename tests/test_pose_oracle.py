"""The numpy restatement of evalYFCC's pose metric (tests/pose_oracle.py) against cv2's results stored by
tests/gen_pose_golden.py from the reference's own functions: RANSAC masks, E, recoverPose's R / t / mask, and the driver's
matches_from_flow + norm_kp points bit for bit."""
import numpy as np
import pytest
from conftest import golden

import pose_oracle as PO

G = golden("yfcc_pose")
THR = float(G["threshold"])


def certified_mask_diff(E_a, E_b, p1, p2, m_a, m_b):
    """Points where two RANSAC masks differ must sit at the threshold under both models: their fp32 Sampson errors straddle
    (float)(t^2) by less than the rounding an E differing in its last bits can move them."""
    d = np.nonzero(m_a != m_b)[0]
    if len(d) == 0:
        return True
    t2 = PO.thr2(THR)
    ea, eb = PO.sampson(E_a, p1[d], p2[d]), PO.sampson(E_b, p1[d], p2[d])
    return bool(np.all(np.abs(ea.astype(np.float64) - t2) <= 1e-6 * t2) and np.all(np.abs(eb.astype(np.float64) - t2) <= 1e-6 * t2))


def scene(s):
    N, outlier, seed, planar = G["scenes"][s]
    p1, p2, R, t = PO.scene(int(N), outlier, int(seed), planar=bool(planar))
    np.testing.assert_array_equal(np.array([p1.sum(), p2.sum()]), G["s%d_checksum" % s])
    return p1, p2


def unpack(bits, n):
    return np.unpackbits(bits)[:n].astype(np.uint8)


@pytest.mark.parametrize("s", range(len(G["scenes"])))
def test_ransac_and_pose_match_cv2(s):
    p1, p2 = scene(s)
    N = len(p1)
    est, r, rp = PO.pose(p1, p2, THR)
    if N < 5:
        assert r is None and not bool(G["s%d_has_pose" % s])
        return
    E_cv = G["s%d_E" % s].reshape(-1, 9)
    m_cv = unpack(G["s%d_mask" % s], N)
    assert r is not None and len(E_cv) == len(r["E"])
    if N == 5:
        # every candidate of the one minimal problem, stacked; cv2's order cannot be reproduced: compare as sets
        A, B = PO.canonical(E_cv), PO.canonical(r["E"])
        for e in A:
            assert np.abs(B - e).max(axis=1).min() < 1e-8
        np.testing.assert_array_equal(r["mask"], m_cv)
    elif np.abs(PO.canonical(E_cv) - PO.canonical(r["E"])).max() < 1e-8:
        assert certified_mask_diff(E_cv[0], r["E"][0], p1, p2, m_cv, r["mask"])
    else:
        # a tie between candidates of the winning sample, which cv2 visits in its own root order: cv2's E must be one of them,
        # with the same count; the pose is then checked from cv2's E
        bi, _ = r["best"]
        same = PO.canonical(r["cands"][bi])
        c = int(np.argmin(np.abs(same - PO.canonical(E_cv)[0]).max(axis=1)))
        assert np.abs(same[c] - PO.canonical(E_cv)[0]).max() < 1e-8 and r["counts"][bi][c] == r["count"] == int(m_cv.sum())
        rp = PO.recover_pose(E_cv, p1, p2, m_cv)
        est = (rp[1], rp[2])
    assert est is not None and bool(G["s%d_has_pose" % s])
    if N == 5:
        # the driver keeps the first stacked candidate with the largest count: with cv2's candidate order unknown, cv2's (R, t)
        # must be the chosen pose of one of the candidates tying at that count
        assert rp[0] == int(G["s%d_pose_count" % s])
        tied = [poses[k] for poses, g, k in rp[4] if g[k] == rp[0]]
        assert any(np.abs(P[:, :3] - G["s%d_R" % s]).max() < 1e-9 and np.abs(P[:, 3:] - G["s%d_t" % s]).max() < 1e-9 for P in tied)
        return
    assert rp[0] == int(G["s%d_pose_count" % s])
    poses, g, _ = rp[4][0]
    if g.count(max(g)) > 1:
        # two poses tie: which one OpenCV's >= order picks depends on its SVD's signs; cv2's must be one of the tied poses
        assert any(np.abs(poses[k][:, :3] - G["s%d_R" % s]).max() < 1e-9 and np.abs(poses[k][:, 3:] - G["s%d_t" % s]).max() < 1e-9
                   for k in range(4) if g[k] == max(g))
        return
    np.testing.assert_allclose(est[0], G["s%d_R" % s], atol=1e-9, rtol=0)
    np.testing.assert_allclose(est[1], G["s%d_t" % s], atol=1e-9, rtol=0)
    np.testing.assert_array_equal(rp[3].astype(np.uint8), unpack(G["s%d_pose_mask" % s], N))
    R_gt, t_gt = G["s%d_R_gt" % s], G["s%d_t_gt" % s]
    assert abs(max(PO.evaluate_R_t(R_gt, t_gt, est[0], est[1])) - float(G["s%d_err" % s])) < 1e-6


@pytest.mark.parametrize("f", range(4))
def test_matches_from_flow_bit_exact(f):
    angle, hB, wB, hA, wA = G["flows"][f]
    p1, p2 = PO.matches_from_flow(G["f%d_flow" % f].copy(), G["f%d_mask" % f], (wA, hA), (wB, hB), int(angle))
    n1 = PO.norm_params(tuple(G["f%d_orgA" % f]), (wA, hA), G["f%d_KA" % f])
    n2 = PO.norm_params(tuple(G["f%d_orgB" % f]), (wB, hB), G["f%d_KB" % f])
    assert np.array_equal(PO.norm_kp(n1, p1), G["f%d_pts1" % f])
    assert np.array_equal(PO.norm_kp(n2, p2), G["f%d_pts2" % f])


def test_sample_stream_redraws_repeats():
    for N in (6, 7, 1000):
        idx = PO.samples(N)
        assert idx.shape == (1000, 5) and idx.min() >= 0 and idx.max() < N
        assert all(len(set(row)) == 5 for row in idx)


def test_update_num_iters_edges():
    assert PO.update_num_iters(0.999, 0.0, 5, 1000) == 0       # every point an inlier: OpenCV's denom < DBL_MIN branch
    assert PO.update_num_iters(0.999, 1.0, 5, 1000) == 1000
    assert PO.update_num_iters(0.999, 0.5, 5, 1000) == int(np.rint(np.log(0.001) / np.log(1 - 0.5 ** 5)))
