"""cv2.findFundamentalMat(FM_8POINT) on the device (rf_fundamental_8point, rf_fundamental_moments) and the driver's non-RANSAC
opencv_decompose / per-pair loop, against tests/fundamental_oracle.py and the cv2 results of tests/golden/yfcc_pose_8point.npz
under the rules of tests/test_pose8_oracle.py."""
import numpy as np
import pytest
import torch
from conftest import golden

import fundamental_oracle as FO
import pose_oracle as PO
from test_pose8_oracle import EPS, conditioning, counts_certified, f_close, points, unpack

pytestmark = pytest.mark.gpu
G = golden("yfcc_pose_8point")
THR = float(G["threshold"])


def dev(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def n_dev(N):
    return torch.tensor([N], dtype=torch.int32, device="cuda")


def padded(p, cap):
    out = torch.full((max(cap, 1), 2), 7.0, dtype=torch.float64, device="cuda")    # rows past N must not be read
    out[:len(p)] = dev(p)
    return out


def run(rf, p1, p2, cap=None):
    ops = rf.ops
    cap = len(p1) if cap is None else cap
    P1, P2 = padded(p1, cap), padded(p2, cap)
    rec, mask = ops.fundamental_8point(P1, P2, n_dev(len(p1)))
    out, _ = ops.recover_pose(P1, P2, mask, rec)
    return ops.read_pose_record(rec), mask[:len(p1)].cpu().numpy(), out[:len(p1)].cpu().numpy()


def moments_rel_err(rf, p1, p2):
    """Relative max-abs error of the device's A against the sequential sums, per lambda_0 (the dA of f_tolerance)."""
    got = rf.ops.fundamental_moments(dev(p1), dev(p2), n_dev(len(p1))).cpu().numpy()
    ref = FO.moments(FO.as_f32(p1), FO.as_f32(p2))
    A = np.zeros((9, 9))
    A[FO.IU] = got[6:]
    return np.abs(A - np.triu(ref[4])).max() / np.linalg.eigvalsh(ref[4])[-1]


@pytest.mark.parametrize("s", [s for s in range(len(G["scenes"])) if G["scenes"][s][0] >= 8 and G["s%d_has_F" % s]])
def test_moments_against_sequential_sums(rf, s):
    p1, p2 = points(s)
    P1, P2, N = dev(p1), dev(p2), n_dev(len(p1))
    got = rf.ops.fundamental_moments(P1, P2, N).cpu().numpy()
    again = rf.ops.fundamental_moments(P1, P2, N).cpu().numpy()
    assert np.array_equal(got.view(np.uint64), again.view(np.uint64))          # no atomics: the same bits every run
    c1, c2, s1, s2, A = FO.moments(FO.as_f32(p1), FO.as_f32(p2))
    np.testing.assert_allclose(got[:4], np.r_[c1, c2], rtol=1e-15, atol=1e-15 * np.abs(np.r_[c1, c2]).max())
    # a mean of N positive distances: the sequential sum itself carries rounding of order sqrt(N) eps, so two summation orders
    # agree to that, not to 1e-15 (which the centroids meet)
    np.testing.assert_allclose(got[4:6], [s1, s2], rtol=max(1e-15, 2 * np.sqrt(len(p1)) * EPS), atol=0)
    ref = A[FO.IU]
    assert np.abs(got[6:] - ref).max() <= 1e-13 * np.abs(ref).max()


@pytest.mark.parametrize("s", range(len(G["scenes"])))
def test_fundamental_against_cv2(rf, s):
    p1, p2 = points(s)
    N = len(p1)
    rec, mask, out = run(rf, p1, p2, cap=N + 37)
    assert rec["n_points"] == N
    if N < 5:
        assert rec["status"] == rf.ops.POSE_TOO_FEW
        return
    if not bool(G["s%d_has_F" % s]):
        assert rec["status"] == rf.ops.POSE_NO_MODEL and not bool(G["s%d_has_pose" % s])
        if bool(G["s%d_has_mask" % s]):
            np.testing.assert_array_equal(mask, unpack(G["s%d_mask" % s], N))      # degenerate input: F None, mask all ones
        return
    assert rec["status"] in (rf.ops.POSE_OK, rf.ops.POSE_NO_POSE)
    np.testing.assert_array_equal(mask, unpack(G["s%d_mask" % s], N))
    F_cv = G["s%d_F" % s]
    dA = moments_rel_err(rf, p1, p2) if N >= 8 else 0.0
    ok, d = f_close(rec["E"].reshape(-1, 9), F_cv, conditioning(p1, p2), dA)
    assert ok, (d, conditioning(p1, p2), dA)
    # N == 7: the same candidates in the same order; every N: the driver's chained counts, equal or certified
    counts = [int(rec["pose_counts"][c][rec["pose_counts"][c].argmax()]) for c in range(rec["n_E"])]
    assert counts_certified(rec["E"].reshape(-1, 9), F_cv, p1, p2, counts, G["s%d_cand_counts" % s]), counts
    if counts == list(G["s%d_cand_counts" % s]) and d <= 1e-9 and bool(G["s%d_has_pose" % s]):
        assert rec["pose_count"] == max(counts)
        c = rec["pose"][0]
        g = list(rec["pose_counts"][c])
        if g.count(max(g)) > 1:
            # tied poses: which one the >= order picks depends on the SVD's signs; cv2's must be one of the tied poses
            assert any(np.abs(P[:, :3] - G["s%d_R" % s]).max() < 1e-8 and np.abs(P[:, 3:] - G["s%d_t" % s]).max() < 1e-8
                       for k, P in enumerate(rec["poses"][c]) if g[k] == max(g))
            return
        np.testing.assert_allclose(rec["R"], G["s%d_R" % s], atol=1e-8, rtol=0)
        np.testing.assert_allclose(rec["t"], G["s%d_t" % s], atol=1e-8, rtol=0)
        if rec["n_E"] == 1:
            np.testing.assert_array_equal(out, unpack(G["s%d_pose_mask" % s], N))


def test_graph_replay_and_two_streams_bit_identical(rf):
    ops = rf.ops
    s = next(s for s in range(len(G["scenes"])) if G["scenes"][s][0] == 300000)
    p1, p2 = points(s)
    cap = 480 * 640
    P1, P2, N = padded(p1, cap), padded(p2, cap), n_dev(len(p1))

    def stages(rec=None):
        rec, mask = ops.fundamental_8point(P1, P2, N, rec)
        out, _ = ops.recover_pose(P1, P2, mask, rec)
        return rec, mask, out

    eager = [t.clone() for t in stages()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        stages()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            outs = stages()
    torch.cuda.current_stream().wait_stream(st)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, outs):
        assert torch.equal(a, b)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    res = []
    for st in streams:
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            res.append(stages())
    torch.cuda.synchronize()
    for r in res:
        for a, b in zip(eager, r):
            assert torch.equal(a, b)


@pytest.mark.parametrize("s", [3, 6, 15, 19, 22])
def test_opencv_decompose_both_branches(rf, s):
    p1, p2 = points(s)
    ops = rf.ops
    res, m = rf.results.opencv_decompose(p1, p2, True, THR)
    P1, P2 = dev(p1), dev(p2)
    rec, mask = ops.essential_ransac(P1, P2, n_dev(len(p1)), THR)
    out, _ = ops.recover_pose(P1, P2, mask, rec)
    r = ops.read_pose_record(rec)
    if r["status"] != ops.POSE_OK or r["pose_count"] <= 0:
        assert res is None and m is None
    else:
        assert np.array_equal(res[0], r["R"]) and np.array_equal(res[1], r["t"])
        assert torch.equal(m.view(-1), out[:len(p1)])
    res8, m8 = rf.results.opencv_decompose(p1, p2, False)
    assert (res8 is not None) == bool(G["s%d_has_pose" % s])
    if res8 is not None:
        r8 = run(rf, p1, p2)[0]
        assert np.array_equal(res8[0], r8["R"]) and np.array_equal(res8[1], r8["t"])
        assert int(m8.sum()) == r8["pose_count"]


def test_yfcc_pose_errors_8point_directory_round_trip(rf, tmp_path):
    """save_pair / save_rotation -> results.yfcc_pose_errors_8point against the driver's loop restated on the oracle."""
    from test_gpu_pose import geometric_pair
    import json
    import os
    rs = np.random.RandomState(12)
    fine, coarse = tmp_path / "fine", tmp_path / "coarse"
    fine.mkdir()
    coarse.mkdir()
    h8, w8 = 12, 16
    H, W = 8 * h8, 8 * w8
    n_img = 8
    K_list = [np.array([[150.0 + 7 * i, 0, 1.5 - i], [0, 155.0 - 3 * i, 0.5 * i], [0, 0, 1]]) for i in range(n_img)]
    org = [(2 * W + i, 2 * H - i) for i in range(n_img)]
    resized = [(W, H)] * n_img
    R_list = [np.eye(3)] * n_img
    T_list = [np.zeros((3, 1))] * n_img
    pairs = [(0, 1), (2, 3), (4, 5), (6, 7), (1, 0)]
    rotation = {}
    for i, (a, b) in enumerate(pairs):
        if i == 3:
            continue                                             # no files: 180
        out, bg, R_ab, t_ab = geometric_pair(rs, h8, w8, K_list[a], K_list[b], org[a], org[b])
        if i == 2:
            out["matchDown8"][:] = 0.1                           # nothing matchable: 180
        if i < 3:
            R_list[b], T_list[b] = R_ab, t_ab
        rf.results.save_pair(str(coarse), str(fine), i, out, bg)
        rotation[i] = 0
    rf.results.save_rotation(str(fine), rotation)
    rot = json.load(open(fine / "rotation.json"))
    errs = rf.results.yfcc_pose_errors_8point(pairs, str(fine), str(coarse), str(fine), rot, R_list, T_list, K_list, org, resized)
    flowList = [item for item in os.listdir(fine) if "flow" in item]
    ref = []
    for i, (a, b) in enumerate(pairs):
        flow, mb = rf.results.getFlow_yfcc_from_files(i, str(fine), flowList, str(coarse), str(fine), True, 0.95)
        if len(flow) == 0:
            ref.append(180)
            continue
        p1, p2 = PO.matches_from_flow(flow.cpu().numpy().copy(), mb.cpu().numpy(), resized[a], resized[b], rot[str(i)])
        if len(p1) == 0:
            ref.append(180)
            continue
        p1 = PO.norm_kp(PO.norm_params(org[a], resized[a], K_list[a]), p1)
        p2 = PO.norm_kp(PO.norm_params(org[b], resized[b], K_list[b]), p2)
        r = R_list[b] @ R_list[a].T
        tt = T_list[b] - r @ T_list[a]
        est = FO.opencv_decompose(p1, p2)[0]
        ref.append(180 if est is None else max(PO.evaluate_R_t(r, tt, est[0], est[1])))
        assert abs(errs[i] - ref[i]) <= 1e-6, (i, errs[i], ref[i])
    assert errs[2] == ref[2] == 180 and errs[3] == ref[3] == 180
    assert rf.results.pose_accuracy(errs) == rf.results.pose_accuracy(ref)
