"""evalYFCC's relative-pose metric on the device (rf_yfcc_matches, rf_essential_ransac, rf_recover_pose) against the numpy
restatement tests/pose_oracle.py, which tests/test_pose_oracle.py ties to cv2."""
import numpy as np
import pytest
import torch
from conftest import golden

import pose_oracle as PO

pytestmark = pytest.mark.gpu
G = golden("yfcc_pose")
THR = float(G["threshold"])


def dev(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def n_dev(N):
    return torch.tensor([N], dtype=torch.int32, device="cuda")


def scene(s):
    N, outlier, seed, planar = G["scenes"][s]
    return PO.scene(int(N), outlier, int(seed), planar=bool(planar))[:2]


def run(rf, p1, p2, threshold=THR):
    ops = rf.ops
    P1, P2 = dev(p1), dev(p2)
    rec, mask = ops.essential_ransac(P1, P2, n_dev(len(p1)), threshold)
    out, bits = ops.recover_pose(P1, P2, mask, rec)
    return ops.read_pose_record(rec), mask[:len(p1)].cpu().numpy(), out[:len(p1)].cpu().numpy(), bits[:len(p1)].cpu().numpy()


@pytest.mark.parametrize("N", [6, 7, 1000, 300000])
def test_sample_table_bit_exact(rf, N):
    idx = rf.ops.essential_samples(n_dev(N)).cpu().numpy()
    np.testing.assert_array_equal(idx, PO.samples(N))


def residuals(E, x1, x2):
    E = E.reshape(3, 3)
    EEt = E @ E.T
    c = 2 * EEt @ E - np.trace(EEt) * E
    ep = np.abs(np.einsum("ni,ij,nj->n", np.c_[x2, np.ones(5)], E, np.c_[x1, np.ones(5)]))
    return abs(np.linalg.det(E)), np.abs(c).max(), ep.max()


@pytest.mark.parametrize("s", [12, 14, 17, 18])
def test_five_point_solutions(rf, s):
    p1, p2 = scene(s)
    idx = PO.samples(len(p1))[:200]
    E, n = rf.ops.essential_five_point(dev(p1), dev(p2), dev(idx, torch.int32))
    E, n = E.cpu().numpy(), n.cpu().numpy()
    for k in range(len(idx)):
        mine = PO.canonical(E[k, :n[k]]) if n[k] else np.zeros((0, 9))
        ref, roots, basis = PO.five_point(p1[idx[k]], p2[idx[k]], return_roots=True)
        for e in mine:
            r = residuals(e, p1[idx[k]], p2[idx[k]])
            assert r[0] < 1e-7 and r[1] < 1e-6 and r[2] < 1e-8, r   # the constraints of a unit-norm E, fp64 elimination
        # A solution of one side without an equal one (1e-6) on the other must be either
        #  - at a real root far from the origin of the oracle's hidden variable (|z| > 1e3: the pencil's eigenvalue, and the E
        #    built from it as z Z + ..., carry an error growing with |z|, and the oracle's eigenvector test may drop it), matched
        #    through z to 1e-5 relative, or
        #  - a near-double root: two of the oracle's ten roots (complex ones included) within 1e-3 (1 + |z|) of its z.
        zb = {id(b): np.array([PO.hidden_z(f, basis) for f in b]) for b in (mine, ref)}
        for a, b in ((mine, ref), (ref, mine)):
            for e in a:
                if len(b) and np.abs(b - e).max(axis=1).min() < 1e-6:
                    continue
                z = PO.hidden_z(e, basis)
                if abs(z) > 1e3 and ((len(b) and np.abs(zb[id(b)] - z).min() <= 1e-5 * abs(z)) or
                                     np.abs(roots[np.abs(roots.imag) <= 1e-9 * abs(roots)] - z).min(initial=np.inf) <= 1e-5 * abs(z)):
                    continue          # at a real root of the pencil; its residuals are checked above
                near = np.abs(roots - z) <= 1e-3 * (1 + abs(z))
                assert near.sum() >= 2, (k, z, np.sort_complex(roots))


def test_scoring_bit_exact(rf):
    p1, p2 = scene(15)
    Es = np.stack([PO.five_point(p1[i], p2[i])[0] for i in PO.samples(len(p1))[:20]])
    counts, err = rf.ops.essential_score(dev(p1), dev(p2), dev(Es), THR, want_err=True)
    err = err.cpu().numpy()
    for m, e in enumerate(Es):
        ref = PO.sampson(e, p1, p2)
        np.testing.assert_array_equal(err[m], ref)
        assert int(counts[m]) == int(np.count_nonzero(ref <= PO.thr2(THR)))


@pytest.mark.parametrize("s", [s for s in range(len(G["scenes"])) if G["scenes"][s][0] >= 5])
def test_end_to_end_against_oracle(rf, s):
    p1, p2 = scene(s)
    N = len(p1)
    rec, mask, out, bits = run(rf, p1, p2)
    est, r, rp = PO.pose(p1, p2, THR)
    assert rec["n_points"] == N and rec["status"] == rf.ops.POSE_OK
    if N == 5:
        A, B = PO.canonical(rec["E"].reshape(-1, 9)), PO.canonical(r["E"])
        assert len(A) == len(B) and all(np.abs(B - e).max(axis=1).min() < 1e-9 for e in A)
        assert mask.all()
        return
    # the device's best and budget against the oracle's own run; the replay of the device's own candidates and counts, launch
    # by launch, is test_gpu_pose_stages.py's test_ransac_stages_bit_exact
    E_dev = PO.canonical(rec["E"].reshape(-1, 9))[0]
    same = np.abs(E_dev - r["E"][0]).max() < 1e-7
    if not same:
        # certified as a tie between candidates of one sample: the device's E is a candidate of the oracle's best sample with
        # the best count
        bi, _ = r["best"]
        assert rec["best"][0] == bi and rec["ransac_count"] == r["count"]
        assert np.abs(PO.canonical(r["cands"][bi]) - E_dev).max(axis=1).min() < 1e-7
        return
    assert rec["best"][0] == r["best"][0] and rec["ransac_count"] == r["count"] and rec["niters"] == r["niters"]
    d = np.nonzero(mask != r["mask"])[0]
    t2 = np.float64(PO.thr2(THR))
    assert np.all(np.abs(PO.sampson(r["E"][0], p1[d], p2[d]).astype(np.float64) - t2) <= 1e-6 * t2)
    # recoverPose on the device's own E and mask
    rp = PO.recover_pose(rec["E"].reshape(-1, 9), p1, p2, mask)
    poses_ref = rp[4][0][0]
    m = mask.astype(bool)
    flips = 0
    for p, P in enumerate(rec["poses"][0]):
        d = [np.abs(P - Q).max() for Q in poses_ref]
        q = int(np.argmin(d))
        assert d[q] < 1e-12, d                      # the same four poses as a set
        # every cheirality decision equals the fp64 one, except where fp64 itself cannot decide it (margin < 1)
        ok_ref = PO.cheirality(poses_ref[q], p1, p2)[0]
        ok_dev = ((bits >> p) & 1).astype(bool)
        diff = np.nonzero(ok_dev != ok_ref)[0]
        if len(diff):
            margin = PO.cheirality_margin(poses_ref[q], p1[diff], p2[diff])
            assert np.all(margin < 1.0), (p, diff[margin >= 1.0][:5], margin[margin >= 1.0][:5])
            flips += int(np.count_nonzero(m[diff]))
    counts_ref = rp[4][0][1]
    if flips == 0:
        assert rec["pose_count"] == rp[0]
        if sorted(counts_ref).count(max(counts_ref)) == 1:
            np.testing.assert_allclose(rec["R"], rp[1], atol=1e-12)
            np.testing.assert_allclose(rec["t"], rp[2], atol=1e-12)
            np.testing.assert_array_equal(out.astype(bool), rp[3])


@pytest.mark.parametrize("f", range(4))
def test_matches_bit_exact(rf, f):
    angle, hB, wB, hA, wA = G["flows"][f]
    flow, mb = G["f%d_flow" % f], G["f%d_mask" % f]
    n1 = PO.norm_params(tuple(G["f%d_orgA" % f]), (wA, hA), G["f%d_KA" % f])
    n2 = PO.norm_params(tuple(G["f%d_orgB" % f]), (wB, hB), G["f%d_KB" % f])
    pts1, pts2, N = rf.ops.yfcc_matches(dev(flow, torch.float32), dev(mb, torch.uint8), int(angle), (wA, hA), (wB, hB), n1, n2)
    N = int(N)
    assert np.array_equal(pts1[:N].cpu().numpy(), G["f%d_pts1" % f]) and np.array_equal(pts2[:N].cpu().numpy(), G["f%d_pts2" % f])


def test_matches_empty_and_shape_mismatch(rf):
    flow = torch.zeros((7, 9, 2), device="cuda")
    _, _, N = rf.ops.yfcc_matches(flow, torch.zeros((7, 9), dtype=torch.uint8, device="cuda"), 0, (5, 5), (9, 7), (0, 0, 1, 1), (0, 0, 1, 1))
    assert int(N) == 0
    with pytest.raises(IndexError):
        rf.ops.yfcc_matches(flow, torch.zeros((7, 9), dtype=torch.uint8, device="cuda"), 90, (5, 5), (9, 7), (0, 0, 1, 1), (0, 0, 1, 1))
    flow = torch.zeros((9, 9, 2), device="cuda")
    _, _, N = rf.ops.yfcc_matches(flow, torch.zeros((9, 9), dtype=torch.uint8, device="cuda"), 0, (5, 5), (9, 9), (0, 0, 1, 1), (0, 0, 1, 1))
    rec, mask = rf.ops.essential_ransac(torch.zeros((81, 2), dtype=torch.float64, device="cuda"),
                                        torch.zeros((81, 2), dtype=torch.float64, device="cuda"), N)
    assert rf.ops.read_pose_record(rec)["status"] == rf.ops.POSE_TOO_FEW


def test_two_streams_and_graph_capture(rf):
    ops = rf.ops
    scenes = [scene(14), scene(16)]
    alone = [run(rf, *sc)[0] for sc in scenes]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    recs = []
    torch.cuda.synchronize()
    for (p1, p2), st in zip(scenes, streams):
        with torch.cuda.stream(st):
            P1, P2 = dev(p1), dev(p2)
            rec, mask = ops.essential_ransac(P1, P2, n_dev(len(p1)), THR)
            ops.recover_pose(P1, P2, mask, rec)
            recs.append((rec, P1, P2, mask))
    torch.cuda.synchronize()
    for a, (rec, *_) in zip(alone, recs):
        b = ops.read_pose_record(rec)
        assert a["best"] == b["best"] and np.array_equal(a["E"], b["E"]) and np.array_equal(a["R"], b["R"])
    # one CUDA graph of the three stages
    p1, p2 = scenes[0]
    H, W = 40, 50
    flow = torch.rand((H, W, 2), device="cuda") * 2 - 1
    mb = (torch.rand((H, W), device="cuda") < 0.7).to(torch.uint8)
    norm = (0.5, 0.25, 30.0, 31.0)

    def stages():
        pts1, pts2, N = ops.yfcc_matches(flow, mb, 0, (W, H), (W, H), norm, norm)
        rec, mask = ops.essential_ransac(pts1, pts2, N, THR)
        out, _ = ops.recover_pose(pts1, pts2, mask, rec)
        return rec, mask, out

    eager = [t.clone() for t in stages()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        stages()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            outs = stages()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, outs):
        assert torch.equal(a, b)


def geometric_pair(rs, h8, w8, K_A, K_B, orgA, orgB, nH=2):
    """What ``results.save_pair`` stores for a synthetic pair whose composed flow follows a smooth-depth two-view scene:
    identity homographies (the composition then reduces to grid + upsampled flowDown8), flowDown8 = the scene's displacement at
    the 8 x 8 block centres, matchabilities above 0.95 on most blocks (hypothesis 1 fills some of hypothesis 0's holes).
    Returns (out dict, maskBG, R_ab, t_ab) with (R_ab, t_ab) the motion from camera A to camera B."""
    H, W = 8 * h8, 8 * w8
    cxA, cyA, fxA, fyA = PO.norm_params(orgA, (W, H), K_A)
    cxB, cyB, fxB, fyB = PO.norm_params(orgB, (W, H), K_B)
    ang = rs.uniform(-0.15, 0.15, 3)
    Kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]])
    import scipy.linalg
    R = scipy.linalg.expm(Kx)                    # X_A = R X_B + t
    t = rs.uniform(-0.5, 0.5, 3)
    ys, xs = np.meshgrid(np.arange(h8) * 8 + 3.5, np.arange(w8) * 8 + 3.5, indexing="ij")
    d = 4 + 0.8 * np.sin(xs / W * 3 + rs.rand()) + 0.6 * np.cos(ys / H * 2 + rs.rand())
    X = np.stack([(xs - cxB) / fxB * d, (ys - cyB) / fyB * d, d], -1) @ R.T + t
    xa, ya = fxA * X[..., 0] / X[..., 2] + cxA, fyA * X[..., 1] / X[..., 2] + cyA
    fl = np.stack([2 * xa / (W - 1) - 1 - (2 * xs / (W - 1) - 1), 2 * ya / (H - 1) - 1 - (2 * ys / (H - 1) - 1)])
    flow = np.repeat(fl[None], nH, 0).astype(np.float32)
    match = np.full((nH, 2, h8, w8), 0.99, np.float32)
    match[0, 0, : h8 // 3] = 0.5
    if nH > 1:
        match[1, 0, : h8 // 6] = 0.5
    bg = np.ones((H, W), bool)
    bg[H // 2:, : W // 4] = False
    out = {"H": np.repeat(np.eye(3, dtype=np.float32)[None], nH, 0), "flowDown8": flow, "matchDown8": match}
    return out, bg, R.T, (-R.T @ t)[:, None]


def device_pose_or_tie(rf, p1, p2, err_dev, err_ref, r, t):
    """True when a device / oracle disagreement on one pair is a certified tie: the device's RANSAC best comes from the
    oracle's best sample with the same count (candidates of one sample visited in a different order), or the pose choice ties."""
    rec, _, _, _ = run(rf, p1, p2)
    est, rr, rp = PO.pose(p1, p2, THR)
    if rr is None:
        return False
    if rec["best"][0] != rr["best"][0] or rec["ransac_count"] != rr["count"]:
        # the replays saw different counts: the device's and the oracle's solutions of a sample agree to ~1e-9, which moves
        # a fp32 Sampson error only for points within ~1e-7 of (float)(t^2).  Certified when the two best counts differ by
        # no more than the points within 1e-4 (relative) of the threshold under either best model.
        t2 = np.float64(PO.thr2(THR))
        Ed = rec["E"].reshape(-1, 9)[0]
        near = np.zeros(len(p1), bool)
        for e in (Ed, rr["E"][0]):
            near |= np.abs(PO.sampson(e, p1, p2).astype(np.float64) - t2) <= 1e-4 * t2
        return abs(rec["ransac_count"] - rr["count"]) <= int(near.sum()) and int(near.sum()) > 0
    E_dev = PO.canonical(rec["E"].reshape(-1, 9))[0]
    if np.abs(E_dev - rr["E"][0]).max() >= 1e-7:
        return np.abs(PO.canonical(rr["cands"][rr["best"][0]]) - E_dev).max(axis=1).min() < 1e-7
    g = rp[4][0][1]
    return g.count(max(g)) > 1


def test_yfcc_pose_errors_directory_round_trip(rf, tmp_path):
    """save_pair / save_rotation -> results.yfcc_pose_errors against the driver's per-pair loop restated on the oracle
    (getResults.py:298-331), the per-pair errors within 1e-6 degrees and the four Acc values equal."""
    rs = np.random.RandomState(11)
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
    import json
    rot = json.load(open(fine / "rotation.json"))
    errs = rf.results.yfcc_pose_errors(pairs, str(fine), str(coarse), str(fine), rot, R_list, T_list, K_list, org, resized)
    flowList = [item for item in __import__("os").listdir(fine) if "flow" in item]
    ref = []
    for i, (a, b) in enumerate(pairs):
        t = rf.results.load_pair(i, str(fine), str(coarse), flowList)
        if t is None:
            ref.append(180)
            continue
        fg, mg = rf.pipeline.getFlow_corr(*t, th=0.95, multiH=True)
        bg = np.load(fine / "maskBG_{}_2H.npy".format(i))
        flow, mb = fg[0].cpu().numpy(), (mg[0, ..., 0].cpu().numpy() >= 0.95) & bg
        fy, my = rf.results.getFlow_yfcc_from_files(i, str(fine), None, str(coarse), str(fine), True, 0.95)
        assert np.array_equal(fy.cpu().numpy(), flow) and np.array_equal(my.cpu().numpy(), mb)
        p1, p2 = PO.matches_from_flow(flow.copy(), mb, resized[a], resized[b], rot[str(i)])
        if len(p1) == 0:
            ref.append(180)
            continue
        p1 = PO.norm_kp(PO.norm_params(org[a], resized[a], K_list[a]), p1)
        p2 = PO.norm_kp(PO.norm_params(org[b], resized[b], K_list[b]), p2)
        r = R_list[b] @ R_list[a].T
        tt = T_list[b] - r @ T_list[a]
        est, _, _ = PO.pose(p1, p2, THR)
        e = 180 if est is None else max(PO.evaluate_R_t(r, tt, est[0], est[1]))
        ref.append(e)
        if abs(errs[i] - e) > 1e-6:
            assert device_pose_or_tie(rf, p1, p2, errs[i], e, r, tt), (i, errs[i], e)
    assert errs[2] == ref[2] == 180 and errs[3] == ref[3] == 180
    assert max(ref[0], ref[1]) < 20                             # the synthetic scenes are solvable
    assert rf.results.pose_accuracy(errs) == rf.results.pose_accuracy(ref)


def test_yfcc_pose_matches_oracle(rf):
    """results.yfcc_pose's (R, t) against the oracle on the same normalised points (ties certified)."""
    rs = np.random.RandomState(3)
    h8, w8 = 10, 14
    H, W = 8 * h8, 8 * w8
    K_A = np.array([[140.0, 0, 2.0], [0, 150.0, -1.0], [0, 0, 1]])
    K_B = np.array([[160.0, 0, -3.0], [0, 145.0, 2.5], [0, 0, 1]])
    orgA, orgB = (2 * W + 1, 2 * H + 3), (3 * W, 3 * H - 2)
    out, bg, _, _ = geometric_pair(rs, h8, w8, K_A, K_B, orgA, orgB, nH=1)
    fg, mg = rf.pipeline.getFlow_corr(out["flowDown8"], out["H"], out["matchDown8"], th=0.95, multiH=True)
    flow, mb = fg[0], (mg[0, ..., 0] >= 0.95)
    got, n = rf.results.yfcc_pose(flow, mb, (W, H), (W, H), 0, K_A, K_B, orgA, orgB)
    p1, p2 = PO.matches_from_flow(flow.cpu().numpy().copy(), mb.cpu().numpy(), (W, H), (W, H), 0)
    p1 = PO.norm_kp(PO.norm_params(orgA, (W, H), K_A), p1)
    p2 = PO.norm_kp(PO.norm_params(orgB, (W, H), K_B), p2)
    est, _, _ = PO.pose(p1, p2, THR)
    assert n == len(p1) and got is not None and est is not None
    # yfcc_pose's own matches + norm_kp give the kernels exactly the oracle's normalised points: the same (R, t) bit for bit
    rec = run(rf, p1, p2)[0]
    assert np.array_equal(got[0], rec["R"]) and np.array_equal(got[1], rec["t"])
    # against the oracle: the two five-point solvers agree to ~1e-8 on E (test_five_point_solutions bounds them at 1e-6 on
    # unit-norm E), and R / t follow E through the well-conditioned decomposition
    if not (np.abs(got[0] - est[0]).max() < 1e-6 and np.abs(got[1] - est[1]).max() < 1e-6):
        assert device_pose_or_tie(rf, p1, p2, None, None, None, None)
    with pytest.raises(NotImplementedError):
        rf.results.yfcc_pose(flow, mb, (W, H), (W, H), 0, K_A, K_B, orgA, orgB, ransac=False)
    acc = rf.results.pose_accuracy([1.0, 7.0, 12.0, 180])
    assert acc == {"Acc@5": 0.25, "Acc@10": 0.5, "Acc@15": 0.75, "Acc@20": 0.75}
    # evaluate_R_t of the results module is the driver's statement
    assert rf.results.evaluate_R_t(np.eye(3), np.ones(3), est[0], est[1]) == PO.evaluate_R_t(np.eye(3), np.ones(3), est[0], est[1])
