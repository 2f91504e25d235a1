"""evalYFCC's pose kernels (csrc/pose.cu) stage by stage on their own intermediates, bit for bit: rf_essential_ransac's subset
table, five-point candidates, per-launch Sampson counts and sequential replay read back from a caller-owned workspace;
rf_essential_score at its 640-model limit; rf_recover_pose's decisions restated from its own cheirality bits, over stacked
candidates and every status; fundamental_8point's reductions; rf_yfcc_matches past one scan pass; and one captured CUDA graph
replayed over changing pairs.  Every buffer the kernels must not write past N is filled with 0xAB first, and rows past N hold
copies of a true inlier pair, so an over-read raises a count or moves a moment.

The only comparisons that are not exact are certified and counted: an iteration budget whose quotient lies within 1e-12
(relative) of a half-integer (CUDA's pow / log against glibc's), and a cheirality decision whose fp64 margin is below 1."""
import numpy as np
import pytest
import torch
from conftest import golden

import fundamental_oracle as FO
import pose_oracle as PO
from test_pose8_oracle import EPS
from test_pose8_oracle import points as points8

pytestmark = pytest.mark.gpu
THR = float(golden("yfcc_pose")["threshold"])
T2 = PO.thr2(THR)
G8 = golden("yfcc_pose_8point")
ITERS, BLOCK, MAXSOL = 1000, 64, 10
NBLOCKS = (ITERS + BLOCK - 1) // BLOCK
POISON = 0xAB
CAP_IMG = 480 * 640                  # H * W of the metric's 480 x 640 targets: the capacity of its real call


def dev(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def n_dev(N):
    return torch.tensor([N], dtype=torch.int32, device="cuda")


def poisoned(n):
    return torch.full((max(n, 1),), POISON, dtype=torch.uint8, device="cuda")


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def padded(p, cap, pad):
    """[max(cap, 1)][2] fp64 on the device: p, then copies of the row ``pad``."""
    out = np.tile(np.asarray(pad, dtype=np.float64), (max(cap, 1), 1))
    out[:len(p)] = p
    return dev(out)


def stage_scene(N, outlier, seed=None):
    """pose_oracle.scene with its outliers, and a true inlier pair (a row the outliers did not replace) to pad with."""
    seed = N if seed is None else seed
    p1, p2 = PO.scene(max(N, 1), outlier, seed)[:2]
    clean = PO.scene(max(N, 1), 0.0, seed)[1]
    i = int(np.nonzero(np.all(p2 == clean, axis=1))[0][0])
    return p1[:N], p2[:N], (p1[i], p2[i])


def far_scene(N, seed):
    """Every point 100 to 200 units deep, a short baseline: every triangulated depth lies beyond recoverPose's 50."""
    rs = np.random.RandomState(seed)
    X = np.c_[rs.uniform(-20, 20, (N, 2)), rs.uniform(100, 200, N)]
    X2 = X + np.array([0.3, -0.2, 0.1])
    return X[:, :2] / X[:, 2:], X2[:, :2] / X2[:, 2:]


# ------------------------------------------------------------------------------------------------ direct C ABI calls
def align256(b):
    return (b + 255) // 256 * 256


# rf_essential_ransac's workspace as include/ransacflow_b200.h documents it: four segments, each 256-byte aligned
ESS_SEGMENTS = [("idx", (ITERS, 5), torch.int32), ("candE", (ITERS, MAXSOL, 9), torch.float64), ("ncand", (ITERS,), torch.int32),
                ("counts", (ITERS, MAXSOL), torch.int32)]


def ess_segments(ws):
    out, off = {}, 0
    for name, shape, dt in ESS_SEGMENTS:
        nb = int(np.prod(shape)) * torch.tensor([], dtype=dt).element_size()
        out[name] = ws[off:off + nb].view(dt).view(shape).cpu().numpy()
        off += align256(nb)
    assert off <= ws.numel()
    return out


def ess_call(rf, P1, P2, N, cap, rec=None):
    """rf_essential_ransac with a caller-owned, 0xAB-filled workspace and mask: (record buffer, mask, workspace bytes)."""
    L, ptr = rf._lib.lib, rf._lib.ptr
    rec = rf.ops.pose_record("cuda") if rec is None else rec
    mask = poisoned(cap)
    wsz = L.rf_essential_ransac_workspace(cap)
    ws = poisoned(wsz)
    rf._lib.check(L.rf_essential_ransac(ptr(P1), ptr(P2), cap, ptr(n_dev(N)), THR, ptr(rec), ptr(mask), ptr(ws), wsz,
                                        rf._lib.stream()))
    torch.cuda.synchronize()
    return rec, mask, ws


def pose_call(rf, P1, P2, cap, mask_in, rec):
    """rf_recover_pose with 0xAB in mask_out and the workspace: (mask_out numpy, cheirality bits uint64 [cap])."""
    L, ptr = rf._lib.lib, rf._lib.ptr
    out = poisoned(cap)
    wsz = L.rf_recover_pose_workspace(cap)
    ws = poisoned(wsz)
    rf._lib.check(L.rf_recover_pose(ptr(P1), ptr(P2), cap, ptr(mask_in), ptr(rec), ptr(out), ptr(ws), wsz, rf._lib.stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), ws[:8 * cap].cpu().numpy().view(np.uint64)


# ------------------------------------------------------------------------------------------------ Sampson restatements
def sampson_torch(E, P1, P2):
    """pose_oracle.sampson as eager fp64 torch ops on the device, models E [M][9] against every row: [M][N] fp32.  Each op is
    its own kernel and rounds once, as each numpy statement does, so the bits are numpy's."""
    e = [E[:, k:k + 1] for k in range(9)]
    u1, v1, u2, v2 = P1[:, 0], P1[:, 1], P2[:, 0], P2[:, 1]
    ex0 = e[0] * u1 + e[1] * v1 + e[2]
    ex1 = e[3] * u1 + e[4] * v1 + e[5]
    ex2 = e[6] * u1 + e[7] * v1 + e[8]
    et0 = e[0] * u2 + e[3] * v2 + e[6]
    et1 = e[1] * u2 + e[4] * v2 + e[7]
    r = u2 * ex0 + v2 * ex1 + ex2
    return (r * r / (ex0 * ex0 + ex1 * ex1 + et0 * et0 + et1 * et1)).to(torch.float32)


class Sampson:
    """The fp32 Sampson errors of models over the rows of p1 / p2: pose_oracle.sampson for small N; for large N sampson_torch,
    first checked bit for bit against pose_oracle.sampson on the first and last 2048 rows of three of the models."""
    LARGE = 8192

    def __init__(self, p1, p2):
        self.p1, self.p2 = p1, p2
        self.large = len(p1) > self.LARGE
        if self.large:
            self.P1, self.P2 = dev(p1), dev(p2)
            self.rows = np.r_[0:2048, len(p1) - 2048:len(p1)]

    def device(self, E):
        """[M][N] fp32 on the device (large N)."""
        E = np.asarray(E, dtype=np.float64).reshape(-1, 9)
        out = torch.cat([sampson_torch(dev(E[s:s + 64]), self.P1, self.P2) for s in range(0, len(E), 64)])
        rows = torch.as_tensor(self.rows, device="cuda")
        for m in sorted({0, len(E) // 2, len(E) - 1}):
            np.testing.assert_array_equal(out[m][rows].cpu().numpy(), PO.sampson(E[m], self.p1[self.rows], self.p2[self.rows]))
        return out

    def errors(self, E):
        E = np.asarray(E, dtype=np.float64).reshape(-1, 9)
        if self.large:
            return self.device(E).cpu().numpy()
        return np.stack([PO.sampson(e, self.p1, self.p2) for e in E]) if len(E) else np.zeros((0, len(self.p1)), np.float32)

    def counts(self, E):
        E = np.asarray(E, dtype=np.float64).reshape(-1, 9)
        if len(E) == 0:
            return np.zeros(0, np.int64)
        if self.large:
            return np.concatenate([(self.device(E[s:s + 512]) <= float(T2)).sum(1).cpu().numpy() for s in range(0, len(E), 512)])
        return np.count_nonzero(self.errors(E) <= T2, axis=1)


# ------------------------------------------------------------------------------------------------ the replay, per launch
def quotient(N, cnt):
    """update_num_iters' num / denom (the value it rounds), or None when it does not round one."""
    ep = min(max((N - cnt) / N, 0.0), 1.0)
    denom = 1.0 - (1.0 - ep) ** 5
    if denom < np.finfo(np.float64).tiny:
        return None
    num, denom = np.log(max(1.0 - PO.CONF, np.finfo(np.float64).tiny)), np.log(denom)
    return None if denom >= 0 else float(num / denom)


def replay_blocks(N, ncand, counts, flip=None):
    """RANSACPointSetRegistrator's sequential rule, launch by launch as ess_replay_kernel runs it: (best_iter, best_cand,
    count, niters, budget before each launch, the quotients of the budget updates).  ``flip``: round that update the other
    way (a certified half-integer tie)."""
    niters, best, bi, bc = ITERS, 0, -1, -1
    before, quots = [], []
    for b in range(NBLOCKS):
        before.append(niters)
        it = b * BLOCK
        while it < min(b * BLOCK + BLOCK, ITERS) and it < niters:
            for c in range(int(ncand[it])):
                cnt = int(counts[it][c])
                if cnt > max(best, 4):
                    best, bi, bc = cnt, it, c
                    new = PO.update_num_iters(PO.CONF, (N - cnt) / N, 5, niters)
                    q = quotient(N, cnt)
                    if flip == len(quots):
                        new = int(np.floor(q)) if new == int(np.floor(q)) + 1 else int(np.floor(q)) + 1
                    quots.append(q)
                    niters = new
            it += 1
    return bi, bc, best, niters, before, quots


class Certified:
    """Counts of the certified disagreements, printed at the end of each test."""

    def __init__(self):
        self.budget = 0
        self.margin = 0

    def report(self, what):
        print("%s: certified budget ties %d, cheirality decisions with margin < 1: %d" % (what, self.budget, self.margin))


def device_replay(N, seg, rec, cert):
    """The replay on the device's candidates and counts, equal to the record's; a budget that differs only through an update
    whose quotient lies within 1e-12 of a half-integer is certified, and the restatement continues with the device's."""
    ncand, counts = seg["ncand"], seg["counts"]
    bi, bc, best, niters = PO.replay(N, ncand, counts)
    mine = replay_blocks(N, ncand, counts)
    assert mine[:4] == (bi, bc, best, niters)
    want = (rec["best"][0], rec["best"][1], rec["ransac_count"], rec["niters"])
    if mine[:4] == want:
        return mine
    ties = [k for k, q in enumerate(mine[5]) if q is not None and abs(q - np.floor(q) - 0.5) <= 1e-12 * abs(q)]
    for k in ties:
        alt = replay_blocks(N, ncand, counts, flip=k)
        if alt[:4] == want:
            cert.budget += 1
            return alt
    raise AssertionError(("replay", mine[:4], want, mine[5]))


# ------------------------------------------------------------------------------------------------ recoverPose restatement
def pose_choice(g):
    if g[0] >= g[1] and g[0] >= g[2] and g[0] >= g[3]:
        return 0
    if g[1] >= g[0] and g[1] >= g[2] and g[1] >= g[3]:
        return 1
    if g[2] >= g[0] and g[2] >= g[1] and g[2] >= g[3]:
        return 2
    return 3


def restate_pose(nE, bits, mask_in, N):
    """Every decision rf_recover_pose derives from its own cheirality bits (bit 4 c + p: pose p of candidate c) and the input
    mask over rows < N: the driver's chain (candidate c + 1 starts from candidate c's output mask; strictly greater wins).
    -> (counts [nE][4], candidate, pose, count, final mask)."""
    cur = np.asarray(mask_in[:N]) != 0
    b = bits[:N]
    best, bc, bp, final, counts = 0, -1, -1, np.zeros(N, np.uint8), []
    for c in range(nE):
        ok = [((b >> np.uint64(4 * c + p)) & np.uint64(1)).astype(bool) for p in range(4)]
        g = [int(np.count_nonzero(o & cur)) for o in ok]
        k = pose_choice(g)
        counts.append(g)
        cur = ok[k] & cur
        if g[k] > best:
            best, bc, bp, final = g[k], c, k, cur.astype(np.uint8)
    return np.array(counts, np.int64).reshape(-1, 4), bc, bp, best, final


def check_pose(rf, status_in, rec, out, bits, mask_in, N, cap):
    """rf_recover_pose's record, mask_out and bits against restate_pose; past N nothing is written."""
    ops = rf.ops
    assert np.all(out[N:cap] == POISON) and np.all(bits[N:cap] == np.uint64(0xABABABABABABABAB))
    if status_in != ops.POSE_OK:
        assert rec["status"] == status_in and rec["pose_count"] == 0 and rec["pose"] == (-1, -1)
        assert np.all(bits == np.uint64(0xABABABABABABABAB))
        np.testing.assert_array_equal(out[:N], np.zeros(N, np.uint8))     # cv2's mask= array when no count is above 0
        return
    counts, bc, bp, best, final = restate_pose(rec["n_E"], bits, mask_in, N)
    np.testing.assert_array_equal(rec["pose_counts"], counts)
    assert rec["pose"] == (bc, bp) and rec["pose_count"] == best
    assert rec["status"] == (ops.POSE_OK if bc >= 0 else ops.POSE_NO_POSE)
    if bc >= 0:
        P = rec["poses"][bc][bp]
        assert same_bits(rec["R"], P[:, :3]) and same_bits(rec["t"], P[:, 3:])
    np.testing.assert_array_equal(out[:N], final)


def check_poses_fp64(rec, bits, p1, p2, cert):
    """Each candidate's four poses against decomposeEssentialMat in fp64 (as a set, to 1e-12), and each cheirality bit against
    fp64's decision unless fp64 cannot decide it (margin < 1)."""
    for c in range(rec["n_E"]):
        ref = PO.decompose(rec["E"][c])
        for p, P in enumerate(rec["poses"][c]):
            d = [np.abs(P - Q).max() for Q in ref]
            q = int(np.argmin(d))
            assert d[q] < 1e-12, (c, p, d)
            ok_ref = PO.cheirality(ref[q], p1, p2)[0]
            ok_dev = ((bits[:len(p1)] >> np.uint64(4 * c + p)) & np.uint64(1)).astype(bool)
            diff = np.nonzero(ok_dev != ok_ref)[0]
            if len(diff):
                margin = PO.cheirality_margin(ref[q], p1[diff], p2[diff])
                assert np.all(margin < 1.0), (c, p, diff[margin >= 1.0][:5], margin[margin >= 1.0][:5])
                cert.margin += len(diff)


# ------------------------------------------------------------------------------------------------ RANSAC, stage by stage
NS = [5, 6, 7, 8, 511, 512, 513, 1023, 1024, 1025, 4097, 307199, 307200]
RATIOS = [0.0, 0.5, 0.9]
# the 307 200-point rows only where their block schedule is what they are there for
LARGE = {(307199, 0.5), (307200, 0.0), (307200, 0.5), (307200, 0.9)}
CASES = [(N, 0.0) for N in (0, 3, 4)] + [(N, r) for N in NS for r in RATIOS if N < 300000 or (N, r) in LARGE]


def capacities(N):
    return sorted({N, N + 1} | ({CAP_IMG} if CAP_IMG >= N else set()))


@pytest.mark.parametrize("N,outlier", CASES)
def test_ransac_stages_bit_exact(rf, N, outlier):
    ops = rf.ops
    cert = Certified()
    p1, p2, pad = stage_scene(N, outlier)
    runs = []
    for cap in capacities(N):
        P1, P2 = padded(p1, cap, pad[0]), padded(p2, cap, pad[1])
        rec_buf, mask, ws = ess_call(rf, P1, P2, N, cap)
        runs.append((cap, P1, P2, rec_buf, mask, ws))
    # every capacity: the same workspace, record and mask bytes over rows < N; nothing written past N
    cap0, _, _, rec0, mask0, ws0 = runs[0]
    for cap, _, _, rec_buf, mask, ws in runs:
        assert torch.equal(ws, ws0) and torch.equal(rec_buf, rec0) and torch.equal(mask[:N], mask0[:N])
        assert bool((mask[N:cap] == POISON).all())
    seg = ess_segments(ws0)
    rec = ops.read_pose_record(rec0)
    mask = mask0[:N].cpu().numpy()
    assert rec["n_points"] == N
    # the subset table
    if N > 5:
        np.testing.assert_array_equal(seg["idx"], PO.samples(N))
    elif N == 5:
        np.testing.assert_array_equal(seg["idx"][0], PO.samples(5)[0])
        assert np.all(seg["idx"][1:].view(np.uint32) == 0xABABABAB)
    else:
        assert np.all(seg["idx"].view(np.uint32) == 0xABABABAB)
    ncand = seg["ncand"]
    assert np.all((ncand >= 0) & (ncand <= MAXSOL))
    if N < 5:
        assert not ncand.any() and not seg["counts"].any()
        assert rec["status"] == ops.POSE_TOO_FEW and rec["n_E"] == 0 and rec["niters"] == ITERS and rec["best"] == (-1, -1)
        np.testing.assert_array_equal(mask, np.zeros(N, np.uint8))
    elif N == 5:
        # ess_final_kernel: the single sample's every solution, no scoring, the mask all ones when there is one
        assert not ncand[1:].any() and not seg["counts"].any()
        n = int(ncand[0])
        assert rec["n_E"] == n and same_bits(rec["E"].reshape(-1, 9), seg["candE"][0][:n])
        assert rec["status"] == (ops.POSE_OK if n else ops.POSE_NO_MODEL) and rec["ransac_count"] == (5 if n else 0)
        assert rec["niters"] == ITERS and rec["best"] == (-1, -1)
        np.testing.assert_array_equal(mask, np.full(N, 1 if n else 0, np.uint8))
    else:
        bi, bc, best, niters, before, _ = device_replay(N, seg, rec, cert)
        # the launch schedule: launch b scores iff b * 64 < the budget the launches before it left
        S = Sampson(p1, p2)
        scored = [b for b in range(NBLOCKS) if b * BLOCK < before[b]]
        counts = seg["counts"]
        for b in range(NBLOCKS):
            its = np.arange(b * BLOCK, min(b * BLOCK + BLOCK, ITERS))
            if b not in scored:
                assert not counts[its].any(), b
                continue
            models = [(it, c) for it in its for c in range(int(ncand[it]))]
            want = np.zeros((len(its), MAXSOL), np.int64)
            got_c = S.counts(np.array([seg["candE"][it][c] for it, c in models]).reshape(-1, 9))
            for (it, c), k in zip(models, got_c):
                want[it - its[0], c] = k
            np.testing.assert_array_equal(counts[its], want, err_msg="launch %d" % b)
        if N >= 511:
            # the budget regime each outlier ratio is there for: collapse in launch 0, an end inside a later launch, or
            # no shrink at all (the partial launch of iterations 960-999 runs)
            if outlier == 0.0:
                assert scored == [0]
            elif outlier == 0.5:
                assert 1 < len(scored) < NBLOCKS and niters % BLOCK != 0
            else:
                assert niters == ITERS and scored == list(range(NBLOCKS))
        if bi < 0:
            assert rec["status"] == ops.POSE_NO_MODEL and rec["n_E"] == 0
            np.testing.assert_array_equal(mask, np.zeros(N, np.uint8))
        else:
            E = seg["candE"][bi][bc]
            assert rec["status"] == ops.POSE_OK and rec["n_E"] == 1 and same_bits(rec["E"].reshape(9), E)
            np.testing.assert_array_equal(mask, (S.errors(E)[0] <= T2).astype(np.uint8))
    # recoverPose on the device's own mask (rows past N still 0xAB) in every capacity
    for k, (cap, P1, P2, rec_buf, mask_buf, _) in enumerate(runs):
        out, bits = pose_call(rf, P1, P2, cap, mask_buf, rec_buf)
        after = ops.read_pose_record(rec_buf)
        check_pose(rf, rec["status"], after, out, bits, mask_buf.cpu().numpy(), N, cap)
        if k == 0 and rec["status"] == ops.POSE_OK and N <= 4097:
            check_poses_fp64(after, bits, p1, p2, cert)
    cert.report("N = %d, %g outliers" % (N, outlier))


# ------------------------------------------------------------------------------------------------ rf_essential_score
@pytest.fixture(scope="module")
def models_640(rf):
    """640 five-point candidates of a 50 % outlier scene, from the device's five-point entry point."""
    p1, p2 = PO.scene(1025, 0.5, 3)[:2]
    idx = PO.samples(1025)[:400]
    E, n = rf.ops.essential_five_point(dev(p1), dev(p2), dev(idx, torch.int32))
    E, n = E.cpu().numpy(), n.cpu().numpy()
    Es = np.concatenate([E[k, :n[k]] for k in range(len(idx))])
    assert len(Es) >= 641
    return Es[:641]


@pytest.mark.parametrize("N", [1, 511, 512, 513, 1025, 307200])
def test_score_640_models(rf, models_640, N):
    p1, p2, pad = stage_scene(N, 0.5)
    E = models_640[:640]
    counts, err = rf.ops.essential_score(dev(p1), dev(p2), dev(E), THR, want_err=True)
    S = Sampson(p1, p2)
    if S.large:
        ref = S.device(E)
        assert torch.equal(err.view(torch.int32), ref.view(torch.int32))
        want = (ref <= float(T2)).sum(1).cpu().numpy()
    else:
        ref = S.errors(E)
        np.testing.assert_array_equal(err.cpu().numpy(), ref)
        want = np.count_nonzero(ref <= T2, axis=1)
    np.testing.assert_array_equal(counts.cpu().numpy(), want)
    with pytest.raises(rf._lib.RFError):
        rf.ops.essential_score(dev(p1), dev(p2), dev(models_640), THR)


# ------------------------------------------------------------------------------------------------ recoverPose, every status
STATUS_CASES = {
    # name: (the stage that fills the record, points, status after recoverPose); "ess" = rf_essential_ransac,
    # "f8" = rf_fundamental_8point
    "ok_single": lambda: ("ess", *stage_scene(50, 0.3, 9)[:2], "OK"),
    "ok_stacked_5": lambda: ("ess", *stage_scene(5, 0.0, 1)[:2], "OK"),
    "ok_stacked_5b": lambda: ("ess", *stage_scene(5, 0.0, 2)[:2], "OK"),
    "no_pose_stacked": lambda: ("ess", *far_scene(5, 1), "NO_POSE"),
    "no_pose_single": lambda: ("ess", *far_scene(40, 0), "NO_POSE"),
    "no_model": lambda: ("f8", *stage_scene(6, 0.0, 4)[:2], "NO_MODEL"),
    "too_few": lambda: ("ess", *stage_scene(3, 0.0, 5)[:2], "TOO_FEW"),
}
# the golden seven-point scenes with three roots: three stacked F through rf_fundamental_8point
SEVEN = [s for s in range(len(G8["scenes"])) if G8["scenes"][s][0] == 7 and G8["scenes"][s][4] == 0 and len(G8["s%d_F" % s]) == 9]


def status_case(name):
    if name.startswith("seven_"):
        p1, p2 = points8(int(name[6:]))
        return "f8", p1, p2, "OK" if bool(G8["s%s_has_pose" % name[6:]]) else "NO_POSE"
    return STATUS_CASES[name]()


@pytest.mark.parametrize("name", list(STATUS_CASES) + ["seven_%d" % s for s in SEVEN])
def test_recover_pose_every_status(rf, name):
    """recoverPose's decisions restated from its own bits over stacked candidates, per-candidate poses and bits against fp64,
    and mask_out[:N] written (0xAB before the call) whatever the status: the winner's chained mask, else zeros."""
    ops = rf.ops
    cert = Certified()
    kind, p1, p2, want = status_case(name)
    N = len(p1)
    for cap in (N, N + 1, CAP_IMG):
        P1, P2 = padded(p1, cap, (p1[0], p2[0])), padded(p2, cap, (p1[0], p2[0]))
        if kind == "ess":
            rec_buf, mask_buf, _ = ess_call(rf, P1, P2, N, cap)
        else:
            rec_buf, mask_buf = ops.fundamental_8point(P1, P2, n_dev(N))
            if N < 7:
                mask_buf.fill_(1)                          # findFundamentalMat gives no mask; any input will do
        rec = ops.read_pose_record(rec_buf)
        out, bits = pose_call(rf, P1, P2, cap, mask_buf, rec_buf)
        after = ops.read_pose_record(rec_buf)
        check_pose(rf, rec["status"], after, out, bits, mask_buf.cpu().numpy(), N, cap)
        assert after["status"] == getattr(ops, "POSE_" + want), (after["status"], want)
        if name.startswith(("ok_stacked", "no_pose_stacked", "seven_")):
            assert after["n_E"] >= 2
        if after["n_E"] and cap == N:
            check_poses_fp64(after, bits, p1, p2, cert)
        if want == "NO_POSE":
            # the scene is what it is for: the driver's loop in fp64 on the device's E keeps no pose
            rp = PO.recover_pose(after["E"].reshape(-1, 9), p1, p2, mask_buf[:N].cpu().numpy())
            assert rp[0] == 0 and all(max(g) == 0 for _, g, _ in rp[4]), [g for _, g, _ in rp[4]]
    cert.report(name)


# ------------------------------------------------------------------------------------------------ eight-point reductions
@pytest.mark.parametrize("N", NS[:-2] + [131072, 131073, 307199, 307200])
def test_fundamental_moments_capacity_and_padding(rf, N):
    p1, p2, pad = stage_scene(N, 0.5)
    c1, c2, s1, s2, A = FO.moments(FO.as_f32(p1), FO.as_f32(p2))
    ref = A[FO.IU]
    for cap in capacities(N):
        got = rf.ops.fundamental_moments(padded(p1, cap, pad[0]), padded(p2, cap, pad[1]), n_dev(N)).cpu().numpy()
        np.testing.assert_allclose(got[:4], np.r_[c1, c2], rtol=1e-15, atol=1e-15 * np.abs(np.r_[c1, c2]).max())
        np.testing.assert_allclose(got[4:6], [s1, s2], rtol=max(1e-15, 2 * np.sqrt(N) * EPS), atol=0)
        assert np.abs(got[6:] - ref).max() <= 1e-13 * np.abs(ref).max(), cap


# ------------------------------------------------------------------------------------------------ matches past one scan pass
def density_mask(H, W, density, rs):
    if density == "last":
        m = np.zeros((H, W), np.uint8)
        m[-1, -1] = 1
        return m
    return (rs.rand(H, W) < density).astype(np.uint8)


@pytest.mark.parametrize("HW", [(1024, 1024), (1024, 1025), (1031, 1033)])
@pytest.mark.parametrize("k", range(4))
def test_matches_scan_passes(rf, HW, k):
    """1024, 1025 and a partial last 1024-element tile: one scan pass, and the carry into a second."""
    H, W = HW
    hB, wB = (H, W) if k % 2 == 0 else (W, H)
    sizeA = (653, 487)
    rs = np.random.RandomState(H + W + k)
    flow = rs.uniform(-1.2, 1.2, (H, W, 2)).astype(np.float32)
    n1 = PO.norm_params((1306, 974), sizeA, np.array([[520.0, 0, 3.5], [0, 515.0, -2.0], [0, 0, 1]]))
    n2 = PO.norm_params((2 * wB + 1, 2 * hB - 1), (wB, hB), np.array([[610.0, 0, -1.5], [0, 600.0, 4.0], [0, 0, 1]]))
    F = dev(flow, torch.float32)
    for density in (0.0, 1.0, 0.5, "last"):
        mb = density_mask(H, W, density, rs)
        pts1, pts2, N = rf.ops.yfcc_matches(F, dev(mb, torch.uint8), 90 * k, sizeA, (wB, hB), n1, n2)
        N = int(N)
        r1, r2 = PO.matches_from_flow(flow.copy(), mb, sizeA, (wB, hB), 90 * k)
        r1, r2 = PO.norm_kp(n1, r1), PO.norm_kp(n2, r2)
        assert N == len(r1) == int(mb.sum()), density
        assert same_bits(pts1[:N].cpu().numpy(), r1) and same_bits(pts2[:N].cpu().numpy(), r2), density


# ------------------------------------------------------------------------------------------------ one graph, changing pairs
GH, GW = 480, 640
G_SIZE_A = (GW, GH)
G_N1 = (GW / 2 - 0.5, GH / 2 - 0.5, 500.0, 500.0)
G_N2 = (GW / 2 + 1.5, GH / 2 - 2.0, 505.0, 495.0)


def scene_flow(seed, outlier=0.3):
    """A composed flow that follows a smooth-depth two-view scene on the 480 x 640 target grid, with a fraction of pixels
    sent to random places."""
    rs = np.random.RandomState(seed)
    ys, xs = np.meshgrid(np.arange(GH, dtype=np.float64), np.arange(GW, dtype=np.float64), indexing="ij")
    cx2, cy2, fx2, fy2 = G_N2
    cx1, cy1, fx1, fy1 = G_N1
    d = 5 + 0.8 * np.sin(xs / GW * 3 + rs.rand()) + 0.6 * np.cos(ys / GH * 2 + rs.rand())
    X = np.stack([(xs - cx2) / fx2 * d, (ys - cy2) / fy2 * d, d], -1)
    ang = rs.uniform(-0.1, 0.1, 3)
    import scipy.linalg
    R = scipy.linalg.expm(np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]]))
    X = X @ R.T + rs.uniform(-0.3, 0.3, 3)
    xa, ya = fx1 * X[..., 0] / X[..., 2] + cx1, fy1 * X[..., 1] / X[..., 2] + cy1
    flow = np.stack([2 * xa / (GW - 1) - 1, 2 * ya / (GH - 1) - 1], -1)
    out = rs.rand(GH, GW) < outlier
    flow[out] = rs.uniform(-1, 1, (int(out.sum()), 2))
    return flow.astype(np.float32)


def pixels(n, seed):
    rs = np.random.RandomState(seed)
    m = np.zeros(GH * GW, np.uint8)
    m[rs.choice(GH * GW, n, replace=False)] = 1
    return m.reshape(GH, GW)


def graph_sequence(minimal):
    """(flow, mask) pairs: a dense pair, 3 matches, none, a minimal set (5 or 7 matches), a small pair, the dense pair again."""
    dense = (scene_flow(1), (np.random.RandomState(2).rand(GH, GW) < 0.7).astype(np.uint8))
    clean = scene_flow(3, outlier=0.0)
    seq = [dense, (scene_flow(4), pixels(3, 5)), (scene_flow(4), np.zeros((GH, GW), np.uint8)),
           (clean, pixels(minimal, 6)), (clean, pixels(300, 7)), dense]
    if minimal == 7:
        seq.insert(4, (clean, pixels(6, 8)))
    return seq


def compare_records(ops, g, e):
    for f in ("status", "n_points", "niters", "best", "ransac_count", "n_E", "pose_count", "pose"):
        assert g[f] == e[f], (f, g[f], e[f])
    assert same_bits(g["E"], e["E"]) and np.array_equal(g["pose_counts"], e["pose_counts"])
    if e["status"] == ops.POSE_OK:
        assert same_bits(g["R"], e["R"]) and same_bits(g["t"], e["t"])


@pytest.mark.parametrize("method", ["ransac", "8point"])
def test_graph_replay_over_changing_pairs(rf, method):
    """matches -> (findEssentialMat | findFundamentalMat) -> recoverPose captured once on fixed caller-owned buffers, replayed
    over a sequence of pairs written into the captured inputs; after each replay the results equal an eager run on fresh
    buffers.  A buffer row that one pair writes and the next does not would show here."""
    ops, L, ptr, check = rf.ops, rf._lib.lib, rf._lib.ptr, rf._lib.check
    import ctypes as C
    cap = GH * GW
    flow = torch.zeros((GH, GW, 2), dtype=torch.float32, device="cuda")
    mbuf = torch.zeros((GH, GW), dtype=torch.uint8, device="cuda")
    pts1 = torch.zeros((cap, 2), dtype=torch.float64, device="cuda")
    pts2 = torch.zeros_like(pts1)
    Nd = torch.zeros(1, dtype=torch.int32, device="cuda")
    rec = ops.pose_record("cuda")
    emask, omask = poisoned(cap), poisoned(cap)
    wsz_m = L.rf_yfcc_matches_workspace(GH, GW)
    wsz_e = L.rf_essential_ransac_workspace(cap) if method == "ransac" else L.rf_fundamental_8point_workspace(cap)
    wsz_p = L.rf_recover_pose_workspace(cap)
    ws_m, ws_e, ws_p = poisoned(wsz_m), poisoned(wsz_e), poisoned(wsz_p)
    n1, n2 = (C.c_double * 4)(*G_N1), (C.c_double * 4)(*G_N2)

    def stages():
        st = rf._lib.stream()
        check(L.rf_yfcc_matches(ptr(flow), ptr(mbuf), GH, GW, 0, GW, GH, G_SIZE_A[0], G_SIZE_A[1], n1, n2, ptr(pts1), ptr(pts2),
                                ptr(Nd), ptr(ws_m), wsz_m, st))
        if method == "ransac":
            check(L.rf_essential_ransac(ptr(pts1), ptr(pts2), cap, ptr(Nd), THR, ptr(rec), ptr(emask), ptr(ws_e), wsz_e, st))
        else:
            check(L.rf_fundamental_8point(ptr(pts1), ptr(pts2), cap, ptr(Nd), ptr(rec), ptr(emask), ptr(ws_e), wsz_e, st))
        check(L.rf_recover_pose(ptr(pts1), ptr(pts2), cap, ptr(emask), ptr(rec), ptr(omask), ptr(ws_p), wsz_p, st))

    seq = graph_sequence(5 if method == "ransac" else 7)
    flow.copy_(dev(seq[0][0], torch.float32))
    mbuf.copy_(dev(seq[0][1], torch.uint8))
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        stages()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            stages()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    seen = set()
    for step, (fl, mb) in enumerate(seq):
        F, M = dev(fl, torch.float32), dev(mb, torch.uint8)
        flow.copy_(F)
        mbuf.copy_(M)
        g.replay()
        torch.cuda.synchronize()
        # eager, fresh buffers
        e1, e2, eN = ops.yfcc_matches(F, M, 0, G_SIZE_A, (GW, GH), G_N1, G_N2)
        if method == "ransac":
            erec, emask_e = ops.essential_ransac(e1, e2, eN, THR)
        else:
            erec, emask_e = ops.fundamental_8point(e1, e2, eN)
        eout, _ = ops.recover_pose(e1, e2, emask_e, erec)
        torch.cuda.synchronize()
        N = int(eN)
        assert int(Nd) == N == int(mb.sum()), step
        gr, er = ops.read_pose_record(rec), ops.read_pose_record(erec)
        compare_records(ops, gr, er)
        assert torch.equal(pts1[:N], e1[:N]) and torch.equal(pts2[:N], e2[:N])
        if method == "ransac" or N >= 7:                   # findFundamentalMat has no mask below 7 points
            assert torch.equal(emask[:N], emask_e[:N]), step
        assert torch.equal(omask[:N], eout[:N]), (step, er["status"])
        seen.add((N if N < 8 else "many", er["status"], er["n_E"] > 1))
    # the sequence reached what it is there for: too few points, a stacked minimal case, full pairs with a pose
    assert (3, ops.POSE_TOO_FEW, False) in seen and (0, ops.POSE_TOO_FEW, False) in seen
    assert ("many", ops.POSE_OK, False) in seen
    minimal = 5 if method == "ransac" else 7
    assert any(k[0] == minimal and k[2] for k in seen), seen
