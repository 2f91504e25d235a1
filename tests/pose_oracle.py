"""numpy fp64 restatement of evalYFCC's relative-pose metric (evaluation/evalYFCC/getResults.py:29-111): the driver's
matches_from_flow / norm_kp statements, cv2.findEssentialMat(RANSAC)'s sample stream and sequential replay, and
cv2.recoverPose with the driver's loop over stacked candidates.

The five-point solver here is built independently of the CUDA kernel's: the null space comes from ``np.linalg.svd`` and the
solutions from the hidden-variable form of the ten cubic constraints (a 10 x 10 matrix polynomial in z, cubic, whose finite real
generalised eigenvalues are the roots), not from an elimination to a degree-10 polynomial."""
import itertools

import numpy as np
import scipy.linalg

ITERS = 1000
CONF = 0.999


# ----------------------------------------------------------------------------------------------------- driver statements
def norm_params(org_size, new_size, K):
    """norm_kp's (cx, cy, fx, fy), in its statement order."""
    w, h = org_size
    w_n, h_n = new_size
    cx = (w - 1.0) * 0.5
    cy = (h - 1.0) * 0.5
    cx += K[0, 2]
    cy += K[1, 2]
    fx = K[0, 0]
    fy = K[1, 1]
    cx *= (w_n / w)
    cy *= (h_n / h)
    fx *= (w_n / w)
    fy *= (h_n / h)
    return float(cx), float(cy), float(fx), float(fy)


def norm_kp(params, kp):
    cx, cy, fx, fy = params
    return (kp - np.array([[cx, cy]])) / np.array([[fx, fy]])


def matches_from_flow(flow, match_binary, sizeA, sizeB, angle):
    """getResults.py:53-71: pixel matches (pts1 fp32, pts2 int64) in boolean-index order."""
    mb = match_binary.astype(bool)
    wA, hA = sizeA
    wB, hB = sizeB
    gx, gy = np.meshgrid(np.arange(wB), np.arange(hB))
    gridB = np.rot90(np.stack((gx, gy), axis=2), angle // 90)
    pts2 = gridB[mb]
    pts1 = flow[mb]
    pts1[:, 0] = (pts1[:, 0] + 1) * (wA - 1) / 2
    pts1[:, 1] = (pts1[:, 1] + 1) * (hA - 1) / 2
    return pts1, pts2


# ------------------------------------------------------------------------------------------------------ sample stream
def samples(N, iters=ITERS):
    """cv::RNG((uint64)-1) + getSubset's redraw of repeated indices: [iters][5] int."""
    if N == 5:
        return np.arange(5)[None].repeat(1, 0)
    state = (1 << 64) - 1
    out = np.zeros((iters, 5), dtype=np.int64)
    for it in range(iters):
        i = 0
        while i < 5:
            state = ((state & 0xFFFFFFFF) * 4164903690 + (state >> 32)) & ((1 << 64) - 1)
            v = (state & 0xFFFFFFFF) % N
            out[it, i] = v
            if v not in out[it, :i]:
                i += 1
    return out


# ------------------------------------------------------------------------------------------------------ five-point
def _pmul(a, b):
    out = {}
    for (ea, ca), (eb, cb) in itertools.product(a.items(), b.items()):
        e = (ea[0] + eb[0], ea[1] + eb[1], ea[2] + eb[2])
        out[e] = out.get(e, 0.0) + ca * cb
    return out


def _padd(*ps, signs=None):
    out = {}
    for p, s in zip(ps, signs or [1.0] * len(ps)):
        for e, c in p.items():
            out[e] = out.get(e, 0.0) + s * c
    return out


XY_MONOS = [(i, j) for i in range(4) for j in range(4) if i + j <= 3]   # the ten (x, y) monomials of degree <= 3


def five_point(x1, x2, imag_tol=1e-9, return_roots=False):
    """Every real E (unit Frobenius norm, largest-magnitude entry positive) with x2^T E x1 = 0 at the five points, det E = 0 and
    2 E E^T E - tr(E E^T) E = 0, sorted by the hidden variable z.  ``return_roots``: also every finite generalised eigenvalue
    (complex included: the ten roots in z) and the null-space basis (rows X, Y, Z, W)."""
    Q = np.stack([x2[:, 0] * x1[:, 0], x2[:, 0] * x1[:, 1], x2[:, 0], x2[:, 1] * x1[:, 0], x2[:, 1] * x1[:, 1], x2[:, 1],
                  x1[:, 0], x1[:, 1], np.ones(5)], axis=1)
    basis = np.linalg.svd(Q)[2][5:]                           # 4 x 9: X, Y, Z, W
    E = [[{(1, 0, 0): basis[0, 3 * i + j], (0, 1, 0): basis[1, 3 * i + j], (0, 0, 1): basis[2, 3 * i + j],
           (0, 0, 0): basis[3, 3 * i + j]} for j in range(3)] for i in range(3)]
    eqs = []
    det = _padd(_pmul(E[0][0], _padd(_pmul(E[1][1], E[2][2]), _pmul(E[1][2], E[2][1]), signs=[1, -1])),
                _pmul(E[0][1], _padd(_pmul(E[1][0], E[2][2]), _pmul(E[1][2], E[2][0]), signs=[1, -1])),
                _pmul(E[0][2], _padd(_pmul(E[1][0], E[2][1]), _pmul(E[1][1], E[2][0]), signs=[1, -1])), signs=[1, -1, 1])
    eqs.append(det)
    EEt = [[_padd(*[_pmul(E[i][k], E[j][k]) for k in range(3)]) for j in range(3)] for i in range(3)]
    tr = _padd(EEt[0][0], EEt[1][1], EEt[2][2])
    for i in range(3):
        for j in range(3):
            t = _padd(*[_pmul(EEt[i][k], E[k][j]) for k in range(3)], signs=[2.0] * 3)
            eqs.append(_padd(t, _pmul(tr, E[i][j]), signs=[1, -1]))
    # M(z) = M0 + z M1 + z^2 M2 + z^3 M3 acting on the (x, y) monomial vector
    Ms = np.zeros((4, 10, 10))
    for r, eq in enumerate(eqs):
        for (i, j, k), c in eq.items():
            Ms[k, r, XY_MONOS.index((i, j))] += c
    n = 10
    A = np.zeros((3 * n, 3 * n))
    B = np.eye(3 * n)
    A[:n, n:2 * n] = np.eye(n)
    A[n:2 * n, 2 * n:] = np.eye(n)
    A[2 * n:, :n] = -Ms[0]
    A[2 * n:, n:2 * n] = -Ms[1]
    A[2 * n:, 2 * n:] = -Ms[2]
    B[2 * n:, 2 * n:] = Ms[3]
    w, V = scipy.linalg.eig(A, B)
    ix, iy, i1 = XY_MONOS.index((1, 0)), XY_MONOS.index((0, 1)), XY_MONOS.index((0, 0))
    sols = []
    for k in range(len(w)):
        z = w[k]
        if not np.isfinite(z) or abs(z.imag) > imag_tol * max(1.0, abs(z)):
            continue
        v = V[:n, k]
        if abs(v[i1]) < 1e-12 * np.abs(v).max():
            continue
        x, y = (v[ix] / v[i1]).real, (v[iy] / v[i1]).real
        e = x * basis[0] + y * basis[1] + z.real * basis[2] + basis[3]
        e = e / np.linalg.norm(e)
        e = e if e[np.argmax(np.abs(e))] > 0 else -e
        sols.append((z.real, e))
    sols.sort(key=lambda s: s[0])
    # a double root appears twice among the eigenvalues: keep one
    out = []
    for z, e in sols:
        if out and np.abs(out[-1][1] - e).max() < 1e-7:
            continue
        out.append((z, e))
    Es = np.array([e for _, e in out]).reshape(-1, 9)
    if return_roots:
        return Es, w[np.isfinite(w) & (np.abs(w) < 1e12)], basis
    return Es


def hidden_z(E, basis):
    """The hidden variable z of a solution E in the basis (rows X, Y, Z, W): E ~ x X + y Y + z Z + W."""
    c = basis @ np.asarray(E, dtype=np.float64).reshape(9)
    return c[2] / c[3]


def canonical(E):
    E = np.asarray(E, dtype=np.float64).reshape(-1, 9)
    E = E / np.linalg.norm(E, axis=1, keepdims=True)
    s = np.sign(E[np.arange(len(E)), np.argmax(np.abs(E), axis=1)])
    return E * s[:, None]


# --------------------------------------------------------------------------------------------------------- scoring
def sampson(E, p1, p2):
    """EMEstimatorCallback::computeError, elementwise numpy (no contraction): fp32 errors."""
    E = np.asarray(E, dtype=np.float64).reshape(9)
    u1, v1, u2, v2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    ex0 = E[0] * u1 + E[1] * v1 + E[2]
    ex1 = E[3] * u1 + E[4] * v1 + E[5]
    ex2 = E[6] * u1 + E[7] * v1 + E[8]
    et0 = E[0] * u2 + E[3] * v2 + E[6]
    et1 = E[1] * u2 + E[4] * v2 + E[7]
    r = u2 * ex0 + v2 * ex1 + ex2
    return (r * r / (ex0 * ex0 + ex1 * ex1 + et0 * et0 + et1 * et1)).astype(np.float32)


def thr2(threshold):
    return np.float32(threshold * threshold)


def update_num_iters(p, ep, model_points, max_iters):
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, np.finfo(np.float64).tiny)
    denom = 1.0 - (1.0 - ep) ** model_points
    if denom < np.finfo(np.float64).tiny:
        return 0
    num, denom = np.log(num), np.log(denom)
    return max_iters if (denom >= 0 or -num >= max_iters * (-denom)) else int(np.rint(num / denom))


def replay(N, ncand, counts):
    """RANSACPointSetRegistrator::run's sequential part: (best_iter, best_cand, best_count, niters)."""
    niters, best, bi, bc = ITERS, 0, -1, -1
    it = 0
    while it < niters:
        for c in range(int(ncand[it])):
            cnt = int(counts[it][c])
            if cnt > max(best, 4):
                best, bi, bc = cnt, it, c
                niters = update_num_iters(CONF, (N - cnt) / N, 5, niters)
        it += 1
    return bi, bc, best, niters


def essential_ransac(p1, p2, threshold, solver=five_point):
    """cv2.findEssentialMat(p1, p2, method=RANSAC, threshold): dict(E (k, 9), mask, count, niters, best) or None."""
    N = len(p1)
    if N < 5:
        return None
    if N == 5:
        E = solver(p1, p2)
        if len(E) == 0:
            return None
        return dict(E=E, mask=np.ones(5, np.uint8), count=5, niters=ITERS, best=(0, 0), cands=[E], counts=None)
    idx = samples(N)
    t2 = thr2(threshold)
    cands, counts = [], []
    niters, best, bi, bc = ITERS, 0, -1, -1
    it = 0
    while it < niters:
        E = solver(p1[idx[it]], p2[idx[it]])
        cands.append(E)
        cs = [int(np.count_nonzero(sampson(e, p1, p2) <= t2)) for e in E]
        counts.append(cs)
        for c, cnt in enumerate(cs):
            if cnt > max(best, 4):
                best, bi, bc = cnt, it, c
                niters = update_num_iters(CONF, (N - cnt) / N, 5, niters)
        it += 1
    if bi < 0:
        return None
    E = cands[bi][bc][None]
    return dict(E=E, mask=(sampson(E[0], p1, p2) <= t2).astype(np.uint8), count=best, niters=niters, best=(bi, bc),
                cands=cands, counts=counts)


# ------------------------------------------------------------------------------------------------------ recoverPose
def decompose(E):
    """decomposeEssentialMat: the four poses [R | t] in OpenCV's order (R1, t), (R2, t), (R1, -t), (R2, -t)."""
    U, _, Vt = np.linalg.svd(np.asarray(E, dtype=np.float64).reshape(3, 3))
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1]], dtype=np.float64)
    R1, R2, t = U @ W @ Vt, U @ W.T @ Vt, U[:, 2]
    return [np.hstack([R1, t[:, None]]), np.hstack([R2, t[:, None]]), np.hstack([R1, -t[:, None]]), np.hstack([R2, -t[:, None]])]


def triangulate(P, p1, p2):
    """cv::triangulatePoints with P0 = [I | 0]: the null vector of each point's 4 x 4 DLT matrix, (N, 4)."""
    P0 = np.hstack([np.eye(3), np.zeros((3, 1))])
    A = np.stack([p1[:, :1] * P0[2] - P0[0], p1[:, 1:] * P0[2] - P0[1], p2[:, :1] * P[2] - P[0], p2[:, 1:] * P[2] - P[1]], axis=1)
    return np.linalg.svd(A)[2][:, 3, :]


def cheirality(P, p1, p2, dist=50.0):
    """recoverPose's per-pose test, with the depths it compares (for certification)."""
    Q = triangulate(P, p1, p2)
    ok = Q[:, 2] * Q[:, 3] > 0
    Qn = Q / Q[:, 3:]
    ok &= Qn[:, 2] < dist
    z2 = Qn @ P[2]
    ok &= (z2 > 0) & (z2 < dist)
    return ok, Qn[:, 2], z2


def cheirality_margin(P, p1, p2, dist=50.0):
    """How far each point's cheirality decision is from flipping, in units of the error a backward-stable fp64 null vector of
    the DLT matrix can carry: the null vector moves by up to ~eps * sigma_1 / (sigma_3 - sigma_4); the tests Q2 Q3 > 0,
    0 < Z < dist and 0 < z2 < dist then move by that times their sensitivity to Q.  A margin below 1 means the decision
    is not determined by fp64 arithmetic."""
    P0 = np.hstack([np.eye(3), np.zeros((3, 1))])
    A = np.stack([p1[:, :1] * P0[2] - P0[0], p1[:, 1:] * P0[2] - P0[1], p2[:, :1] * P[2] - P[0], p2[:, 1:] * P[2] - P[1]], axis=1)
    _, S, Vt = np.linalg.svd(A)
    Q = Vt[:, 3, :]
    dQ = 64 * np.finfo(np.float64).eps * S[:, 0] / np.maximum(S[:, 2] - S[:, 3], 1e-300)
    q3 = np.maximum(np.abs(Q[:, 3]), 1e-300)
    Z = Q[:, 2] / Q[:, 3]
    z2 = (Q / Q[:, 3:]) @ P[2]
    scale = dQ * (1.0 + np.abs(Z) + np.abs(z2) + np.abs(Q[:, :3]).sum(axis=1) / q3) / q3
    m = np.abs(Q[:, 2] * Q[:, 3]) / (2 * dQ)
    for v in (Z, Z - dist, z2, z2 - dist):
        m = np.minimum(m, np.abs(v) / scale)
    return m


def recover_pose(E_stack, p1, p2, mask):
    """The driver's loop (getResults.py:96-104) over cv2.recoverPose calls, with cv2 writing each call's mask into ``mask``:
    (count, R, t, mask_final, per-candidate (poses, pose counts, choice))."""
    mask = np.asarray(mask).reshape(-1).astype(bool).copy()
    num, R, t, mfinal, info = 0, None, None, None, []
    for E in np.asarray(E_stack).reshape(-1, 9):
        poses = decompose(E)
        oks = [cheirality(P, p1, p2)[0] & mask for P in poses]
        g = [int(o.sum()) for o in oks]
        if g[0] >= g[1] and g[0] >= g[2] and g[0] >= g[3]:
            k = 0
        elif g[1] >= g[0] and g[1] >= g[2] and g[1] >= g[3]:
            k = 1
        elif g[2] >= g[0] and g[2] >= g[1] and g[2] >= g[3]:
            k = 2
        else:
            k = 3
        info.append((poses, g, k))
        mask = oks[k].copy()
        if g[k] > num:
            num, R, t, mfinal = g[k], poses[k][:, :3], poses[k][:, 3:], mask.copy()
    return num, R, t, mfinal, info


def evaluate_R_t(R_gt, t_gt, R_pred, t_pred):
    t_gt = t_gt.flatten()
    t_pred = t_pred.flatten()
    R = R_gt @ R_pred.T
    err_q = np.arccos((np.trace(R) - 1) / 2) * 180 / np.pi
    t_pred = t_pred / (np.linalg.norm(t_pred))
    t_gt = t_gt / (np.linalg.norm(t_gt))
    err_t = np.arccos(t_gt[None, :] @ t_pred[:, None]).item() * 180 / np.pi
    return err_q, err_t


def pose(p1, p2, threshold):
    """opencv_decompose(p1, p2, True, threshold) restated: ((R, t) or None, ransac result, recoverPose result)."""
    r = essential_ransac(p1, p2, threshold)
    if r is None:
        return None, None, None
    rp = recover_pose(r["E"], p1, p2, r["mask"])
    return ((rp[1], rp[2]) if rp[0] > 0 else None), r, rp


# --------------------------------------------------------------------------------------------------------- scenes
def scene(N, outlier=0.3, seed=0, noise=1e-4, planar=False):
    """Seeded two-view scene in normalised coordinates: (p1, p2, R, t)."""
    rs = np.random.RandomState(seed)
    X = rs.uniform(-1.5, 1.5, (N, 3))
    X[:, 2] = rs.uniform(3.0, 8.0, N) if not planar else 5.0 + 0.01 * rs.randn(N)
    ang = rs.uniform(-0.2, 0.2, 3)
    Kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]])
    R = scipy.linalg.expm(Kx)
    t = rs.uniform(-1, 1, 3)
    t[2] *= 0.3
    X2 = X @ R.T + t
    p1 = X[:, :2] / X[:, 2:]
    p2 = X2[:, :2] / X2[:, 2:]
    p1 = p1 + noise * rs.randn(N, 2)
    p2 = p2 + noise * rs.randn(N, 2)
    nout = int(round(outlier * N))
    if nout:
        sel = rs.choice(N, nout, replace=False)
        p2[sel] = rs.uniform(-0.6, 0.6, (nout, 2))
    return p1, p2, R, t
