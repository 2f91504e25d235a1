"""numpy fp64 restatement of the non-RANSAC branch of evalYFCC's opencv_decompose (evaluation/evalYFCC/getResults.py:75-111):
cv2.findFundamentalMat(pts1, pts2, method=cv2.FM_8POINT), in OpenCV's statement order, fed to recoverPose as if F were E.

  * the points are cast to fp32 first (findFundamentalMat's convertTo(CV_32F)); every later step is fp64;
  * N < 7: no model and no mask; N == 7: the seven-point solver (1..3 stacked candidates) whatever the method; N >= 8: the
    eight-point solver; the mask is all ones whenever N >= 7, even when the solver finds no model;
  * eight-point: centroids and mean distances by sequential sums, A = sum r r^T over the normalised points, the eigenvector of
    A's smallest eigenvalue (LAPACK eigh here), rank 2 by a 3 x 3 SVD, de-normalisation, F /= F22;
  * seven-point: the same normalisation; the null space of the 7 x 9 system in the basis OpenCV's own SVD completes it with
    (two random sign vectors of cv::RNG(0x12345678), Gram-Schmidt against the row space), the cubic det(l f1 + (1 - l) f2) = 0,
    its real roots in solveCubic's order (trigonometric case: smallest, largest, middle), F22 = 1 per root."""
import numpy as np

import pose_oracle as PO

FLT_EPSILON = float(np.finfo(np.float32).eps)
DBL_EPSILON = float(np.finfo(np.float64).eps)


def as_f32(p):
    return np.asarray(p, dtype=np.float64).astype(np.float32).astype(np.float64)


def seqsum(x):
    """x[0] + x[1] + ... left to right along axis 0 (np.cumsum accumulates sequentially), in chunks."""
    x = np.asarray(x, dtype=np.float64)
    acc = np.zeros(x.shape[1:])
    for s in range(0, len(x), 65536):
        acc = np.cumsum(np.concatenate([acc[None], x[s:s + 65536]]), axis=0)[-1]
    return acc


def normalisation(m1, m2):
    """run8Point / run7Point's centroids and scales over fp32 points (sequential fp64 sums): (m1c, m2c, scale1, scale2) or
    None when a mean distance is below FLT_EPSILON."""
    t = 1.0 / len(m1)
    c1, c2 = seqsum(m1) * t, seqsum(m2) * t
    d1, d2 = m1 - c1, m2 - c2
    s1 = seqsum(np.sqrt(d1[:, 0] * d1[:, 0] + d1[:, 1] * d1[:, 1])) * t
    s2 = seqsum(np.sqrt(d2[:, 0] * d2[:, 0] + d2[:, 1] * d2[:, 1])) * t
    if s1 < FLT_EPSILON or s2 < FLT_EPSILON:
        return None
    return c1, c2, np.sqrt(2.0) / s1, np.sqrt(2.0) / s2


def rows(m1, m2, norm):
    """The epipolar rows r = (x2 x1, x2 y1, x2, y2 x1, y2 y1, y2, x1, y1, 1) of the normalised points, (n, 9)."""
    c1, c2, s1, s2 = norm
    x1, y1 = (m1[:, 0] - c1[0]) * s1, (m1[:, 1] - c1[1]) * s1
    x2, y2 = (m2[:, 0] - c2[0]) * s2, (m2[:, 1] - c2[1]) * s2
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones_like(x1)], axis=1)


IU = np.triu_indices(9)


def moments(m1, m2):
    """(m1c, m2c, scale1, scale2, A 9 x 9) by sequential sums, or None (degenerate normalisation)."""
    norm = normalisation(m1, m2)
    if norm is None:
        return None
    A = np.zeros((9, 9))
    for s in range(0, len(m1), 65536):
        r = rows(m1[s:s + 65536], m2[s:s + 65536], norm)
        A[IU] = seqsum(np.concatenate([A[IU][None], r[:, IU[0]] * r[:, IU[1]]]))
    A = np.triu(A) + np.triu(A, 1).T
    return norm + (A,)


def transforms(norm):
    c1, c2, s1, s2 = norm
    T1 = np.array([[s1, 0, -s1 * c1[0]], [0, s1, -s1 * c1[1]], [0, 0, 1.0]])
    T2 = np.array([[s2, 0, -s2 * c2[0]], [0, s2, -s2 * c2[1]], [0, 0, 1.0]])
    return T1, T2


def run8point(m1, m2, mom=None):
    """F (3 x 3) or None, with the eigen gap (lambda_7 - lambda_8) / lambda_0 used to bound comparisons: (F, gap)."""
    mom = moments(m1, m2) if mom is None else mom
    if mom is None:
        return None, 0.0
    *norm, A = mom
    w, V = np.linalg.eigh(A)
    w, V = w[::-1], V[:, ::-1]                     # descending, as cv::eigen
    if np.any(np.abs(w[:8]) < DBL_EPSILON):
        return None, 0.0
    F0 = V[:, 8].reshape(3, 3)
    U, S, Vt = np.linalg.svd(F0)
    F0 = U @ np.diag([S[0], S[1], 0.0]) @ Vt
    T1, T2 = transforms(norm)
    F = T2.T @ F0 @ T1
    if abs(F[2, 2]) > FLT_EPSILON:
        F = F * (1.0 / F[2, 2])
    return F, float((w[7] - w[8]) / w[0])


def cv_rng_signs(count, seed=0x12345678):
    """cv::RNG(seed).next() & 256 as +-1, ``count`` draws."""
    state = seed
    out = []
    for _ in range(count):
        state = ((state & 0xFFFFFFFF) * 4164903690 + (state >> 32)) & ((1 << 64) - 1)
        out.append(1.0 if (state & 0xFFFFFFFF) & 256 else -1.0)
    return np.array(out)


def null_basis_7(A7):
    """The last two rows of OpenCV's full Vt of the 7 x 9 system: two random sign vectors (cv::RNG(0x12345678)), each
    orthogonalised twice against the row space and the vectors before it, normalised."""
    Q = np.linalg.svd(A7)[2][:7]                   # an orthonormal basis of the row space
    signs = cv_rng_signs(18).reshape(2, 9) / 9.0
    out = []
    for v in signs:
        prev = np.vstack([Q] + out)
        for _ in range(2):
            for q in prev:
                v = v - (v @ q) * q
        out.append(v / np.linalg.norm(v))
    return out


def solve_cubic(c):
    """cv::solveCubic for c[0] x^3 + c[1] x^2 + c[2] x + c[3] (c[0] != 0): the real roots in its order."""
    a1, a2, a3 = c[1] / c[0], c[2] / c[0], c[3] / c[0]
    Q = (a1 * a1 - 3 * a2) * (1.0 / 9)
    R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1.0 / 54)
    Qcubed = Q * Q * Q
    d = Qcubed - R * R
    if d > 0:
        theta = np.arccos(R / np.sqrt(Qcubed))
        t0 = -2 * np.sqrt(Q)
        t1 = theta * (1.0 / 3)
        t2 = a1 * (1.0 / 3)
        return [t0 * np.cos(t1) - t2, t0 * np.cos(t1 + 2.0 * np.pi / 3) - t2, t0 * np.cos(t1 - 2.0 * np.pi / 3) - t2]
    e = np.cbrt(np.sqrt(-d) + abs(R))
    if R > 0:
        e = -e
    return [(e + Q / e) - a1 * (1.0 / 3)]


def cubic_coeffs(f1, f2):
    """run7Point's coefficients of det(l f1 + f2) with f1 := f1 - f2 (c[0] = the l^3 coefficient)."""
    t0 = f2[4] * f2[8] - f2[5] * f2[7]
    t1 = f2[3] * f2[8] - f2[5] * f2[6]
    t2 = f2[3] * f2[7] - f2[4] * f2[6]
    c3 = f2[0] * t0 - f2[1] * t1 + f2[2] * t2
    c2 = (f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6])
          - f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) - f1[7] * (f2[0] * f2[5] - f2[2] * f2[3])
          + f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]))
    t0 = f1[4] * f1[8] - f1[5] * f1[7]
    t1 = f1[3] * f1[8] - f1[5] * f1[6]
    t2 = f1[3] * f1[7] - f1[4] * f1[6]
    c1 = (f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6])
          - f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) - f2[7] * (f1[0] * f1[5] - f1[2] * f1[3])
          + f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]))
    c0 = f1[0] * t0 - f1[1] * t1 + f1[2] * t2
    return np.array([c0, c1, c2, c3])


def run7point(m1, m2, normalise=True):
    """The stacked candidates (n, 3, 3), n = 0..3, in OpenCV's order."""
    norm = normalisation(m1, m2) if normalise else (np.zeros(2), np.zeros(2), 1.0, 1.0)
    if norm is None:
        return np.zeros((0, 3, 3))
    A7 = rows(m1, m2, norm)
    f1, f2 = null_basis_7(A7)
    f1 = f1 - f2
    c = cubic_coeffs(f1, f2)
    if c[0] == 0:
        return np.zeros((0, 3, 3))
    T1, T2 = transforms(norm)
    out = []
    for r in solve_cubic(c):
        lam, mu = r, 1.0
        s = f1[8] * r + f2[8]
        f = np.empty(9)
        if abs(s) > DBL_EPSILON:
            mu = 1.0 / s
            lam *= mu
            f[8] = 1.0
        else:
            f[8] = 0.0
        f[:8] = f1[:8] * lam + f2[:8] * mu
        F = T2.T @ f.reshape(3, 3) @ T1
        if abs(F[2, 2]) > FLT_EPSILON:
            F = F * (1.0 / F[2, 2])
        out.append(F)
    return np.array(out).reshape(-1, 3, 3)


def fundamental(p1, p2):
    """cv2.findFundamentalMat(p1, p2, method=cv2.FM_8POINT): (F stacked (3 n, 3) or None, mask (N,) u8 or None, gap)."""
    N = len(p1)
    if N < 7:
        return None, None, 0.0
    m1, m2 = as_f32(p1), as_f32(p2)
    mask = np.ones(N, np.uint8)
    if N == 7:
        F = run7point(m1, m2)
        return (F.reshape(-1, 3) if len(F) else None), mask, 1.0
    F, gap = run8point(m1, m2)
    return F, mask, gap


def opencv_decompose(p1, p2):
    """opencv_decompose(p1, p2, False, threshold) restated: ((R, t) or None, mask_final, F, recoverPose result)."""
    if len(p1) < 5:
        return None, None, None, None
    F, mask, _ = fundamental(p1, p2)
    if F is None:
        return None, None, None, None
    rp = PO.recover_pose(F.reshape(-1, 9), p1, p2, mask)
    return ((rp[1], rp[2]) if rp[0] > 0 else None), rp[3], F, rp


def golden_points(row):
    """The points of one golden scene row (N, outlier, seed, planar, kind): kind 0 = pose_oracle.scene, 1 = N copies of one
    point pair, 2 = N points on one line in each image."""
    N, outlier, seed, planar, kind = row
    N, seed, kind = int(N), int(seed), int(kind)
    if kind == 0:
        return PO.scene(N, outlier, seed, planar=bool(planar))[:2]
    if kind == 1:
        return np.tile([[0.125, -0.25]], (N, 1)), np.tile([[0.3, 0.1]], (N, 1))
    t = np.random.RandomState(seed).uniform(-1, 1, N)
    return np.stack([0.1 + 0.5 * t, -0.2 + 0.25 * t], 1), np.stack([0.3 - 0.4 * t, 0.05 + 0.6 * t], 1)
