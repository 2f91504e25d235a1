"""The RANSAC homography of utils/outil.py:117-164 restated on a supplied DLT, certified count bounds for any admissible DLT,
and the hand-built cases that reach the kernel's edges (helper of the RANSAC tests, not a test module; CPU only).

``ransac_given_H`` is the reference's RANSAC with the homography of every unique sample supplied by the caller.  Given the
kernel's own DLT output (``ops.homography_dlt``) it predicts ``ransac_kernel``'s outputs bit for bit; given LAPACK's
(``outil_oracle.Homography``) it is ``outil_oracle.RANSAC_from_samples``.  The scoring is the oracle's no-FMA
``Prediction`` and ``det3``: the oracle is this project's contract for them, whatever torch's ``bmm`` / ``det`` round to.

``certify`` bounds every hypothesis' gated inlier count over all null vectors ``geometry_ref.dlt_ref`` admits, LAPACK's and
the kernel's Householder recurrence alike.  Derivation (u = 2^-24, gamma_n = n u / (1 - n u), Higham 2nd ed. section 3.1):

1. H.  ``dlt_ref`` gives LAPACK's h and an element-wise bound b with |h' - h| <= b for every admissible fp32 output h'
   (its own rounding to fp32 included).  A row whose bound is infinite (sigma_8 <= e: numerically degenerate) or not
   below 1 (``dlt_check`` does not hold the kernel to it, the sign is free) gets the count bounds [0, M].
2. est_k = (y0 h_k0 + y1 h_k1) + y2 h_k2.  Exactly, over the box h +- b, est_k lies in c_k +- sum_j |y_j| b_kj (linear in
   h: the interval is exact).  The fp32 evaluation adds at most gamma_3 sum_j |y_j h'_kj| <= gamma_3 sum_j |y_j| (|h_kj| +
   b_kj), plus 3 * 2^-149 for underflow, and the fp64 evaluation of the centre gamma_3(2^-53) of the same sum.
3. ex = est_0 / est_2, ey = est_1 / est_2.  If the interval of est_2 holds 0 every match is ambiguous.  Otherwise the
   quotient is monotone in each argument over the box, so its range is spanned by the four corners; the fp32 division
   adds u |q|.
4. dx = x0 - ex, dx^2, dx^2 + dy^2, sqrt: each fp32 operation is one rounding, so each interval is widened by u of its
   largest magnitude (dx) or relatively by (1 +- u) (the non-negative rest), plus 2^-149 per square for underflow.  Every
   widening uses 2u instead of u, which covers the fp64 rounding of the interval arithmetic itself (2^-53 per operation).
   The result [E_lo, E_hi] holds the fp32 error of every admissible h'.  A match is a certain inlier when E_hi < tol, a
   certain outlier when E_lo >= tol (tol rounded to fp32, as the kernel and the oracle compare), ambiguous otherwise.
5. det gate.  ``det3`` is a partial-pivoting LU in fp32: L^U^ = P(H' + dA) with |dA| <= gamma_3 |L^||U^| (Higham Thm
   9.3).  |l| <= 1, and every |h'| <= 1 + 2^-22 (unit norm), so the rows of U^ are below 1.01, 2.03 and 4.1 and every
   entry of |L^||U^| is below 8: the computed det is det(H' + dA) (1 + theta_2) with |dA| <= 8 gamma_3.  Interval
   arithmetic over the box h +- (b + 8 gamma_3) (cofactor expansion; each interval product and sum is an enclosure)
   widened by gamma_2 of its magnitude and 2^-40 absolute for fp64 gives [D_lo, D_hi].  The gate (det > 1e-6 in fp32)
   passes surely when D_lo > 1e-6, fails surely when D_hi <= 1e-6, and is undecided otherwise.
6. Count bounds: gate sure to fail -> [0, 0]; sure to pass -> [certain inliers, certain + ambiguous]; undecided ->
   [0, certain + ambiguous].

Case builders take ``H_of(X, Y)``: (N, 4, 3) fp32 sources and targets -> (N, 3, 3) fp32 homographies, the DLT under which a
case is built (the kernel's in the GPU tests, LAPACK's in the CPU tests).  Each returns (match1, match2, samples, tol).
"""
import itertools

import numpy as np
import torch

import fma_ref as FR
import geometry_ref as G
from oracle import outil_oracle as OO

f32 = np.float32
OK, NONE, NO_MODEL, TOO_FEW = 0, 1, 2, 3          # RF_RANSAC_* of the library
DET_MIN = f32(1e-6)                              # utils/outil.py:113
U = G.U
ETA = 2.0 ** -149
BLOCK = 8192                                     # hypotheses per Prediction block


def unique_rows(samples):
    """Positions of the rows of ``samples`` without a repeated index (utils/outil.py:123-133 keeps these, in order)."""
    s = np.asarray(samples).reshape(-1, 4)
    dup = ((s[:, 0] == s[:, 1]) | (s[:, 0] == s[:, 2]) | (s[:, 0] == s[:, 3]) |
           (s[:, 1] == s[:, 2]) | (s[:, 1] == s[:, 3]) | (s[:, 2] == s[:, 3]))
    return np.nonzero(~dup)[0]


def lapack_H(m1, m2, samples):
    """outil_oracle.Homography of the unique rows of ``samples``: (nU, 3, 3) fp32."""
    us = np.asarray(samples)[unique_rows(samples)]
    if len(us) == 0:
        return np.zeros((0, 3, 3), f32)
    return OO.Homography(m1[us], m2[us])


def predict_fma(match1, match2, H):
    """``Prediction`` with the contractions a compiler would make: est_k = fma(y2, H_k2, fma(y1, H_k1, y0 H_k0)) and
    dx^2 + dy^2 = fma(dx, dx, dy dy).  The kernel must not compute this."""
    X = torch.from_numpy(np.asarray(match1, f32)).double()
    Y = torch.from_numpy(np.asarray(match2, f32)).double()
    Hm = torch.from_numpy(np.asarray(H, f32).reshape(-1, 9)).double()
    y0, y1, y2 = (Y[None, :, j] for j in range(3))
    e = []
    for k in range(3):
        p = (y0 * Hm[:, 3 * k, None]).float().double()
        e.append(FR.fma32(y2, Hm[:, 3 * k + 2, None], FR.fma32(y1, Hm[:, 3 * k + 1, None], p)))
    with np.errstate(all="ignore"):
        ex = (e[0].float() / e[2].float()).double()
        ey = (e[1].float() / e[2].float()).double()
        dx = (X[None, :, 0] - ex).float().double()
        dy = (X[None, :, 1] - ey).float().double()
        s = FR.fma32(dx, dx, (dy * dy).float().double())
        return torch.sqrt(s.float()).numpy()


class Rules:
    """The statements of utils/outil.py:117-164, one method each, so that a test can replace exactly one of them."""

    def errors(self, match1, match2, H):
        return OO.Prediction(match1, match2, H)                      # :97-100, fp32, no FMA

    def inliers(self, err, tol):
        return err < f32(tol)                                         # :112

    def gate(self, H):
        return OO.det3(H) > DET_MIN                                   # :113

    def chunks(self, rows, nbIter, chunk):
        """(unique positions, full chunk?) in order: chunks by rank among the unique rows (:134-160)."""
        n = len(rows)
        out = [(np.arange(c * chunk, (c + 1) * chunk), True) for c in range(n // chunk)]
        if n % chunk:
            out.append((np.arange(n // chunk * chunk, n), False))
        return out

    def pick(self, counts):
        return int(np.argmax(counts))                                 # first arg-max within a chunk

    def better(self, a, b):
        return a > b                                                  # strict across chunks (:147, :158)

    def zero_check(self, full):
        return full                                                   # the remainder chunk is not checked (:153-160)


def ransac_given_H(match1, match2, samples, tol, H_unique, chunk=100, rules=None):
    """utils/outil.py:117-164 on ``samples`` (nbIter, 4) indices with ``H_unique`` (nU, 3, 3) fp32, the homography of
    every unique row in order.  Returns a dict: status (OK / NONE / NO_MODEL; the reference returns None for NONE and raises
    TypeError for NO_MODEL), best (winning unique index or None), H (3, 3) fp32, nbInlier, mask (M,) bool, counts (nU,)
    gated per-hypothesis counts, rows (the unique rows' positions in ``samples``)."""
    rules = rules or Rules()
    match1 = np.asarray(match1, f32)
    match2 = np.asarray(match2, f32)
    rows = unique_rows(samples)
    H = np.asarray(H_unique, f32).reshape(-1, 3, 3)
    assert len(H) == len(rows)
    counts = np.zeros(len(rows), np.int64)
    for b in range(0, len(rows), BLOCK):
        Hb = H[b:b + BLOCK]
        counts[b:b + BLOCK] = rules.inliers(rules.errors(match1, match2, Hb), tol).sum(1) * rules.gate(Hb)
    out = dict(status=OK, best=None, H=np.zeros((3, 3), f32), nbInlier=0, mask=np.zeros(len(match1), bool),
               counts=counts, rows=rows)
    best, bestInlier = None, 0
    for idx, full in rules.chunks(rows, len(np.asarray(samples).reshape(-1, 4)), chunk):
        if len(idx) == 0:
            continue
        j = int(idx[rules.pick(counts[idx])])
        if rules.zero_check(full) and counts[j] == 0:
            out["status"] = NONE
            return out
        if rules.better(counts[j], bestInlier):
            best, bestInlier = j, counts[j]
    if best is None:
        out["status"] = NO_MODEL
        return out
    out.update(best=best, H=H[best].copy(), nbInlier=int(bestInlier),
               mask=rules.inliers(rules.errors(match1, match2, H[best][None])[0], tol))
    return out


# --------------------------------------------------------------------------- certification
def _imul(a, b):
    """Interval product of (lo, hi) pairs of arrays."""
    p = np.stack([a[0] * b[0], a[0] * b[1], a[1] * b[0], a[1] * b[1]])
    return p.min(0), p.max(0)


def _isub(a, b):
    return a[0] - b[1], a[1] - b[0]


def _iadd(a, b):
    return a[0] + b[0], a[1] + b[1]


def det_interval(h, r):
    """Enclosure of det over the box h +- r, (N, 9) each, by interval cofactor expansion."""
    iv = [(h[:, k] - r[:, k], h[:, k] + r[:, k]) for k in range(9)]
    a, b, c, d, e, f, g, hh, i = iv
    t0 = _imul(a, _isub(_imul(e, i), _imul(f, hh)))
    t1 = _imul(b, _isub(_imul(d, i), _imul(f, g)))
    t2 = _imul(c, _isub(_imul(d, hh), _imul(e, g)))
    return _iadd(_isub(t0, t1), t2)


def certify(match1, match2, samples, tol):
    """Count bounds of every unique hypothesis over all DLT outputs ``dlt_ref`` admits (module docstring).  Returns a dict:
    lo, hi (nU,) int; inlier, ambiguous (nU, M) bool (certain inliers, undecided matches; all of a row undecided for a
    degenerate hypothesis); gate (nU,) +1 sure to pass, -1 sure to fail, 0 undecided; tight (nU,) the rows certified
    element-wise; rows (unique positions)."""
    m1 = np.asarray(match1, f32)
    m2 = np.asarray(match2, f32)
    rows = unique_rows(samples)
    us = np.asarray(samples)[rows]
    N, M = len(rows), len(m1)
    t = float(f32(tol))
    lo = np.zeros(N, np.int64)
    hi = np.full(N, M, np.int64)
    inlier = np.zeros((N, M), bool)
    ambiguous = np.ones((N, M), bool)
    gate = np.zeros(N, np.int64)
    if N == 0:
        return dict(lo=lo, hi=hi, inlier=inlier, ambiguous=ambiguous, gate=gate, tight=np.zeros(0, bool), rows=rows)
    h, b, _ = G.dlt_ref(m1[us], m2[us])
    tight = np.isfinite(b).all(1) & (b < 1).all(1)
    X = m1.astype(np.float64)
    Y = m2.astype(np.float64)
    ay = np.abs(Y)
    for s in range(0, N, BLOCK):
        sl = slice(s, min(N, s + BLOCK))
        tt = tight[sl]
        hs, bs = h[sl][tt], b[sl][tt]
        if len(hs) == 0:
            continue
        est = []
        for k in range(3):
            hk, bk = hs[:, 3 * k:3 * k + 3], bs[:, 3 * k:3 * k + 3]
            c = hk @ Y.T                                                        # (n, M)
            mag = (np.abs(hk) + bk) @ ay.T
            rad = bk @ ay.T + G.gamma(3) * mag + G.gamma(3, G.U64) * (np.abs(hk) @ ay.T) + 3 * ETA
            est.append((c - rad, c + rad))
        zero = (est[2][0] <= 0) & (est[2][1] >= 0)
        with np.errstate(all="ignore"):
            E = []
            for k in range(2):
                q = np.stack([est[k][i] / est[2][j] for i in (0, 1) for j in (0, 1)])
                qlo, qhi = q.min(0), q.max(0)
                w = 2 * U * np.maximum(np.abs(qlo), np.abs(qhi))
                dlo, dhi = X[None, :, k] - (qhi + w), X[None, :, k] - (qlo - w)
                w = 2 * U * np.maximum(np.abs(dlo), np.abs(dhi))
                dlo, dhi = dlo - w, dhi + w
                sq_hi = np.maximum(dlo * dlo, dhi * dhi)
                sq_lo = np.where((dlo <= 0) & (dhi >= 0), 0.0, np.minimum(dlo * dlo, dhi * dhi))
                E.append((sq_lo * (1 - 2 * U) - ETA, sq_hi * (1 + 2 * U) + ETA))
            slo = np.maximum((E[0][0] + E[1][0]) * (1 - 2 * U), 0.0)
            shi = (E[0][1] + E[1][1]) * (1 + 2 * U)
            elo, ehi = np.sqrt(slo) * (1 - 2 * U), np.sqrt(shi) * (1 + 2 * U)
        sure_in = ~zero & (ehi < t)
        sure_out = ~zero & (elo >= t)
        idx = np.arange(sl.start, sl.stop)[tt]
        inlier[idx] = sure_in
        ambiguous[idx] = ~(sure_in | sure_out)
        dl, dh = det_interval(hs, bs + 8 * G.gamma(3))
        wd = G.gamma(2) * np.maximum(np.abs(dl), np.abs(dh)) + 2.0 ** -40
        dl, dh = dl - wd, dh + wd
        dmin = float(DET_MIN)
        gate[idx] = np.where(dl > dmin, 1, np.where(dh <= dmin, -1, 0))
        nin, namb = sure_in.sum(1), (~(sure_in | sure_out)).sum(1)
        lo[idx] = np.where(dl > dmin, nin, 0)
        hi[idx] = np.where(dh <= dmin, 0, nin + namb)
    return dict(lo=lo, hi=hi, inlier=inlier, ambiguous=ambiguous, gate=gate, tight=tight, rows=rows)


def outcome_bounds(cert):
    """The score (nbInlier) every admissible DLT can give when no chunk is zero: the largest count, in [max lo, max hi]."""
    return int(cert["lo"].max(initial=0)), int(cert["hi"].max(initial=0))


# --------------------------------------------------------------------------- cases
def _rows3(xy):
    xy = np.asarray(xy, np.float64)
    return np.concatenate([xy, np.ones((len(xy), 1))], 1).astype(f32)


def _project(H, y):
    """fp64 x = H y (dehomogenised), y (N, 2)."""
    p = _rows3(y).astype(np.float64) @ np.asarray(H, np.float64).T
    return p[:, :2] / p[:, 2:]


def _quad(rs, lo=-0.8, hi=0.8):
    """Four points of a well-conditioned quadrilateral (a jittered square)."""
    base = np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]], np.float64) * 0.6
    return np.clip(base + rs.uniform(-0.1, 0.1, (4, 2)), lo, hi)


def _outliers(rs, n, H, tol, avoid=3.0):
    """n random matches whose fp64 error under H exceeds ``avoid`` tol: far from any decision."""
    out1, out2 = [], []
    while len(out1) < n:
        y = rs.uniform(-1, 1, (4 * n, 2))
        x = rs.uniform(-1, 1, (4 * n, 2))
        with np.errstate(all="ignore"):
            far = np.linalg.norm(x - _project(H, y), axis=1) > avoid * tol
        out1 += list(x[far])
        out2 += list(y[far])
    return _rows3(out1[:n]), _rows3(out2[:n])


def boundary_case(H_of, seed=0, tol=0.05, per_kind=6):
    """Matches whose fp32 error under the provider's H of the first sample (matches 0..3) is exactly tol, one ulp below it
    or one ulp above it, and matches where the FMA evaluation (``predict_fma``) and the plain one fall on opposite sides of
    tol; plus 40 far outliers and 30 random samples of the outliers.  The first sample wins, so its mask shows every
    boundary match."""
    rs = np.random.RandomState(seed)
    ys = _quad(rs)
    Hgt = np.array([[1.05, 0.04, 0.02], [-0.03, 0.97, -0.01], [0.03, -0.02, 1.0]])
    xs = _project(Hgt, ys)
    X4, Y4 = _rows3(xs), _rows3(ys)
    H = np.asarray(H_of(X4[None], Y4[None]), f32)[0]
    t = f32(tol)
    want = {"eq": t, "below": np.nextafter(t, f32(0)), "above": np.nextafter(t, f32(1))}
    found = {k: [] for k in list(want) + ["fma"]}
    for _ in range(200):
        # targets whose fp32 prediction ex is small, so x0 = ex +- tol lies in tol's binade and each ulp step of x0 moves
        # the error by one ulp of tol
        y = rs.uniform(-1, 1, (4096, 2))
        Y = _rows3(y)
        e = [(Y[:, 0] * H[k, 0] + Y[:, 1] * H[k, 1]) + Y[:, 2] * H[k, 2] for k in range(3)]
        ex, ey = e[0] / e[2], e[1] / e[2]
        ok = np.abs(ex) < 4e-3
        for j in np.nonzero(ok)[0][:64]:
            for sgn in (1, -1):
                x0 = f32(ex[j] + sgn * t)
                cand = [x0]
                for _ in range(4):
                    cand = [np.nextafter(cand[0], f32(-1))] + cand + [np.nextafter(cand[-1], f32(1))]
                m1 = _rows3(np.stack([np.array(cand, np.float64), np.full(len(cand), float(ey[j]))], 1))
                m2 = np.repeat(Y[j:j + 1], len(cand), 0)
                err = OO.Prediction(m1, m2, H[None])[0]
                errf = predict_fma(m1, m2, H[None])[0]
                for c in range(len(cand)):
                    for k, v in want.items():
                        if err[c] == v and len(found[k]) < per_kind:
                            found[k].append((m1[c], m2[c]))
                    if (err[c] < t) != (errf[c] < t) and len(found["fma"]) < per_kind:
                        found["fma"].append((m1[c], m2[c]))
                # dy != 0: x1 one tol-ish away too, a second chance for the contraction to matter
                m1b = m1.copy()
                m1b[:, 1] = f32(ey[j] + sgn * f32(0.03))
                err = OO.Prediction(m1b, m2, H[None])[0]
                errf = predict_fma(m1b, m2, H[None])[0]
                for c in range(len(cand)):
                    if (err[c] < t) != (errf[c] < t) and len(found["fma"]) < per_kind:
                        found["fma"].append((m1b[c], m2[c]))
        if all(len(v) >= per_kind for v in found.values()):
            break
    for k, v in found.items():
        assert v, "boundary case: no match of kind %r found" % k
    b1 = np.array([p[0] for v in found.values() for p in v], f32)
    b2 = np.array([p[1] for v in found.values() for p in v], f32)
    o1, o2 = _outliers(rs, 40, Hgt, tol)
    m1 = np.concatenate([X4, b1, o1])
    m2 = np.concatenate([Y4, b2, o2])
    no = len(o1)
    first = len(m1) - no
    others = first + np.stack([rs.choice(no, 4, replace=False) for _ in range(30)])
    samples = np.concatenate([[[0, 1, 2, 3]], others]).astype(np.int64)
    return m1, m2, samples, tol


def tie_case(H_of, seed=1, tol=0.05, repeat=5):
    """The same four points in all 24 orders, ``repeat`` times over (24 repeat > 100 rows: a full chunk and a remainder):
    the four sample points and 30 outliers far from all 24 homographies, so every order counts the same (4), while the H
    bits of the orders differ.  On a well-conditioned quadrilateral the orders' fp64 null vectors round to the same fp32
    bits, so the quadrilateral is nearly degenerate (one corner within eps of the diagonal, sigma_8 ~ eps): the orders'
    rounding differences grow by 1 / eps and reach fp32.  The order table puts orders whose H bits differ from the first
    one's at the last row of the full chunk and the first of the remainder, so that the returned H shows which row won."""
    rs = np.random.RandomState(seed)
    Hgt = np.array([[0.9, 0.1, 0.05], [0.05, 1.1, -0.05], [0.02, 0.03, 1.0]])
    perms = np.array(list(itertools.permutations(range(4))), np.int64)
    for _ in range(200):
        ys = _quad(rs)
        eps = 10.0 ** -rs.uniform(3, 6)
        ys[1] = (ys[0] + ys[2]) / 2 + eps * rs.uniform(-1, 1, 2)
        X4, Y4 = _rows3(_project(Hgt, ys)), _rows3(ys)
        H = np.asarray(H_of(X4[perms], Y4[perms]), f32).reshape(24, 9)
        differ = [i for i in range(1, 24) if not np.array_equal(H[i].view(np.int32), H[0].view(np.int32))]
        if len(differ) >= 2 and (OO.det3(H.reshape(24, 3, 3)) > DET_MIN).all():
            break
    else:
        raise AssertionError("tie case: no quadrilateral whose 24 orders give 3 distinct H under this DLT")
    o1, o2 = [], []
    while len(o1) < 30:
        x, y = _rows3(rs.uniform(-1, 1, (1, 2))), _rows3(rs.uniform(-1, 1, (1, 2)))
        if (OO.Prediction(x, y, H.reshape(24, 3, 3)) > 3 * tol).all():
            o1.append(x[0]), o2.append(y[0])
    m1 = np.concatenate([X4, np.array(o1)])
    m2 = np.concatenate([Y4, np.array(o2)])
    assert 24 * repeat > 100 and 99 % 24 + 1 == 100 % 24
    order = [0] + [i for i in range(1, 24) if i not in differ[:2]]
    order.insert(99 % 24, differ[0])                  # raw row 99: the last of the full chunk
    order.insert(100 % 24, differ[1])                 # raw row 100: the first of the remainder
    samples = np.tile(perms[order], (repeat, 1))
    return m1, m2, samples, tol


def _good_and_reflected(H_of, rs, tol, n_good=24, n_refl=40):
    """Matches 0 .. n_good - 1 on a homography (noise-free inliers of each other), then n_refl matches on a reflection.
    Returns (m1, m2, good quadruples (K, 4), gated reflection quadruples (K', 4)): the latter are quadruples whose H under
    the provider has det3 <= 1e-6 (the gate drops them; their 4 points alone would count)."""
    Hg = np.array([[1.0, 0.05, 0.02], [-0.04, 0.95, 0.03], [0.01, 0.02, 1.0]])
    R = np.array([[-0.9, 0.1, 0.05], [0.08, 1.05, -0.02], [0.0, 0.02, 1.0]])       # det < 0: a reflection
    yg = rs.uniform(-0.9, 0.9, (n_good, 2))
    yr = rs.uniform(-0.9, 0.9, (n_refl, 2))
    m1 = _rows3(np.concatenate([_project(Hg, yg), _project(R, yr)]))
    m2 = _rows3(np.concatenate([yg, yr]))
    good = np.stack([rs.choice(n_good, 4, replace=False) for _ in range(600)]).astype(np.int64)
    good = good[OO.det3(np.asarray(H_of(m1[good], m2[good]), f32)) > DET_MIN]      # the null vector's sign is the DLT's
    cand = n_good + np.stack([rs.choice(n_refl, 4, replace=False) for _ in range(4000)]).astype(np.int64)
    gated = cand[~(OO.det3(np.asarray(H_of(m1[cand], m2[cand]), f32)) > DET_MIN)]
    assert len(good) >= 300 and len(gated) >= 150, "too few quadruples of either kind under this DLT"
    return m1, m2, good, gated


def late_zero_case(H_of, seed=2, tol=0.05, remainder=False):
    """Two chunks of good hypotheses, then 100 det-gated reflection hypotheses: a full zero chunk after good ones (status
    NONE).  ``remainder``: the gated block is a 50-row remainder instead (status OK: the remainder is not checked)."""
    rs = np.random.RandomState(seed)
    m1, m2, good, gated = _good_and_reflected(H_of, rs, tol)
    z = gated[:50] if remainder else np.concatenate([gated[:100], good[200:230]])
    return m1, m2, np.concatenate([good[:200], z]), tol


def duplicate_case(H_of, seed=3, tol=0.05):
    """Raw rows 0..99: 50 rows with a repeated index and 50 det-gated hypotheses; rows 100..199: good hypotheses.  By rank
    among the unique rows the first chunk holds the 50 gated and 50 good ones (status OK); chunks of raw indices would make
    rows 0..99 a zero chunk."""
    rs = np.random.RandomState(seed)
    m1, m2, good, gated = _good_and_reflected(H_of, rs, tol)
    dup = rs.randint(0, len(m1), (50, 4))
    dup[:, 3] = dup[:, rs.randint(0, 3)]
    head = np.concatenate([dup, gated[:50]])
    head = head[rs.permutation(100)]
    return m1, m2, np.concatenate([head, good[:100]]).astype(np.int64), tol


def degenerate_case(H_of=None, seed=4, tol=0.05, h16=30, w16=40):
    """Matches on a 16-pixel feature grid (getWHTensor cell centres) related by a shift of whole cells, and samples of four
    collinear cells (one row, one column, a diagonal) mixed with random ones: a (nearly) two-dimensional null space where
    the DLT's answer is not determined.  ``H_of`` is unused (the case is the same under every DLT)."""
    rs = np.random.RandomState(seed)
    W, Hc = OO.getWHTensor(h16, w16)                  # W: rows (y), Hc: columns (x), flattened row-major
    M = 200
    r = rs.randint(0, h16 - 3, M)
    c = rs.randint(0, w16 - 3, M)
    tgt = r * w16 + c
    src = (r + 1) * w16 + (c + 2)
    m2 = np.stack([Hc[tgt], W[tgt], np.ones(M, f32)], 1).astype(f32)
    m1 = np.stack([Hc[src], W[src], np.ones(M, f32)], 1).astype(f32)
    out = rs.permutation(M)[:60]
    m1[out, :2] = np.stack([Hc[rs.randint(0, h16 * w16, 60)], W[rs.randint(0, h16 * w16, 60)]], 1)
    rows = []
    for key in (r, c, r - c):
        for v in np.unique(key):
            idx = np.nonzero(key == v)[0]
            # distinct cells on one line
            _, first = np.unique(tgt[idx], return_index=True)
            idx = idx[first]
            if len(idx) >= 4:
                rows.append(rs.choice(idx, 4, replace=False))
    rand = np.stack([rs.choice(M, 4, replace=False) for _ in range(300 - len(rows))])
    samples = np.concatenate([np.array(rows, np.int64).reshape(-1, 4), rand])[rs.permutation(300)].astype(np.int64)
    return m1, m2, samples, tol


BUILDERS = {"boundary": boundary_case, "tie": tie_case, "late_zero": late_zero_case,
            "zero_remainder": lambda H_of: late_zero_case(H_of, remainder=True), "duplicates": duplicate_case,
            "degenerate": degenerate_case}


def lapack_provider(X, Y):
    return OO.Homography(X, Y)
