"""fp64 references, with element-wise error allowances, for the kernels after the correlation: the homography grid
(warp_grid_kernel), bilinear sampling (grid_sample_kernel), bilinear resizing (upsample_kernel), the fused composition
(compose_fine_kernel), the match gather (build_matches_kernel) and the 4-point DLT (dlt_kernel).

Every reference reads the fp32 values the kernel reads and evaluates the operation in fp64.  Every allowance follows from
the kernel's fp32 arithmetic, u = 2^-24 and gamma_n = n u / (1 - n u) (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., section 3.1); none is measured.  Each allowance is a multiple of u with a small explicit constant, so
a kernel that carries any intermediate in fp16 or bf16 (relative error 2^-11 or 2^-8) fails it.

Bilinear sampling with zero padding is continuous and piecewise linear in the sample position.  A coordinate error of
delta_x source pixels therefore moves the value by at most Lx * delta_x, where Lx is the largest |difference| between
horizontally adjacent input values (zero padding included) in the cells within one pixel of the sample; the same holds
for y.  This also covers a cell flip at an integer coordinate.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import outil_oracle as OO

U = 2.0 ** -24
U64 = 2.0 ** -53
f32 = np.float32


def gamma(n, u=U):
    return n * u / (1 - n * u)


# --------------------------------------------------------------------------- homography grid
def lin11(i, n):
    """torch.linspace(-1, 1, n)[i] as the kernel computes it: step = 2 / (n - 1) (IEEE division), then two branches
    meeting at n / 2, each ONE fused multiply-add (the compiled code contracts `-1 + step * i` and `1 - step * (n-1-i)`).
    The fp64 product of a float32 step and an integer below 2^24 is exact and so is its sum with -1 / +1 (at most 48
    significant bits), so rounding that sum to float32 once is the FMA."""
    i = np.asarray(i, dtype=np.int64)
    if n == 1:
        return np.full(i.shape, -1.0, dtype=f32)
    step = float(f32(2.0) / f32(n - 1))
    lo = (i.astype(np.float64) * step - 1.0).astype(f32)
    hi = (1.0 - (n - 1 - i).astype(np.float64) * step).astype(f32)
    return np.where(i < n // 2, lo, hi).astype(f32)


def warp_grid_f32(Hm, h, w):
    """(N, 3, 3) float32 -> (N, h, w, 2) float32: the kernel's exact IEEE sequence, one rounding per operation,
    ((H0 x + H1 y) + H2) / ((H6 x + H7 y) + H8) with x = lin11(c, w), y = lin11(r, h).  No epsilon on the division
    (kornia 0.1.4): pz = 0 gives +-inf or NaN, as on the device."""
    Hm = np.asarray(Hm, dtype=f32).reshape(-1, 9)
    x = lin11(np.arange(w), w)[None, None, :]
    y = lin11(np.arange(h), h)[None, :, None]
    c = [Hm[:, k][:, None, None] for k in range(9)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        px = (c[0] * x + c[1] * y) + c[2]
        py = (c[3] * x + c[4] * y) + c[5]
        pz = (c[6] * x + c[7] * y) + c[8]
        return np.stack(np.broadcast_arrays(px / pz, py / pz), -1).astype(f32)


# --------------------------------------------------------------------------- bilinear sampling
def unnormalize64(g, size, align_corners):
    """The source pixel coordinate of a normalised grid value, in fp64."""
    g = np.asarray(g, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (g + 1.0) / 2.0 * (size - 1) if align_corners else ((g + 1.0) * size - 1.0) / 2.0


def coord_delta(ix):
    """Bound on the kernel's fp32 error in the source coordinate, in pixels, for g a float32 grid value.
    align_corners=False: t = fl(g + 1), then fl(t * size - 1) (fused or not), then an exact halving: the three roundings
    give at most u|g + 1| size (1 + u) + u |t size - 1| + u |t size| <= 2u(2|ix| + 1) + u(2|ix| + 1) over 2, i.e.
    3u|ix| + 1.5u.  align_corners=True: fl(g + 1) * 0.5 (exact) * (size - 1) rounded: gamma_2 |ix|.  4u(|ix| + 1) covers
    both and the fp64 evaluation of the reference itself."""
    return 4.0 * U * (np.abs(ix) + 1.0)


def _window_max(M, y0, x0, rows, cols, pad):
    """max of M (C, Hp, Wp) over rows y0 + rows, cols x0 + cols (indices into the unpadded image; clipped to the padded
    border, which is zero in every map this is used on)."""
    Hp, Wp = M.shape[1], M.shape[2]
    out = None
    for dy in rows:
        yi = np.clip(y0 + dy + pad, 0, Hp - 1)
        for dx in cols:
            xi = np.clip(x0 + dx + pad, 0, Wp - 1)
            v = M[:, yi, xi]
            out = v if out is None else np.maximum(out, v)
    return out


def bilinear_zeros(P, ix, iy):
    """Bilinear sampling with zero padding of P (C, Hin, Win) at fp64 pixel coordinates ix, iy (any shape S), as
    torch's CUDA grid sampler defines it: a coordinate that is not finite or lies beyond the int range (|c| >= 2^31)
    is moved outside the image (`safe_downgrade_to_int_range`), so it samples nothing.
    Returns (val, absval, Lx, Ly, outside), the first four of shape (C,) + S: the value, the same on |P|, and the local
    horizontal / vertical Lipschitz constants (see the module docstring); ``outside`` marks the downgraded coordinates."""
    P = np.asarray(P, dtype=np.float64)
    C, Hin, Win = P.shape
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(ix) & np.isfinite(iy) & (np.abs(ix) < 2.0 ** 31) & (np.abs(iy) < 2.0 ** 31)
    ix = np.where(ok, ix, -100.0)
    iy = np.where(ok, iy, -100.0)
    fx, fy = np.floor(ix), np.floor(iy)
    x0 = np.clip(fx, -2 ** 40, 2 ** 40).astype(np.int64)
    y0 = np.clip(fy, -2 ** 40, 2 ** 40).astype(np.int64)
    wx1, wy1 = ix - fx, iy - fy
    wx0, wy0 = 1.0 - wx1, 1.0 - wy1
    pad = 4
    Pp = np.zeros((C, Hin + 2 * pad, Win + 2 * pad))
    Pp[:, pad:pad + Hin, pad:pad + Win] = P
    Ap = np.abs(Pp)

    def at(M, dy, dx):
        yi = np.clip(y0 + dy + pad, 0, M.shape[1] - 1)
        xi = np.clip(x0 + dx + pad, 0, M.shape[2] - 1)
        return M[:, yi, xi]

    val = wy0 * (wx0 * at(Pp, 0, 0) + wx1 * at(Pp, 0, 1)) + wy1 * (wx0 * at(Pp, 1, 0) + wx1 * at(Pp, 1, 1))
    absval = wy0 * (wx0 * at(Ap, 0, 0) + wx1 * at(Ap, 0, 1)) + wy1 * (wx0 * at(Ap, 1, 0) + wx1 * at(Ap, 1, 1))
    DX = np.zeros_like(Pp)
    DX[:, :, :-1] = np.abs(np.diff(Pp, axis=2))          # DX[.., x] = |P[.., x + 1] - P[.., x]|
    DY = np.zeros_like(Pp)
    DY[:, :-1, :] = np.abs(np.diff(Pp, axis=1))
    Lx = _window_max(DX, y0, x0, (-1, 0, 1, 2), (-1, 0, 1), pad)
    Ly = _window_max(DY, y0, x0, (-1, 0, 1), (-1, 0, 1, 2), pad)
    return val, absval, Lx, Ly, ~ok


def grid_sample_ref(inp, grid, align_corners):
    """F.grid_sample(inp, grid, bilinear, zeros) in fp64 at the fp64 coordinates of the float32 grid.
    inp (N, C, Hin, Win), grid (N, Hout, Wout, 2).  Returns (ref, allowance, outside), ref and allowance (N, C, Hout, Wout).

    Allowance = gamma_7 absref + Lx delta_x + Ly delta_y.  gamma_7: each weight is a product of two differences
    (fx + 1 - ix, ix - fx, each rounded at most once) rounded once, times the value (one rounding, or none when fused),
    summed over at most four terms (three additions): seven roundings per term, relative to sum |v| w = absref.
    delta: ``coord_delta``.  Outside coordinates (non-finite, |c| >= 2^31) have ref = 0 and allowance 0: the kernel
    must return exactly 0 there, as torch's CUDA F.grid_sample does."""
    inp = np.asarray(inp, dtype=np.float64)
    g = np.asarray(grid, dtype=np.float64)
    N, C, Hin, Win = inp.shape
    refs, allows, outs = [], [], []
    for n in range(N):
        ix = unnormalize64(g[n, ..., 0], Win, align_corners)
        iy = unnormalize64(g[n, ..., 1], Hin, align_corners)
        val, absval, Lx, Ly, outside = bilinear_zeros(inp[n], ix, iy)
        with np.errstate(invalid="ignore"):
            allow = gamma(7) * absval + Lx * coord_delta(np.where(outside, 0, ix)) + Ly * coord_delta(np.where(outside, 0, iy))
        allow = np.where(outside[None], 0.0, allow)
        refs.append(val), allows.append(allow), outs.append(outside)
    return np.stack(refs), np.stack(allows), np.stack(outs)


# --------------------------------------------------------------------------- bilinear resizing
def up_source(out_size, in_size):
    """F.interpolate(bilinear, align_corners=False) source coordinate per output index, in fp64: max(0, s (d + 0.5) - 0.5)
    with s = in / out, and its fp32 error bound: fl(in / out) is off by u relatively, the product with the exact d + 0.5
    and the subtraction of 0.5 (fused or not) add at most two more roundings, so |src_f - src| <= gamma_2 (src + 0.5) +
    u |src| <= 4u (src + 1); the clamp at 0 is 1-Lipschitz."""
    d = np.arange(out_size, dtype=np.float64)
    src = np.maximum(in_size / out_size * (d + 0.5) - 0.5, 0.0)
    return src, 4.0 * U * (src + 1.0)


def upsample_ref(x, H, W):
    """F.interpolate(x, (H, W), bilinear, align_corners=False) in fp64 (torch CPU float64), x (NC, h, w) float32 values.
    Returns (ref, allowance), both (NC, H, W).

    Allowance = gamma_6 absref + Lx delta_x + Ly delta_y.  gamma_6: l1 = src - trunc(src) is exact (Sterbenz), l0 = 1 - l1
    is rounded once; each term ly * (lx * v) carries the two l0 roundings and four operation roundings (two products, the
    inner sum, the outer product; the outer sum is the fourth for the second half), relative to absref = the same
    interpolation of |x|.  delta: ``up_source``.  Lx is the largest |horizontal difference| of x in the cells within one
    pixel (edge-clamped, as the kernel clamps i1 at the border)."""
    x = np.asarray(x, dtype=np.float64)
    NC, h, w = x.shape
    t = torch.from_numpy(x)[None]
    ref = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=False)[0].numpy()
    absref = F.interpolate(t.abs(), size=(H, W), mode="bilinear", align_corners=False)[0].numpy()
    sy, dy = up_source(H, h)
    sx, dx = up_source(W, w)
    y0 = np.floor(sy).astype(np.int64)[:, None] * np.ones((1, W), np.int64)
    x0 = np.floor(sx).astype(np.int64)[None, :] * np.ones((H, 1), np.int64)
    pad = 4
    DX = np.zeros((NC, h + 2 * pad, w + 2 * pad))
    DY = np.zeros((NC, h + 2 * pad, w + 2 * pad))
    DX[:, pad:pad + h, pad:pad + w - 1] = np.abs(np.diff(x, axis=2))
    DY[:, pad:pad + h - 1, pad:pad + w] = np.abs(np.diff(x, axis=1))
    Lx = _window_max(DX, y0, x0, (-1, 0, 1, 2), (-1, 0, 1), pad)
    Ly = _window_max(DY, y0, x0, (-1, 0, 1), (-1, 0, 1, 2), pad)
    allow = gamma(6) * absref + Lx * dx[None, None, :] + Ly * dy[None, :, None]
    return ref, allow


# --------------------------------------------------------------------------- fused composition
def compose_fine_ref(flow8, m12, m21, coarse, H, W, clamp=True, align_corners=False):
    """The chain compose_fine_kernel fuses, in fp64, with propagated allowances.
    flow8 (2, h8, w8), m12 / m21 (h8, w8) or None, coarse (Hc, Wc, 2): float32 values.

    1. flowUp = upsample(flow8, (H, W)) + lin11 (the kernel's float32 base grid): allowance e = a_up (1 + u) + u |flowUp|
       (one rounding for the addition).
    2. clamp to [-1, 1] (1-Lipschitz; where the unclamped value is beyond +-1 by more than e both sides clamp to exactly
       +-1 and e becomes 0).
    3. flow12 = grid_sample(coarse, flowUp) at the coarse grid's own (Hc, Wc): an error e in normalised coordinates moves
       the sample by e Wc / 2 pixels (e (Wc - 1) / 2 with align_corners), added to ``coord_delta``; the sampling itself
       adds gamma_7 absref as in ``grid_sample_ref``.
    4. match = upsample(m12, (H, W)), times grid_sample(upsample(m21, (H, W)), flowUp) when m21 is given: the sampled
       corners carry their own upsampling allowance (the weights sum to 1), the product a_m |mm| + a_mm |m| + a_m a_mm plus
       one rounding.
    5. times the inside mask (|flow12.x| <= 1 and |flow12.y| <= 1).  The mask is decided wherever each component of the
       reference flow12 is farther from +-1 than its allowance; ``decided`` marks those pixels.
    Returns a dict of fp64 arrays: flowUp / a_flowUp (H, W, 2), flow12 / a_flow12 (H, W, 2), inside, decided (H, W),
    match / a_match (H, W) (without the mask; None without m12)."""
    flow8 = np.asarray(flow8, dtype=np.float64)
    up, a_up = upsample_ref(flow8, H, W)
    base = np.stack(np.broadcast_arrays(lin11(np.arange(W), W)[None, :].astype(np.float64),
                                        lin11(np.arange(H), H)[:, None].astype(np.float64)), 0)
    fu = up + base
    e = a_up * (1 + U) + U * np.abs(fu)
    if clamp:
        surely = np.abs(fu) - 1.0 > e
        fu = np.clip(fu, -1.0, 1.0)
        e = np.where(surely, 0.0, e)
    coarse = np.asarray(coarse, dtype=np.float64)
    Hc, Wc = coarse.shape[0], coarse.shape[1]

    def sample(P, Hs, Ws):
        ix = unnormalize64(fu[0], Ws, align_corners)
        iy = unnormalize64(fu[1], Hs, align_corners)
        sx = (Ws - 1) / 2.0 if align_corners else Ws / 2.0
        sy = (Hs - 1) / 2.0 if align_corners else Hs / 2.0
        val, absval, Lx, Ly, _ = bilinear_zeros(P, ix, iy)
        dx = coord_delta(np.abs(ix) + sx * e[0]) + sx * e[0]
        dy = coord_delta(np.abs(iy) + sy * e[1]) + sy * e[1]
        return val, gamma(7) * absval + Lx * dx + Ly * dy, (ix, iy)

    o, a_o, _ = sample(coarse.transpose(2, 0, 1), Hc, Wc)
    out = {"flowUp": fu.transpose(1, 2, 0), "a_flowUp": e.transpose(1, 2, 0),
           "flow12": o.transpose(1, 2, 0), "a_flow12": a_o.transpose(1, 2, 0)}
    dist = np.abs(np.abs(o) - 1.0)
    out["decided"] = (dist > a_o).all(0)
    out["inside"] = (np.abs(o) <= 1.0).all(0)
    out["match"] = out["a_match"] = None
    if m12 is not None:
        m, a_m = upsample_ref(np.asarray(m12, dtype=np.float64)[None], H, W)
        m, a_m = m[0], a_m[0]
        if m21 is not None:
            U21, a_U21 = upsample_ref(np.asarray(m21, dtype=np.float64)[None], H, W)
            mm, a_mm, (ix, iy) = sample(U21, H, W)
            mm, a_mm = mm[0], a_mm[0]
            pad = 4
            Ap = np.zeros((1, H + 2 * pad, W + 2 * pad))
            Ap[:, pad:pad + H, pad:pad + W] = a_U21
            x0 = np.clip(np.floor(ix), -2 ** 40, 2 ** 40).astype(np.int64)
            y0 = np.clip(np.floor(iy), -2 ** 40, 2 ** 40).astype(np.int64)
            a_mm = a_mm + _window_max(Ap, y0, x0, (-1, 0, 1, 2), (-1, 0, 1, 2), pad)[0]
            a = np.abs(m) * a_mm + np.abs(mm) * a_m + a_m * a_mm
            a = a + U * (np.abs(m) + a_m) * (np.abs(mm) + a_mm)
            m, a_m = m * mm, a
        out["match"], out["a_match"] = m, a_m
    return out


# --------------------------------------------------------------------------- match gather
def build_matches_ref(idx1, idx2, count, W1, H1, W2, H2, valid16, capacity):
    """build_matches_kernel in numpy: the first min(count, capacity) index pairs, those whose idx2 passes valid16 (all
    when None) in their order, as rows (H1[a], W1[a], 1) / (H2[b], W2[b], 1) float32 (gathers, no arithmetic: exact)."""
    n = min(int(count), int(capacity))
    a, b = np.asarray(idx1[:n]), np.asarray(idx2[:n])
    keep = np.ones(n, bool) if valid16 is None else np.asarray(valid16)[b] != 0
    a, b = a[keep], b[keep]
    one = np.ones(len(a), f32)
    m1 = np.stack([np.asarray(H1, f32)[a], np.asarray(W1, f32)[a], one], 1)
    m2 = np.stack([np.asarray(H2, f32)[b], np.asarray(W2, f32)[b], one], 1)
    return m1, m2, b.astype(np.int64), len(a)


# --------------------------------------------------------------------------- 4-point DLT
DLT_C = 288          # 16 reflectors of length <= 9: backward error 16 gamma~_9 ||A||_F with gamma~_9 = 2 * 9 * u64


def dlt_ref(X, Y):
    """Null vector of the 8x9 DLT matrix (oracle dlt_matrix: fp32 products upcast to fp64) from np.linalg.svd, the LAPACK
    routine the reference calls, with its element-wise bound.  X, Y (N, 4, 3) float32.

    The kernel runs LAPACK's dgebd2 reflector recurrence in fp64 (8 left + 8 right Householder reflectors of length <= 9),
    so both it and LAPACK return the exact null vector of some A + dA with ||dA||_F <= e = 16 gamma~_9 ||A||_F, gamma~_9 =
    2 * 9 * 2^-53 (Higham Thm 19.4).  By Wedin's theorem each is within e / (sigma_8 - e) of the exact null vector, sigma_8
    the smallest nonzero singular value, so they are within 2 e / (sigma_8 - e) of each other; the kernel then rounds to
    fp32 (2^-24 |h|).  Bound = 2^-24 |h| + 2 e / (sigma_8 - e), i.e. c = 2 * 288 over sigma_8 to first order; infinite
    when sigma_8 <= e (numerically degenerate).  Returns (h (N, 9), bound (N, 9), sigma_8 / ||A||_F (N,))."""
    A = OO.dlt_matrix(X, Y)
    _, s, vh = np.linalg.svd(A)
    h = vh[:, 8]
    nrm = np.sqrt((A * A).sum((1, 2)))
    e = DLT_C * U64 * nrm
    s8 = s[:, 7]
    with np.errstate(divide="ignore"):
        geo = np.where(s8 > e, 2 * e / np.maximum(s8 - e, 1e-300), np.inf)
    return h, U * np.abs(h) + geo[:, None], s8 / nrm


def dlt_check(got, X, Y, degenerate=None):
    """Compare kernel null vectors (N, 9) with ``dlt_ref``: sign included wherever the bound is below 1; elsewhere (and for
    the rows flagged ``degenerate``) only finite and unit norm within 2^-22.  Returns (worst ratio, rows checked
    element-wise, rows checked for norm only)."""
    got = np.asarray(got, dtype=np.float64).reshape(len(got), 9)
    h, bound, _ = dlt_ref(X, Y)
    tight = (bound < 1).all(1)
    if degenerate is not None:
        tight &= ~np.asarray(degenerate, bool)
    assert np.isfinite(got).all(), "non-finite DLT output"
    assert np.all(np.abs(np.sqrt((got * got).sum(1)) - 1.0) <= 2.0 ** -22), "DLT output is not unit norm"
    ratio = np.abs(got - h)[tight] / bound[tight]
    worst = float(ratio.max()) if ratio.size else 0.0
    assert worst <= 1.0, "DLT outside its bound: worst ratio %.3g (row %d)" % (worst, int(np.argwhere(tight)[ratio.max(1).argmax()][0]))
    return worst, int(tight.sum()), int((~tight).sum())


# --------------------------------------------------------------------------- checks
def check(got, ref, allow, what=""):
    """|got - ref| <= allow element-wise (NaN in got fails).  Returns the worst |got - ref| / allow (0 / 0 counts 0)."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.broadcast_to(np.asarray(ref, dtype=np.float64), got.shape)
    allow = np.broadcast_to(np.asarray(allow, dtype=np.float64), got.shape)
    err = np.abs(got - ref)
    bad = ~(err <= allow)
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d elements outside the allowance, first at %s: got %r ref %r allow %.3g"
                             % (what, int(bad.sum()), i, got[i], ref[i], allow[i]))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / allow)
    return float(r.max()) if r.size else 0.0


def compose_check(ref, flow12, match=None, flowUp=None, what=""):
    """Check compose_fine outputs ((H, W, 2), (H, W), (H, W, 2) arrays) against ``compose_fine_ref``.  Where the inside mask
    is decided the match must be the masked reference within its allowance (exactly 0 outside); in the undecided band
    either the unmasked value or 0 is accepted.  Returns ({output: worst ratio}, number of undecided pixels)."""
    r = {"flow12": check(flow12, ref["flow12"], ref["a_flow12"], what + " flow12")}
    if flowUp is not None:
        r["flowUp"] = check(flowUp, ref["flowUp"], ref["a_flowUp"], what + " flowUp")
    undecided = int((~ref["decided"]).sum())
    if match is not None:
        d, ins = ref["decided"], ref["inside"]
        match = np.asarray(match, dtype=np.float64)
        r["match"] = check(match[d], (ref["match"] * ins)[d], (ref["a_match"] * ins)[d], what + " match")
        u = ~d
        ok = (match[u] == 0) | (np.abs(match[u] - ref["match"][u]) <= ref["a_match"][u])
        assert ok.all(), what + " match in the undecided band is neither 0 nor the unmasked value"
    return r, undecided


def border_check(flowUp, flow12, match):
    """Identity coarse grid with align_corners=True: a flowUp component clamped to exactly +-1 samples the border column
    (row) with weight exactly 1, so flow12 is exactly +-1 there, which the inside test `|c| <= 1` keeps (match != 0)."""
    at = np.abs(flowUp) == 1.0
    assert at.any(), "the case has no clamped border pixel"
    assert np.array_equal(flow12[at], flowUp[at]), "flow12 is not exactly +-1 where flowUp is"
    assert (match[at.any(-1)] != 0).all(), "the inside test drops pixels whose flow12 is exactly +-1"
    return int(at.any(-1).sum())
