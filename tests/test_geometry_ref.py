"""The fp64 references of tests/geometry_ref.py on the CPU: they agree with the fp32 torch-CPU ops and the oracle within
their allowances, and their checks reject float32 numpy restatements of subtly wrong kernels (so the allowances are not
vacuous).  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import geometry_ref as G
from oracle import outil_oracle as OO
from oracle import warp_oracle as WO

f32 = np.float32


# --------------------------------------------------------------------------- float32 restatements of the kernels
def grid_sample_f32(inp, grid, ac, swap=False, border=False, w16=False):
    """grid_sample_kernel in numpy float32 (finite grids).  swap: the two unnormalize formulas exchanged; border: corners
    clamped into the image instead of skipped; w16: sampling weights carried in fp16."""
    inp, g = np.asarray(inp, f32), np.asarray(grid, f32)
    N, C, Hin, Win = inp.shape
    a = (not ac) if swap else ac

    def un(c, size):
        c1 = c + f32(1)
        return (c1 / f32(2)) * f32(size - 1) if a else (c1 * f32(size) - f32(1)) / f32(2)
    out = np.zeros((N, C) + g.shape[1:3], f32)
    for n in range(N):
        ix, iy = un(g[n, ..., 0], Win), un(g[n, ..., 1], Hin)
        fx, fy = np.floor(ix), np.floor(iy)
        x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
        wx = ((fx + f32(1)) - ix, ix - fx)
        wy = ((fy + f32(1)) - iy, iy - fy)
        for dy in (0, 1):
            for dx in (0, 1):
                w = wx[dx] * wy[dy]
                if w16:
                    w = w.astype(np.float16).astype(f32)
                xi, yi = x0 + dx, y0 + dy
                valid = (xi >= 0) & (xi < Win) & (yi >= 0) & (yi < Hin)
                if border:
                    valid = np.ones_like(valid)
                v = inp[n][:, np.clip(yi, 0, Hin - 1), np.clip(xi, 0, Win - 1)]
                out[n] += np.where(valid, v * w, f32(0))
    return out


def up_coord_f32(out_n, in_n, half=True, clamp0=True):
    scale = f32(in_n) / f32(out_n)
    d = np.arange(out_n).astype(f32)
    src = scale * (d + f32(0.5)) - f32(0.5) if half else scale * d
    if clamp0:
        src = np.maximum(src, f32(0))
    i0 = src.astype(np.int64)                       # (int): truncation toward zero
    i1 = i0 + (i0 < in_n - 1)
    l1 = src - i0.astype(f32)
    return i0, i1, f32(1) - l1, l1


def upsample_f32(x, H, W, half=True, clamp0=True):
    """upsample_kernel in numpy float32.  half: the half-pixel offset; clamp0: `if (src < 0) src = 0`."""
    x = np.asarray(x, f32)
    y0, y1, ly0, ly1 = up_coord_f32(H, x.shape[1], half, clamp0)
    x0, x1, lx0, lx1 = up_coord_f32(W, x.shape[2], half, clamp0)
    r0, r1 = x[:, y0][:, :, None], x[:, y1][:, :, None]     # (NC, H, 1, w)
    a = (lambda r: lx0 * r[..., x0] + lx1 * r[..., x1])
    return (ly0[:, None] * a(r0[:, :, 0]) + ly1[:, None] * a(r1[:, :, 0])).astype(f32)


def compose_f32(flow8, m12, m21, coarse, H, W, clamp, ac, m21_coarse=False, lt=False, lin=G.lin11):
    """compose_fine_kernel in numpy float32.  m21_coarse: match21 upsampled to (and sampled at) the coarse grid's size
    instead of (H, W); lt: `<` instead of `<=` in the inside test; lin: the base-grid formula."""
    Hc, Wc = coarse.shape[0], coarse.shape[1]
    up = upsample_f32(flow8, H, W)
    fu = np.stack([up[0] + lin(np.arange(W), W)[None, :], up[1] + lin(np.arange(H), H)[:, None]], -1).astype(f32)
    if clamp:
        fu = np.clip(fu, f32(-1), f32(1))
    o = grid_sample_f32(np.asarray(coarse, f32).transpose(2, 0, 1)[None], fu[None], ac)[0].transpose(1, 2, 0)
    m = upsample_f32(np.asarray(m12, f32)[None], H, W)[0]
    if m21 is not None:
        hs, ws = (Hc, Wc) if m21_coarse else (H, W)
        m = m * grid_sample_f32(upsample_f32(np.asarray(m21, f32)[None], hs, ws)[None], fu[None], ac)[0, 0]
    inside = ((o > -1) & (o < 1)) if lt else ((o >= -1) & (o <= 1))
    return fu, o, (m * inside.all(-1)).astype(f32)


# --------------------------------------------------------------------------- inputs
def rand_grid(rs, n, h, w, lim=1.3):
    return rs.uniform(-lim, lim, (n, h, w, 2)).astype(f32)


def edge_grid(h, w, Hin, Win):
    """lines exactly on +-1 and on +-(1 + 1/W): every column / row of the output takes one of those x / y values."""
    xs = np.array([-1, 1, -1 - 1 / Win, 1 + 1 / Win, 0.5], f32)
    ys = np.array([-1, 1, -1 - 1 / Hin, 1 + 1 / Hin, -0.25], f32)
    gx = np.resize(xs, w)[None, :].repeat(h, 0)
    gy = np.resize(ys, h)[:, None].repeat(w, 1)
    return np.stack([gx, gy], -1)[None].astype(f32)


def compose_inputs(seed, h8, w8, Hc, Wc, scale=0.05):
    rs = np.random.RandomState(seed)
    f8 = (rs.randn(2, h8, w8) * scale).astype(f32)
    m12, m21 = rs.rand(h8, w8).astype(f32), rs.rand(h8, w8).astype(f32)
    Hm = (np.eye(3) + rs.uniform(-0.08, 0.08, (3, 3))).astype(f32)
    return f8, m12, m21, G.warp_grid_f32(Hm, Hc, Wc)[0]


def border_inputs(h8, w8, H, W):
    """Identity coarse grid and flows that push every pixel past the border: the `<=` case of the inside test."""
    rs = np.random.RandomState(5)
    f8 = np.sign(rs.randn(2, h8, w8)).astype(f32) * f32(2.5)
    m12 = (rs.rand(h8, w8) * 0.5 + 0.5).astype(f32)
    return f8, m12, G.warp_grid_f32(np.eye(3, dtype=f32), H, W)[0]


# --------------------------------------------------------------------------- the references agree with torch-CPU and the oracle
@pytest.mark.parametrize("shape,hw", [((2, 3, 20, 26), (31, 45)), ((1, 5, 9, 11), (12, 7)), ((2, 1, 5, 7), (6, 6)),
                                      ((1, 1, 1, 9), (4, 5)), ((1, 2, 1, 1), (3, 3))])
@pytest.mark.parametrize("ac", [False, True])
def test_grid_sample_ref_vs_torch_cpu(shape, hw, ac):
    rs = np.random.RandomState(sum(shape) + hw[0])
    inp = rs.randn(*shape).astype(f32)
    for grid in (rand_grid(rs, shape[0], *hw), np.repeat(edge_grid(*hw, shape[2], shape[3]), shape[0], 0)):
        ref, allow, _ = G.grid_sample_ref(inp, grid, ac)
        cpu = F.grid_sample(torch.from_numpy(inp), torch.from_numpy(grid), mode="bilinear", padding_mode="zeros", align_corners=ac)
        G.check(cpu.numpy(), ref, allow, "torch-CPU")
        G.check(grid_sample_f32(inp, grid, ac), ref, allow, "float32 restatement")


def test_grid_sample_ref_outside_coordinates():
    """+-inf, +-1e30, NaN and |c| beyond 2^31 pixels sample nothing (torch's CUDA safe_downgrade_to_int_range)."""
    inp = np.ones((1, 1, 4, 4), f32)
    vals = np.array([np.inf, -np.inf, 1e30, -1e30, np.nan, 2.0 ** 31], f32)
    grid = np.stack([np.stack([vals, np.zeros_like(vals)], -1), np.stack([np.zeros_like(vals), vals], -1)])[None].reshape(1, 2, 6, 2)
    ref, allow, outside = G.grid_sample_ref(inp, grid, False)
    assert outside.all() and not ref.any() and not allow.any()


@pytest.mark.parametrize("hw,HW", [((6, 9), (47, 121)), ((60, 80), (480, 640)), ((1, 1), (5, 3)), ((480, 640), (30, 40)),
                                   ((376, 1241), (24, 78)), ((1, 50), (7, 1)), ((3, 4), (3, 4))])
def test_upsample_ref_vs_torch_cpu(hw, HW):
    rs = np.random.RandomState(hw[0] + HW[1])
    x = rs.randn(2, *hw).astype(f32)
    ref, allow = G.upsample_ref(x, *HW)
    cpu = F.interpolate(torch.from_numpy(x)[None], size=HW, mode="bilinear", align_corners=False)[0].numpy()
    G.check(cpu, ref, allow, "torch-CPU")
    got = upsample_f32(x, *HW)
    G.check(got, ref, allow, "float32 restatement")
    if hw == HW:
        assert np.array_equal(got, x)


@pytest.mark.parametrize("h8,w8,Hc,Wc,H,W", [(6, 8, 48, 64, 48, 64), (6, 9, 48, 64, 56, 80), (6, 9, 96, 128, 48, 64),
                                             (6, 9, 30, 100, 47, 121), (3, 1, 20, 1, 20, 1), (1, 4, 1, 30, 1, 30)])
@pytest.mark.parametrize("ac", [False, True])
def test_compose_fine_ref_vs_oracle(h8, w8, Hc, Wc, H, W, ac):
    f8, m12, m21, coarse = compose_inputs(Hc + W, h8, w8, Hc, Wc)
    ref = G.compose_fine_ref(f8, m12, m21, coarse, H, W, True, ac)
    base = torch.from_numpy(np.stack(np.broadcast_arrays(G.lin11(np.arange(W), W)[None, :], G.lin11(np.arange(H), H)[:, None]), -1)[None])
    if not ac:           # the oracle's chain is the reference's (torch-CPU fp32, align_corners=False)
        flow12, flowUp = WO.compose_fine(torch.from_numpy(f8)[None], torch.from_numpy(coarse)[None], base)
        mt = WO.interpolate_bilinear(torch.from_numpy(m12)[None, None], (H, W))
        mt = mt * WO.grid_sample(WO.interpolate_bilinear(torch.from_numpy(m21)[None, None], (H, W)), flowUp)
        G.compose_check(ref, flow12[0].numpy(), mt[0, 0].numpy() * WO.inside_mask(flow12)[0, 0].numpy(), flowUp[0].numpy(), "oracle")
    fu, o, m = compose_f32(f8, m12, m21, coarse, H, W, True, ac)
    G.compose_check(ref, o, m, fu, "float32 restatement")


def test_warp_grid_f32_vs_oracle():
    """warp_grid_f32 against the oracle's kornia restatement (torch-CPU, CPU linspace): a few ulps away from pz ~ 0."""
    rs = np.random.RandomState(0)
    Hs = np.stack([np.eye(3) + rs.uniform(-0.1, 0.1, (3, 3)) for _ in range(4)]).astype(f32)
    for h, w in ((31, 45), (480, 640), (1, 7), (9, 1)):
        a = G.warp_grid_f32(Hs, h, w)
        b = WO.warp_grid(Hs, h, w).numpy()
        assert np.all(np.abs(a - b) <= 16 * G.U * (np.abs(b) + 1)), (h, w)
    for n in (2, 3, 45, 640, 1241):
        assert np.abs(G.lin11(np.arange(n), n) - torch.linspace(-1, 1, n).numpy()).max() <= 2.0 ** -23


def test_warp_grid_f32_non_finite():
    """Third row (1, 0, 0) at an odd width: the middle column has pz = 0 exactly, 0/0 for a zero numerator and +-inf else."""
    Hm = np.array([[1, 0, 0], [0, 1, 0.5], [1, 0, 0]], f32)
    g = G.warp_grid_f32(Hm, 3, 5)[0]
    assert np.isnan(g[:, 2, 0]).all() and np.isinf(g[:, 2, 1]).all()
    assert np.isfinite(g[:, [0, 1, 3, 4]]).all()


def test_dlt_ref_bound_holds_for_the_recurrence_the_kernel_runs():
    """The dgebd2 reflector recurrence (oracle householder_null_vector, the kernel's algorithm in fp64) against
    np.linalg.svd within dlt_ref's bound, sign included, on seeded well-conditioned and near-collinear quadruples and a
    golden RANSAC case's samples; exactly collinear quadruples give an infinite bound."""
    X, Y = dlt_quadruples(7)
    h = np.stack([OO.householder_null_vector(a) for a in OO.dlt_matrix(X, Y)]).astype(f32)
    worst, tight, loose = G.dlt_check(h, X, Y)
    assert tight >= len(X) - 8 and worst <= 1
    Xc, Yc = collinear_quadruples(7)
    _, bound, s = G.dlt_ref(Xc, Yc)
    assert (bound >= 1).all() or (s < 1e-12).all()


def dlt_quadruples(seed, n=200):
    """Seeded quadruples in [-1, 1]^2: half generic, half near-collinear (the 4th point within 1e-4 .. 1e-2 of a line)."""
    rs = np.random.RandomState(seed)
    X = rs.uniform(-1, 1, (n, 4, 3))
    Y = rs.uniform(-1, 1, (n, 4, 3))
    for P in (X, Y):
        t = rs.uniform(-1, 1, (n // 2, 1))
        P[n // 2:, 3, :2] = P[n // 2:, 0, :2] + t * (P[n // 2:, 1, :2] - P[n // 2:, 0, :2]) + rs.uniform(1e-4, 1e-2, (n // 2, 2))
    X[..., 2] = Y[..., 2] = 1
    return X.astype(f32), Y.astype(f32)


def collinear_quadruples(seed, n=32):
    """All four points on one axis-parallel or diagonal line in both images, with exactly representable coordinates."""
    rs = np.random.RandomState(seed)
    X = np.zeros((n, 4, 3), f32)
    Y = np.zeros((n, 4, 3), f32)
    for P in (X, Y):
        t = rs.randint(-8, 9, (n, 4)) / 8.0
        c = rs.randint(-4, 5, (n, 1)) / 8.0
        kind = np.arange(n) % 3
        P[..., 0] = np.where(kind[:, None] == 0, c, t)
        P[..., 1] = np.where(kind[:, None] == 1, c, t)
        P[..., 2] = 1
    return X, Y


# --------------------------------------------------------------------------- the checks reject restatements of wrong kernels
def test_rejects_swapped_align_corners():
    rs = np.random.RandomState(1)
    inp, grid = rs.randn(1, 3, 20, 26).astype(f32), rand_grid(rs, 1, 31, 45)
    ref, allow, _ = G.grid_sample_ref(inp, grid, False)
    with pytest.raises(AssertionError):
        G.check(grid_sample_f32(inp, grid, False, swap=True), ref, allow)


def test_rejects_border_padding():
    rs = np.random.RandomState(2)
    inp, grid = rs.randn(1, 3, 20, 26).astype(f32), rand_grid(rs, 1, 31, 45)
    ref, allow, _ = G.grid_sample_ref(inp, grid, True)
    with pytest.raises(AssertionError):
        G.check(grid_sample_f32(inp, grid, True, border=True), ref, allow)


def test_rejects_upsampling_without_half_pixel_offset():
    x = np.random.RandomState(3).randn(2, 60, 80).astype(f32)
    ref, allow = G.upsample_ref(x, 480, 640)
    with pytest.raises(AssertionError):
        G.check(upsample_f32(x, 480, 640, half=False), ref, allow)


def test_rejects_upsampling_without_the_zero_clamp():
    x = np.random.RandomState(4).randn(2, 6, 9).astype(f32)
    ref, allow = G.upsample_ref(x, 47, 121)
    with pytest.raises(AssertionError):
        G.check(upsample_f32(x, 47, 121, clamp0=False), ref, allow)


def test_rejects_fp16_sampling_weights():
    rs = np.random.RandomState(5)
    inp, grid = rs.randn(1, 3, 20, 26).astype(f32), rand_grid(rs, 1, 31, 45)
    ref, allow, _ = G.grid_sample_ref(inp, grid, False)
    with pytest.raises(AssertionError):
        G.check(grid_sample_f32(inp, grid, False, w16=True), ref, allow)


def test_rejects_match21_at_the_coarse_size():
    f8, m12, m21, coarse = compose_inputs(6, 6, 9, 96, 128)
    ref = G.compose_fine_ref(f8, m12, m21, coarse, 48, 64, True, False)
    fu, o, m = compose_f32(f8, m12, m21, coarse, 48, 64, True, False, m21_coarse=True)
    with pytest.raises(AssertionError):
        G.compose_check(ref, o, m, fu)


def test_rejects_single_branch_linspace():
    one = lambda i, n: (f32(-1) + (f32(2) / f32(n - 1)) * np.asarray(i).astype(f32)).astype(f32)
    Hm = np.eye(3, dtype=f32)[None]
    assert not np.array_equal(G.warp_grid_f32(Hm, 30, 41), np.stack(np.broadcast_arrays(
        one(np.arange(41), 41)[None, None, :], one(np.arange(30), 30)[None, :, None]), -1))


def test_rejects_strict_inside_test():
    f8, m12, coarse = border_inputs(6, 8, 48, 64)
    fu, o, m = compose_f32(f8, m12, None, coarse, 48, 64, True, True)
    assert G.border_check(fu, o, m) > 0
    fu, o, m = compose_f32(f8, m12, None, coarse, 48, 64, True, True, lt=True)
    with pytest.raises(AssertionError):
        G.border_check(fu, o, m)
