"""The kernels after the correlation against the fp64 references of tests/geometry_ref.py, element by element:
warp_grid_kernel (bit for bit), grid_sample_kernel, upsample_kernel, compose_fine_kernel, build_matches_kernel and
dlt_kernel.  Every output is NaN-filled (or sentinel-filled) before the call, so an element the kernel never writes fails.
The C entry points are called as the wrappers call them; the wrappers themselves are called where their own behaviour
(output layout, refusals) is under test."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import geometry_ref as G
from conftest import golden
from oracle import outil_oracle as OO
from test_geometry_ref import border_inputs, collinear_quadruples, compose_inputs, dlt_quadruples, edge_grid

pytestmark = pytest.mark.gpu
f32 = np.float32


def nan_like(shape, memory_format=torch.contiguous_format):
    return torch.full(shape, float("nan"), device="cuda").contiguous(memory_format=memory_format)


def bit_equal(a, b):
    """Same bits, NaN payloads aside (the device's canonical NaN is not numpy's)."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


# --------------------------------------------------------------------------- warp_grid
def homographies():
    rs = np.random.RandomState(11)
    Hs = [np.eye(3), 4 * np.eye(3), 0.3 * np.eye(3)]
    Hs += [np.eye(3) + rs.uniform(-0.1, 0.1, (3, 3)) for _ in range(10)]
    Hs += [np.array([[1, 0.1, 0], [0.05, 1, 0], [0.8, 0.3, 0.1]]),           # horizon crosses the image
           np.array([[0.9, 0, 0.2], [0, 1.1, 0], [0, -0.7, 0.05]]),
           np.array([[1, 0, 0], [0, 1, 0.5], [1, 0, 0]])]                      # pz = 0 exactly on the middle column of odd widths
    return np.stack(Hs).astype(f32)


def warp_grid_device(rf, Hs, h, w):
    Hd = torch.from_numpy(Hs).cuda()
    out = nan_like((len(Hs), h, w, 2))
    rf._lib.check(rf.ops.lib.rf_warp_grid(rf.ops.ptr(Hd), len(Hs), h, w, rf.ops.ptr(out), rf.ops.stream()))
    return out.cpu().numpy()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (9, 1), (2, 2), (31, 45), (480, 640), (376, 1241), (5, 9)])
def test_warp_grid_bit_exact(rf, h, w):
    Hs = homographies()
    assert len(Hs) == 16
    ref = G.warp_grid_f32(Hs, h, w)
    all16 = warp_grid_device(rf, Hs, h, w)
    assert bit_equal(all16, ref), (h, w)
    assert bit_equal(warp_grid_device(rf, Hs[:3], h, w), ref[:3])
    for i in range(len(Hs)):
        assert bit_equal(warp_grid_device(rf, Hs[i:i + 1], h, w), all16[i:i + 1]), i
    if (h, w) == (5, 9):
        assert np.isnan(all16[-1, :, 4, 0]).all() and not np.isfinite(all16[-1, :, 4, 1]).any()
    print("warp_grid %dx%d: bit-exact, %d non-finite values" % (h, w, int((~np.isfinite(all16)).sum())))


# --------------------------------------------------------------------------- grid_sample
def layouts(x, name):
    """(N, C, H, W) CPU tensor -> a CUDA tensor with the same values in the named layout."""
    N, Cc, Hh, Ww = x.shape
    if name == "nchw":
        return x.cuda()
    if name == "cl":
        return x.cuda().contiguous(memory_format=torch.channels_last)
    if name == "wstride":
        big = torch.full((N, Cc, Hh, 2 * Ww), float("nan"), device="cuda")
        big[..., ::2] = x.cuda()
        return big[..., ::2]
    if name == "narrow":
        big = torch.full((N, Cc + 2, Hh, Ww), float("nan"), device="cuda")
        big[:, 1:1 + Cc] = x.cuda()
        return big.narrow(1, 1, Cc)
    if name == "expand":
        return x[:1].cuda().expand(N, Cc, Hh, Ww)
    raise ValueError(name)


def grid_sample_device(rf, inp, grid, ac):
    """rf_grid_sample into a NaN-filled output in the layout the wrapper picks (channels-last for a channels-last input)."""
    N, Cc, Hin, Win = inp.shape
    Hout, Wout = grid.shape[1], grid.shape[2]
    cl = inp.stride(1) == 1 and Cc > 1
    out = nan_like((N, Hout, Wout, Cc)).permute(0, 3, 1, 2) if cl else nan_like((N, Cc, Hout, Wout))
    is_ = (C.c_longlong * 4)(*inp.stride())
    os_ = (C.c_longlong * 4)(*out.stride())
    g = grid.cuda().contiguous()
    rf._lib.check(rf.ops.lib.rf_grid_sample(rf.ops.ptr(inp), N, Cc, Hin, Win, is_, rf.ops.ptr(g), Hout, Wout, int(ac),
                                            rf.ops.ptr(out), os_, rf.ops.stream()))
    return out


def non_finite_grid(rs, n, h, w):
    g = np.asarray(rs.uniform(-1.3, 1.3, (n, h, w, 2)), f32)
    bad = np.array([np.inf, -np.inf, 1e30, -1e30, np.nan], f32)
    sel = rs.rand(n, h, w, 2) < 0.3
    g[sel] = bad[rs.randint(0, len(bad), int(sel.sum()))]
    return g


SAMPLE_CASES = [((1, 3, 480, 640), (480, 640), ["cl", "nchw"]), ((4, 3, 20, 26), (31, 45), ["nchw", "cl", "wstride", "narrow", "expand"]),
                ((3, 64, 9, 11), (12, 7), ["nchw", "cl", "narrow", "expand"]), ((2, 1, 5, 7), (6, 6), ["nchw", "wstride", "expand"]),
                ((1, 1, 1, 9), (4, 5), ["nchw", "wstride"]), ((1, 2, 1, 1), (3, 3), ["nchw", "cl"])]


@pytest.mark.parametrize("shape,hw,names", SAMPLE_CASES)
@pytest.mark.parametrize("ac", [False, True])
def test_grid_sample_vs_fp64(rf, shape, hw, names, ac):
    N = shape[0]
    rs = np.random.RandomState(shape[1] * 7 + hw[1] + ac)
    x = torch.from_numpy(rs.randn(*shape).astype(f32))
    if hw == (480, 640):          # the pair path: a homography grid over the full image
        Hm = np.stack([np.eye(3) + rs.uniform(-0.15, 0.15, (3, 3))]).astype(f32)
        grids = {"homography": G.warp_grid_f32(Hm, *hw)}
    else:
        grids = {"random": np.asarray(rs.uniform(-1.3, 1.3, (N,) + hw + (2,)), f32),
                 "edges": np.repeat(edge_grid(*hw, shape[2], shape[3]), N, 0)}
    grids["non-finite"] = non_finite_grid(rs, N, *hw)
    worst = 0.0
    for name in names:
        inp = layouts(x, name)
        vals = inp.cpu().numpy()
        for gname, grid in grids.items():
            ref, allow, outside = G.grid_sample_ref(vals, grid, ac)
            got = grid_sample_device(rf, inp, torch.from_numpy(grid), ac)
            worst = max(worst, G.check(got.cpu().numpy(), ref, allow, "%s %s %s" % (shape, name, gname)))
            if gname == "non-finite":     # +-inf / 1e30 / NaN rows: pinned to torch's CUDA grid sampler
                tc = torch_cuda_grid_sample(inp.contiguous(), torch.from_numpy(grid).cuda(), ac).cpu().numpy()
                o = np.broadcast_to(outside[:, None], tc.shape)
                assert np.array_equal(got.cpu().numpy()[o], tc[o]) and not tc[o].any()
    print("grid_sample %s -> %s ac=%d: worst error / allowance %.3g" % (shape, hw, ac, worst))


def torch_cuda_grid_sample(inp, grid, ac):
    """torch's own CUDA grid sampler (ATen's kernel).  With align_corners=True F.grid_sample would hand a contiguous fp32
    input to cuDNN instead, which differs on non-finite coordinates (see below)."""
    with torch.backends.cudnn.flags(enabled=False):
        return F.grid_sample(inp, grid, mode="bilinear", padding_mode="zeros", align_corners=ac)


@pytest.mark.parametrize("ac", [False, True])
def test_grid_sample_cuda_reference_on_outside_coordinates(rf, ac):
    """What torch's CUDA grid sampler returns for +-inf, +-1e30 and NaN coordinates, and the kernel's value at each: both 0
    (ATen's safe_downgrade_to_int_range).  F.grid_sample's cuDNN path (align_corners=True) is printed for the record."""
    inp = torch.ones(1, 1, 4, 4, device="cuda")
    vals = [float("inf"), float("-inf"), 1e30, -1e30, float("nan")]
    g = torch.tensor([[[[v, 0.0] for v in vals], [[0.0, v] for v in vals]]], device="cuda")
    tc = torch_cuda_grid_sample(inp, g, ac)
    dnn = F.grid_sample(inp, g, mode="bilinear", padding_mode="zeros", align_corners=ac)
    got = grid_sample_device(rf, inp, g, ac)
    print("align_corners=%d, x / y = %s: ATen CUDA %s, F.grid_sample %s, kernel %s" % (ac, vals, tc[0, 0].tolist(), dnn[0, 0].tolist(), got[0, 0].tolist()))
    assert torch.equal(got, tc) and not tc.any()


@pytest.mark.parametrize("name,cl_out", [("nchw", False), ("cl", True), ("wstride", False), ("narrow", False), ("expand", False)])
def test_grid_sample_wrapper_layout(rf, name, cl_out):
    rs = np.random.RandomState(3)
    x = torch.from_numpy(rs.randn(2, 3, 20, 26).astype(f32))
    grid = torch.from_numpy(rs.uniform(-1.3, 1.3, (2, 9, 11, 2)).astype(f32))
    inp = layouts(x, name)
    out = rf.ops.grid_sample(inp, grid.cuda(), False)
    expect = (9 * 11 * 3, 1, 11 * 3, 3) if cl_out else (3 * 9 * 11, 9 * 11, 11, 1)
    assert out.stride() == expect and tuple(out.shape) == (2, 3, 9, 11)
    assert torch.equal(out, grid_sample_device(rf, inp, grid, False))


def test_grid_sample_wrapper_refusals(rf):
    inp = torch.zeros(2, 3, 5, 7, device="cuda")
    for bad in (torch.zeros(1, 4, 4, 2), torch.zeros(2, 4, 4, 3), torch.zeros(4, 4, 2), torch.zeros(3, 4, 4, 2)):
        with pytest.raises(ValueError):
            rf.ops.grid_sample(inp, bad.cuda())


# --------------------------------------------------------------------------- upsample
def upsample_device(rf, x, H, W):
    xd = torch.from_numpy(x).cuda()
    out = nan_like((x.shape[0], H, W))
    rf._lib.check(rf.ops.lib.rf_upsample_bilinear(rf.ops.ptr(xd), x.shape[0], x.shape[1], x.shape[2], H, W, rf.ops.ptr(out), rf.ops.stream()))
    return out.cpu().numpy()


@pytest.mark.parametrize("hw,HW,ncs", [((60, 80), (480, 640), (1, 2)), ((6, 9), (47, 121), (1, 2, 98)), ((1, 1), (5, 3), (1, 2, 98)),
                                       ((3, 4), (3, 4), (1, 2, 98)), ((480, 640), (30, 40), (1, 2, 98)),
                                       ((376, 1241), (24, 78), (1, 2)), ((1, 50), (7, 1), (1, 2, 98))])
def test_upsample_vs_fp64(rf, hw, HW, ncs):
    worst = 0.0
    for nc in ncs:
        x = np.random.RandomState(nc + hw[1]).randn(nc, *hw).astype(f32)
        got = upsample_device(rf, x, *HW)
        if hw == HW:
            assert np.array_equal(got, x), "scale 1 must copy bit for bit"
        ref, allow = G.upsample_ref(x, *HW)
        worst = max(worst, G.check(got, ref, allow, "%s -> %s nc %d" % (hw, HW, nc)))
    print("upsample %s -> %s: worst error / allowance %.3g" % (hw, HW, worst))


@pytest.mark.parametrize("hw,HW", [((480, 640), (30, 40)), ((376, 1241), (24, 78)), ((60, 80), (30, 40)), ((97, 131), (7, 9))])
def test_mask_downsampling_decision(rf, hw, HW):
    """Binary (0/1) masks down-sampled at the mask ratios of the pair path, then thresholded at > 0.5 (the matches RANSAC
    sees): the decision equals the fp64 decision wherever the fp64 value is farther from 0.5 than its allowance."""
    rs = np.random.RandomState(hw[0])
    blocks = rs.rand(2, hw[0] // 8 + 1, hw[1] // 8 + 1) < 0.5
    m = np.kron(blocks, np.ones((8, 8)))[:, :hw[0], :hw[1]]
    m = np.where(rs.rand(*m.shape) < 0.02, 1 - m, m).astype(f32)          # salt: isolated pixels flip
    got = upsample_device(rf, m, *HW)
    ref, allow = G.upsample_ref(m, *HW)
    G.check(got, ref, allow, "mask")
    decided = np.abs(ref - 0.5) > allow
    assert np.array_equal((got > 0.5)[decided], (ref > 0.5)[decided])
    print("mask %s -> %s: %d of %d values in the undecided band of 0.5" % (hw, HW, int((~decided).sum()), ref.size))


# --------------------------------------------------------------------------- compose_fine
def compose_device(rf, f8, m12, m21, coarse, H, W, clamp, ac, want_match=True, legacy=False):
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    fd, md12, md21, cd = dev(f8), dev(m12), dev(m21), dev(coarse)
    h8, w8 = f8.shape[1], f8.shape[2]
    Hc, Wc = coarse.shape[0], coarse.shape[1]
    flow12, flowUp = nan_like((H, W, 2)), nan_like((H, W, 2))
    match = nan_like((H, W)) if want_match else None
    p, s = rf.ops.ptr, rf.ops.stream()
    if legacy:
        assert (Hc, Wc) == (H, W)
        rc = rf.ops.lib.rf_compose_fine(p(fd), p(md12), p(md21), h8, w8, p(cd), H, W, int(clamp), int(ac), p(flow12), p(match), p(flowUp), s)
    else:
        rc = rf.ops.lib.rf_compose_fine_ex(p(fd), p(md12), p(md21), h8, w8, p(cd), Hc, Wc, H, W, int(clamp), int(ac),
                                           p(flow12), p(match), p(flowUp), s)
    rf._lib.check(rc)
    return flow12.cpu().numpy(), None if match is None else match.cpu().numpy(), flowUp.cpu().numpy()


COMPOSE_SHAPES = [(60, 80, 480, 640, 480, 640), (6, 8, 48, 64, 48, 64), (6, 9, 48, 64, 56, 80), (6, 9, 40, 56, 40, 56),
                  (6, 9, 96, 128, 48, 64), (6, 9, 30, 100, 47, 121), (3, 1, 20, 1, 20, 1), (1, 4, 1, 30, 1, 30)]


@pytest.mark.parametrize("h8,w8,Hc,Wc,H,W", COMPOSE_SHAPES)
def test_compose_fine_vs_fp64(rf, h8, w8, Hc, Wc, H, W):
    f8, m12, m21, coarse = compose_inputs(Hc + W, h8, w8, Hc, Wc, 0.1)
    worst, undecided = {}, 0
    for use21 in (False, True):
        for clamp in (True, False):
            for ac in (False, True):
                ref = G.compose_fine_ref(f8, m12, m21 if use21 else None, coarse, H, W, clamp, ac)
                o, m, fu = compose_device(rf, f8, m12, m21 if use21 else None, coarse, H, W, clamp, ac)
                r, u = G.compose_check(ref, o, m, fu, "m21 %d clamp %d ac %d" % (use21, clamp, ac))
                undecided += u
                for k, v in r.items():
                    worst[k] = max(worst.get(k, 0.0), v)
                if (Hc, Wc) == (H, W) and use21:
                    lo, lm, lu = compose_device(rf, f8, m12, m21, coarse, H, W, clamp, ac, legacy=True)
                    assert bit_equal(lo, o) and bit_equal(lm, m) and bit_equal(lu, fu)
    o, m, fu = compose_device(rf, f8, None, None, coarse, H, W, True, False, want_match=False)
    G.compose_check(G.compose_fine_ref(f8, None, None, coarse, H, W, True, False), o, None, fu)
    print("compose_fine %dx%d -> coarse %dx%d, out %dx%d: worst ratios %s, %d undecided inside-mask pixels"
          % (h8, w8, Hc, Wc, H, W, {k: round(v, 3) for k, v in worst.items()}, undecided))


@pytest.mark.parametrize("h8,w8,H,W", [(6, 8, 48, 64), (60, 80, 480, 640), (3, 2, 24, 9)])
def test_compose_fine_inside_test_keeps_the_border(rf, h8, w8, H, W):
    """Identity coarse grid, align_corners=True, flows pushed past the border: flow12 is exactly +-1 at the clamped pixels
    and the inside test (`<=`) keeps them."""
    f8, m12, coarse = border_inputs(h8, w8, H, W)
    o, m, fu = compose_device(rf, f8, m12, None, coarse, H, W, True, True)
    n = G.border_check(fu, o, m)
    G.compose_check(G.compose_fine_ref(f8, m12, None, coarse, H, W, True, True), o, m, fu)
    print("border case %dx%d: %d pixels exactly on the border" % (H, W, n))


def test_compose_fine_wrapper_refusals(rf):
    f8, m, c = torch.zeros(1, 2, 6, 8).cuda(), torch.zeros(1, 1, 6, 8).cuda(), torch.zeros(1, 48, 64, 2).cuda()
    rf.ops.compose_fine(f8, m, m, c)                                        # the accepted shapes
    for args in ((torch.zeros(2, 2, 6, 8).cuda(), m, m, c), (f8, torch.zeros(2, 1, 6, 8).cuda(), m, c),
                 (f8, m, torch.zeros(2, 1, 6, 8).cuda(), c), (f8, m, m, torch.zeros(2, 48, 64, 2).cuda()),
                 (f8, torch.zeros(1, 1, 5, 8).cuda(), None, c), (torch.zeros(1, 3, 6, 8).cuda(), m, None, c)):
        with pytest.raises(ValueError):
            rf.ops.compose_fine(*args)


# --------------------------------------------------------------------------- build_matches
@pytest.mark.parametrize("count", [0, 1, 31, 32, 255, 256, 257, 4097, 13065, 60000])
@pytest.mark.parametrize("valid", ["none", "zeros", "ones", "p0.3"])
def test_build_matches_bit_exact(rf, count, valid):
    rs = np.random.RandomState(count + len(valid))
    P1, P2 = count + 37, count + 53
    idx1 = rs.permutation(P1)[:count].astype(np.int64)
    idx2 = rs.permutation(P2)[:count].astype(np.int64)
    W1, H1, W2, H2 = (rs.uniform(-1, 1, n).astype(f32) for n in (P1, P1, P2, P2))
    v16 = {"none": None, "zeros": np.zeros(P2, np.uint8), "ones": np.ones(P2, np.uint8),
           "p0.3": (rs.rand(P2) < 0.3).astype(np.uint8)}[valid]
    keep = [None if a is None else torch.from_numpy(a).cuda() for a in (W1, H1, W2, H2, v16)]      # alive until the launch ran
    dW1, dH1, dW2, dH2, dv16 = keep
    caps = [max(count, 1)] + ([count // 2 + 1] if count > 1 else [])
    for cap in caps:
        rows = max(count, 1) + 8                 # room beyond the capacity: rows the kernel must leave alone
        m1, m2 = nan_like((rows, 3)), nan_like((rows, 3))
        kept = torch.full((rows,), -7, dtype=torch.int64, device="cuda")
        cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        di1 = torch.from_numpy(idx1 if count else np.zeros(1, np.int64)).cuda()
        di2 = torch.from_numpy(idx2 if count else np.zeros(1, np.int64)).cuda()
        cin = torch.tensor([count], dtype=torch.int32, device="cuda")
        p = rf.ops.ptr
        rf._lib.check(rf.ops.lib.rf_build_matches(p(di1), p(di2), p(cin), p(dW1), p(dH1), p(dW2), p(dH2), p(dv16),
                                                  p(m1), p(m2), p(kept), p(cnt), cap, rf.ops.stream()))
        e1, e2, ek, n = G.build_matches_ref(idx1, idx2, count, W1, H1, W2, H2, v16, cap)
        m1, m2, kept, cnt = m1.cpu().numpy(), m2.cpu().numpy(), kept.cpu().numpy(), int(cnt.item())
        assert cnt == n, (cap, cnt, n)
        assert bit_equal(m1[:n], e1) and bit_equal(m2[:n], e2) and np.array_equal(kept[:n], ek)
        assert np.isnan(m1[n:]).all() and np.isnan(m2[n:]).all() and (kept[n:] == -7).all()


# --------------------------------------------------------------------------- DLT
def dlt_device(rf, X, Y):
    Xd, Yd = torch.from_numpy(np.ascontiguousarray(X)).cuda(), torch.from_numpy(np.ascontiguousarray(Y)).cuda()
    out = nan_like((len(X), 3, 3))
    rf._lib.check(rf.ops.lib.rf_homography_dlt(rf.ops.ptr(Xd), rf.ops.ptr(Yd), len(X), rf.ops.ptr(out), rf.ops.stream()))
    return out.cpu().numpy().reshape(len(X), 9)


@pytest.mark.parametrize("name", ["ransac_m120", "ransac_m636", "ransac_grid", "ransac_remainder_only", "ransac_none", "ransac_lowinlier"])
def test_dlt_every_golden_sample(rf, name):
    g = golden(name)
    us = OO.unique_samples(g["samples"])
    X, Y = g["match1"][us], g["match2"][us]
    worst, tight, loose = G.dlt_check(dlt_device(rf, X, Y), X, Y)
    print("DLT %s: %d samples within the bound (worst ratio %.3g), %d ill-conditioned (norm only)" % (name, tight, worst, loose))


def test_dlt_seeded_and_collinear(rf):
    X, Y = dlt_quadruples(3, 2000)
    worst, tight, loose = G.dlt_check(dlt_device(rf, X, Y), X, Y)
    Xc, Yc = collinear_quadruples(3)
    G.dlt_check(dlt_device(rf, Xc, Yc), Xc, Yc, degenerate=np.ones(len(Xc), bool))
    print("DLT seeded: %d within the bound (worst ratio %.3g), %d ill-conditioned; %d exactly collinear" % (tight, worst, loose, len(Xc)))
