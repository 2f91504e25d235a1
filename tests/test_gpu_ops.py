"""Kernel-level parity of the conv / pooling / warp kernels against torch-CPU fp32 (the library calls the
reference makes) and the oracle's restatements."""
import numpy as np
import PIL.Image as Image
import pytest
import torch
import torch.nn.functional as F

import wgmma_ref as R
from oracle import model_oracle as MO
from oracle import warp_oracle as WO

pytestmark = pytest.mark.gpu


def ragged(rf, xs):
    """list of (1,C,H,W) CPU tensors -> Ragged on the GPU."""
    data = torch.cat([x[0].permute(1, 2, 0).reshape(-1, x.shape[1]) for x in xs], 0).contiguous().cuda()
    return rf.ops.Ragged(data, [(x.shape[2], x.shape[3]) for x in xs])


def close(a, b, tol):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(1.0, float(np.abs(b).max()))
    assert np.abs(a - b).max() <= tol * scale, (np.abs(a - b).max(), scale)


@pytest.mark.parametrize("cin,cout,k,stride,pad,sizes", [
    (3, 64, 3, 1, 1, [(20, 28)]), (3, 64, 7, 2, 3, [(32, 48), (18, 22)]), (64, 64, 3, 1, 1, [(24, 32), (9, 7)]),
    (64, 128, 3, 2, 1, [(24, 32)]), (64, 256, 1, 1, 0, [(13, 17), (6, 5), (1, 1)]), (256, 512, 1, 2, 0, [(14, 18)]),
    (128, 128, 3, 1, 1, [(16, 16), (16, 16)]), (49, 512, 3, 1, 1, [(6, 8)]), (128, 49, 3, 1, 1, [(6, 8)]),
    (128, 1, 3, 1, 1, [(6, 8), (6, 8)]), (1024, 256, 1, 1, 0, [(15, 20), (30, 40)]), (16, 20, 3, 1, 1, [(5, 5)])])
@pytest.mark.parametrize("relu,res", [(True, False), (True, True), (False, False)])
def test_conv2d_fp32(rf, cin, cout, k, stride, pad, sizes, relu, res):
    g = torch.Generator().manual_seed(cin * 7 + cout + k)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, k, k, generator=g) / np.sqrt(cin * k * k)
    bias = torch.randn(cout, generator=g)
    refs = [F.conv2d(x, w, bias, stride=stride, padding=pad) for x in xs]
    rs = [torch.randn(r.shape, generator=g) for r in refs] if res else None
    if res:
        refs = [a + b for a, b in zip(refs, rs)]
    if relu:
        refs = [F.relu(r) for r in refs]
    wp = w.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().cuda()
    y = rf.ops.conv2d(ragged(rf, xs), wp, bias.cuda(), cout, k, stride, pad, relu, ragged(rf, rs) if res else None, rf.ops.ENGINE_FP32)
    for i, r in enumerate(refs):
        assert tuple(y.image(i).shape) == tuple(r.shape)
        close(y.image(i).cpu(), r, 2e-5)


def test_pool_blur_norm(rf):
    g = torch.Generator().manual_seed(0)
    xs = [torch.randn(1, 64, 17, 23, generator=g), torch.randn(1, 64, 8, 6, generator=g)]
    x = ragged(rf, xs)
    for i, t in enumerate(xs):
        close(rf.ops.maxpool2d(x, 2, 1, 0).image(i).cpu(), F.max_pool2d(t, 2, 1), 0)
        close(rf.ops.maxpool2d(x, 3, 2, 1).image(i).cpu(), F.max_pool2d(t, 3, 2, 1), 0)
        close(rf.ops.blur_downsample(x, 2).image(i).cpu(), MO.blur_downsample(t, 2), 1e-6)
        close(rf.ops.blur_downsample(x, 1).image(i).cpu(), MO.blur_downsample(t, 1), 1e-6)
    t = torch.randn(1, 256, 6, 8, generator=g)
    n = rf.ops.l2norm(ragged(rf, [t]).data)
    close(n.view(1, 6, 8, 256).permute(0, 3, 1, 2).cpu(), F.normalize(t), 1e-6)
    z = torch.zeros(3, 8).cuda()
    assert torch.equal(rf.ops.l2norm(z), z)                               # eps clamp: 0 / 1e-12 = 0
    mask = torch.tensor([1, 0, 1], dtype=torch.uint8).cuda()
    m = rf.ops.l2norm(torch.ones(3, 8).cuda(), mask)
    assert float(m[1].abs().sum()) == 0 and abs(float(m[0].norm()) - 1) < 1e-6


def test_corr_neigh_and_heads_epilogues(rf):
    g = torch.Generator().manual_seed(1)
    a = F.normalize(torch.randn(2, 256, 6, 8, generator=g))
    b = F.normalize(torch.randn(2, 256, 6, 8, generator=g))
    got = rf.model.CorrNeigh(7)(a.cuda(), b.cuda()).cpu()
    close(got, MO.corr_neigh(a, b, 7), 1e-6)
    logits = torch.randn(2, 49, 5, 9, generator=g) * 3
    p = F.softmax(logits, dim=1)
    gx = (torch.arange(49) % 7 - 3).float().view(1, 49, 1, 1)
    gy = (torch.arange(49) // 7 - 3).float().view(1, 49, 1, 1)
    ref = torch.cat(((p * gx).sum(1, keepdim=True) / 9 * 2, (p * gy).sum(1, keepdim=True) / 5 * 2), 1)
    close(rf.ops.softmax_flow(rf.ops.Ragged.from_nchw(logits.cuda()), 7).cpu(), ref, 1e-6)
    x = torch.randn(1000, generator=g) * 5
    close(rf.ops.sigmoid(x.cuda()).cpu(), torch.sigmoid(x), 1e-6)


@pytest.mark.parametrize("n,c,h,w,k,ldo,mode", [(1, 256, 60, 80, 7, 64, 2), (2, 256, 6, 8, 7, 49, 0), (1, 64, 5, 3, 7, 64, 1),
                                                (3, 128, 9, 11, 3, 16, 2), (1, 256, 1, 1, 7, 64, 0)])
def test_corr_neigh_pair_is_bit_identical_to_two_calls(rf, n, c, h, w, k, ldo, mode):
    """rf_corr_neigh_pair_nhwc: CorrNeigh(x, y) and CorrNeigh(y, x) from one launch (yx[p][d] = xy[p+d][-d], each dot
    product stored twice) == two rf_corr_neigh_nhwc launches, bit for bit, for fp32 / TF32-rounded / fp16 outputs."""
    g = torch.Generator().manual_seed(n * 100 + h)
    a = rf.ops.Ragged.from_nchw(F.normalize(torch.randn(n, c, h, w, generator=g)).cuda())
    b = rf.ops.Ragged.from_nchw(F.normalize(torch.randn(n, c, h, w, generator=g)).cuda())
    xy, yx = rf.ops.corr_neigh(a, b, k, ldo, mode), rf.ops.corr_neigh(b, a, k, ldo, mode)
    pxy, pyx, both = rf.ops.corr_neigh_pair(a, b, k, ldo, mode)
    torch.cuda.synchronize()
    assert pxy.data.dtype == xy.data.dtype and both.data.shape == (2 * n * h * w, ldo) and both.hw == xy.hw + yx.hw
    assert torch.equal(pxy.data, xy.data) and torch.equal(pyx.data, yx.data)
    assert torch.equal(both.data[:n * h * w], xy.data) and torch.equal(both.data[n * h * w:], yx.data)


def corr_neigh_ref(x, y, k):
    """fp64 CorrNeigh(x, y) of (N, C, h, w) CPU tensors as [N*h*w, k*k] rows (tap i*k + j reads y at (r + i - k//2,
    c + j - k//2), zero outside), and the same on |x|, |y|."""
    x, y, p = x.double(), y.double(), k // 2
    h, w = x.shape[2], x.shape[3]
    yp, ap = F.pad(y, (p, p, p, p)), F.pad(y.abs(), (p, p, p, p))
    taps = [(i, j) for i in range(k) for j in range(k)]
    ref = torch.stack([(x * yp[:, :, i:i + h, j:j + w]).sum(1) for i, j in taps], -1)
    absref = torch.stack([(x.abs() * ap[:, :, i:i + h, j:j + w]).sum(1) for i, j in taps], -1)
    return ref.reshape(-1, k * k), absref.reshape(-1, k * k)


@pytest.mark.parametrize("n,c,h,w,ldo", [(1, 256, 60, 80, 64), (2, 256, 6, 8, 49), (1, 64, 5, 3, 64), (1, 1024, 4, 7, 64), (1, 256, 1, 1, 96)])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_corr_neigh_kernels_match_fp64_reference(rf, k, n, c, h, w, ldo):
    """corr_neigh7_kernel (k = 7: 49 sums in registers, one multi-value butterfly, coalesced row store) and corr_neigh_kernel
    (other odd k: one warp reduction per tap) against fp64, element by element, in every output mode (fp32, TF32-rounded, fp16),
    single and pair: |y - ref| <= r_out |ref| + gamma_C (1 + r_out) sum |x y| + atol, with gamma_C = C u / (1 - C u) the fp32
    accumulation bound of a C-term sum (u = 2^-24).  Padding channels are zero, the pair's halves equal the two single calls bit
    for bit, and the split form (engine 4) rebuilds both halves to 2^-21."""
    g = torch.Generator().manual_seed(n * 10 + h + k)
    xa = F.normalize(torch.randn(n, c, h, w, generator=g))
    xb = F.normalize(torch.randn(n, c, h, w, generator=g))
    a, b = rf.ops.Ragged.from_nchw(xa.cuda()), rf.ops.Ragged.from_nchw(xb.cuda())
    refs = {"xy": corr_neigh_ref(xa, xb, k), "yx": corr_neigh_ref(xb, xa, k)}
    gamma = c * 2.0 ** -24 / (1 - c * 2.0 ** -24)
    for mode, r_out, atol in ((0, 0.0, 0.0), (1, R.R_TF32, 0.0), (2, R.R_F16, R.ATOL["f16"])):
        xy, yx = rf.ops.corr_neigh(a, b, k, ldo, mode).data, rf.ops.corr_neigh(b, a, k, ldo, mode).data
        pxy, pyx, _ = rf.ops.corr_neigh_pair(a, b, k, ldo, mode)
        torch.cuda.synchronize()
        assert torch.equal(pxy.data, xy) and torch.equal(pyx.data, yx), mode
        for name, got in (("xy", xy), ("yx", yx)):
            ref, absref = refs[name]
            R.check(got[:, :k * k].cpu(), ref, absref, r_out, gamma * (1 + r_out), atol, "k %d mode %d %s" % (k, mode, name))
            assert not bool(got[:, k * k:].any()), "padding channels"
    P = n * h * w
    full, swapped = rf.ops.corr_neigh(a, b, k, ldo, 0).data, rf.ops.corr_neigh(b, a, k, ldo, 0).data
    c12, both = rf.ops.corr_neigh_pair_split(a, b, k, ldo)
    c12, both = c12.data, both.data
    assert c12.shape == (2, P, ldo) and both.shape == (2, 2 * P, ldo)
    assert (rf.ops.from_split(c12) - full).abs().max().item() < 2.0 ** -21
    assert torch.equal(both[:, :P], c12)
    assert (rf.ops.from_split(both[:, P:].contiguous()) - swapped).abs().max().item() < 2.0 ** -21


@pytest.mark.parametrize("h,w,skip", [(33, 47, 0), (16, 16, 0), (1, 3, 0), (33, 47, 1), (480, 640, 0), (7, 4, 4)])
def test_preproc_bit_exact(rf, h, w, skip):
    """ToTensor (+ Normalize) in torchvision's op order, bit exact.  Covers the 12-bytes-per-thread kernel with and without a
    tail, inputs shorter than one group, and a view that starts `skip` pixels into the buffer (3 * skip bytes: the
    vector kernel needs 4-byte alignment, odd offsets take the byte kernel)."""
    rs = np.random.RandomState(h * w + skip)
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    flat = torch.from_numpy(img).reshape(-1, 3)
    t = flat[skip:].float().div(255)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3)
    dev = flat.cuda()[skip:]
    assert torch.equal(rf.ops.preproc_u8(dev, True).cpu(), (t - mean) / std)
    assert torch.equal(rf.ops.preproc_u8(dev, False).cpu(), t)


@pytest.mark.parametrize("size", [(96, 64), (20, 11), (53, 80), (1280, 960), (320, 240)])
def test_device_lanczos_bit_exact_vs_pil(rf, size):
    rs = np.random.RandomState(1)
    img = rs.randint(0, 256, (480, 640, 3)).astype(np.uint8) if size[0] >= 320 else rs.randint(0, 256, (37, 53, 3)).astype(np.uint8)
    ref = np.asarray(Image.fromarray(img).resize(size, resample=Image.LANCZOS))
    got = rf.ops.resize_lanczos_u8(torch.from_numpy(img).cuda(), size[0], size[1]).cpu().numpy()
    assert np.array_equal(got, ref)


def test_warp_grid_and_grid_sample(rf):
    rs = np.random.RandomState(2)
    Hs = np.stack([np.eye(3) + rs.uniform(-0.1, 0.1, (3, 3)) for _ in range(3)]).astype(np.float32)
    g = rf.ops.warp_grid(torch.from_numpy(Hs).cuda(), 31, 45)
    close(g.cpu(), WO.warp_grid(Hs, 31, 45), 2e-6)
    w = rf.kornia_geometry.HomographyWarper(31, 45).warp_grid(torch.from_numpy(Hs).cuda())
    assert torch.equal(w, g)
    img = torch.rand(3, 3, 20, 26)
    grid = WO.warp_grid(Hs, 31, 45) * 1.2                                  # some samples fall outside
    for ac in (False, True):
        ref = F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=ac)
        close(rf.ops.grid_sample(img.cuda(), grid.cuda(), ac).cpu(), ref, 2e-6)
        cl = img.cuda().contiguous(memory_format=torch.channels_last)
        close(rf.ops.grid_sample(cl, grid.cuda(), ac).cpu(), ref, 2e-6)
    x = torch.rand(2, 2, 6, 8)
    close(rf.ops.upsample_bilinear(x.cuda(), (48, 64)).cpu(), F.interpolate(x, size=(48, 64), mode="bilinear"), 1e-6)
    big = torch.rand(1, 1, 48, 64)
    close(rf.ops.upsample_bilinear(big.cuda(), (3, 4)).cpu(), F.interpolate(big, size=(3, 4), mode="bilinear"), 1e-6)


@pytest.mark.parametrize("m21", [False, True])
def test_compose_fine(rf, m21):
    rs = np.random.RandomState(3)
    H, W = 48, 64
    f8 = torch.from_numpy((rs.randn(1, 2, 6, 8) * 0.05).astype(np.float32))
    m12 = torch.from_numpy(rs.rand(1, 1, 6, 8).astype(np.float32))
    m21t = torch.from_numpy(rs.rand(1, 1, 6, 8).astype(np.float32))
    Hm = (np.eye(3) + rs.uniform(-0.1, 0.1, (3, 3))).astype(np.float32)[None]
    coarse = WO.warp_grid(Hm, H, W)
    grid = WO.base_grid(H, W)
    flow12, flowUp = WO.compose_fine(f8, coarse, grid, clamp=True)
    match = WO.interpolate_bilinear(m12, (H, W))
    if m21:
        match = match * WO.grid_sample(WO.interpolate_bilinear(m21t, (H, W)), flowUp)
    match = match * WO.inside_mask(flow12)
    g12, gm, gup = rf.ops.compose_fine(f8.cuda(), m12.cuda(), m21t.cuda() if m21 else None, coarse.cuda(), want_flowUp=True)
    close(gup.cpu(), flowUp, 2e-6)
    close(g12.cpu(), flow12, 5e-6)
    # the inside-mask is a hard threshold at |flow| == 1: compare away from the threshold
    far = (np.abs(np.abs(flow12.numpy()) - 1) > 1e-4).all(-1)[0]
    assert np.abs(gm.cpu().numpy()[0, 0] - match.numpy()[0, 0])[far].max() < 5e-6
    # no clamp (quick_start/align2images.py:91-95)
    f_nc, _ = WO.compose_fine(f8, coarse, grid, clamp=False)
    g_nc, _, _ = rf.ops.compose_fine(f8.cuda(), None, None, coarse.cuda(), clamp=False, want_match=False)
    close(g_nc.cpu(), f_nc, 5e-6)


def test_warp_grid_reference_internal_consistency(rf):
    """rf_warp_grid under the pin the reference itself offers for kornia 0.1.4 (see tests/test_oracle_golden.py): the identity
    (and any power-of-two multiple of it) reproduces, bit for bit, the base grid the fine flow is added to on this side
    (pipeline.base_grid = torch.linspace on the device = what compose_fine regenerates) - the consistency the reference has
    between kornia's meshgrid and the drivers' own linspace grid, both built by the same CPU linspace - and Homography(X, Y)
    -> warp_grid carries the four target sample points onto their source points.  (CPU torch.linspace itself is only defined
    up to an ulp: its vectorised kernel adds lane offsets to a per-vector base, so it depends on the host's SIMD width.)"""
    from oracle import outil_oracle as OO
    from oracle import warp_oracle as WO
    for h, w in ((48, 64), (30, 41), (2, 2), (480, 640)):
        for scale in (1.0, 4.0):
            got = rf.ops.warp_grid(scale * torch.eye(3).cuda().view(1, 3, 3), h, w)
            assert torch.equal(got, rf.pipeline.base_grid(h, w))
            assert (got.cpu() - WO.base_grid(h, w)).abs().max().item() <= 1.2e-7
    rs = np.random.RandomState(0)
    h, w = 33, 47
    Y = np.array([[-1, -1, 1], [1, -1, 1], [-1, 1, 1], [1, 1, 1]], dtype=np.float32)
    Hgt = np.eye(3) + rs.uniform(-0.2, 0.2, (3, 3))
    Hgt[2, :2] = rs.uniform(-0.05, 0.05, 2)
    X = Y @ Hgt.T
    X = (X / X[:, 2:]).astype(np.float32)
    H = rf.outil.Homography(torch.from_numpy(X[None]).cuda(), torch.from_numpy(Y[None]).cuda())
    np.testing.assert_allclose(H.cpu().numpy(), OO.Homography(X[None], Y[None]), atol=2e-6)
    g = rf.kornia_geometry.HomographyWarper(h, w).warp_grid(H)[0].cpu().numpy()
    corners = np.stack([g[0, 0], g[0, w - 1], g[h - 1, 0], g[h - 1, w - 1]])
    assert np.abs(corners - X[:, :2]).max() < 1e-5
