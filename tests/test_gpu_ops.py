"""Kernel-level parity of the pooling / correlation / warp kernels against torch-CPU fp32 (the library calls the
reference makes) and the oracle's restatements.  The exact-FMA convolution is held bit for bit to its FMA chains in
tests/test_gpu_simt_exact.py."""
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


def test_corr_neigh_module_matches_oracle(rf):
    """model.CorrNeigh(7) (NCHW in and out) against the oracle's CorrNeigh; the kernels themselves are held to fp64 below,
    the pooling, blur, L2 normalisation and head epilogues in tests/test_gpu_layer_ops.py."""
    g = torch.Generator().manual_seed(1)
    a = F.normalize(torch.randn(2, 256, 6, 8, generator=g))
    b = F.normalize(torch.randn(2, 256, 6, 8, generator=g))
    got = rf.model.CorrNeigh(7)(a.cuda(), b.cuda()).cpu()
    close(got, MO.corr_neigh(a, b, 7), 1e-6)


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
