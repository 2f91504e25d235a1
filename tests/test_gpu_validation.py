"""The MegaDepth validation (train/validation.py) on the device.

  affine sample : ``rf_affine_sample_u8`` against an fp64 restatement within geometry_ref's sampling bound, and against
                  torch's ``F.affine_grid`` + ``F.grid_sample`` on the GPU within that bound widened by the grid's cuBLAS
                  product (any order of the three terms, fused or not: gamma_3 of |t0 x| + |t1 y| + |t2| per coordinate,
                  times W / 2 pixels per unit and the local Lipschitz constant of the image)
  grid helpers  : the affine base grid equals torch's (identity theta: the bmm is exact) and ``lin11`` equals the CPU
                  ``torch.linspace(-1, 1, n)`` the reference adds to the flow, bit for bit
  keypoint tail : ``rf_val_keypoints`` against an fp64 restatement (counts equal for every keypoint certified away from a
                  threshold), torch's index rule, the error word, zero keypoints, accumulation; against the reference's
                  torch composition on the same device operands
  dataset       : ``validation`` against the reference's golden on engines fp32 and f16x3, with no host synchronisation
                  in the loop, and the CLI on two checkpoints
"""
import os
import pickle

import numpy as np
import PIL.Image as Image
import pytest
import torch
import torch.nn.functional as F

from conftest import golden
from geometry_ref import U, bilinear_zeros, coord_delta, gamma, lin11, unnormalize64
from oracle import synth
from oracle import validation_oracle as VO
from oracle.gen_validation_golden import pair_images

pytestmark = pytest.mark.gpu
f32 = np.float32


def affine_base(n):
    """The kernel's ``affine_base``: CUDA linspace * (n - 1), times the fp32 reciprocal of n (ATen's division by a scalar)."""
    if n <= 1:
        return np.zeros(n, dtype=f32)
    return (lin11(np.arange(n), n) * f32(n - 1)).astype(f32) * (f32(1) / f32(n))


def affine_image(theta, h, w):
    """The h x w affine grid in fp64 from the kernel's fp32 base coordinates: (2, h, w) values and (2,) bounds on the sum of
    the terms' magnitudes."""
    t = np.asarray(theta, dtype=np.float64).reshape(2, 3)
    x = affine_base(w).astype(np.float64)[None, :]
    y = affine_base(h).astype(np.float64)[:, None]
    P = np.stack([t[k, 0] * x + t[k, 1] * y + t[k, 2] for k in range(2)])
    S = np.abs(t).sum(axis=1)
    return P, S


def _dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda() if dtype is None else torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _src(seed, h, w):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


AFFINE_CASES = [  # (Hin, Win, h, w, theta)
    (37, 53, 37, 53, [[1, 0, 0], [0, 1, 0]]),                                      # odd sizes, identity
    (100, 130, 61, 77, [[0.9, -0.2, 0.05], [0.15, 1.1, -0.08]]),                   # source != output, partial last block
    (64, 80, 48, 64, [[1.4, 0.1, 0.5], [-0.05, 1.3, -0.45]]),                     # partly outside
    (480, 640, 480, 640, [[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]]),
]


@pytest.mark.parametrize("case", range(len(AFFINE_CASES)))
def test_affine_sample_fp64_and_torch(rf, case):
    Hin, Win, h, w, theta = AFFINE_CASES[case]
    src = _src(case, Hin, Win)
    th = np.asarray(theta, dtype=f32)
    got = rf.validation.affine_sample_u8(_dev(th.reshape(-1)), _dev(src), h, w).cpu().numpy().astype(np.float64)
    got = got.reshape(h, w, 3).transpose(2, 0, 1)
    Pimg = (src.astype(f32) / f32(255)).transpose(2, 0, 1)
    G, S = affine_image(th, h, w)
    ix, iy = unnormalize64(G[0], Win, False), unnormalize64(G[1], Hin, False)
    val, absval, Lx, Ly, outside = bilinear_zeros(Pimg, ix, iy)
    dx, dy = Win / 2.0 * gamma(2) * S[0], Hin / 2.0 * gamma(2) * S[1]
    allow = gamma(7) * absval + Lx * (coord_delta(ix) + dx) + Ly * (coord_delta(iy) + dy)
    assert np.all(np.abs(got - val) <= allow), np.max(np.abs(got - val) - allow)
    # torch: the same base grid, theta applied by cuBLAS (each side within gamma_3 of the exact product)
    grid = F.affine_grid(torch.from_numpy(th)[None].cuda(), (1, 3, h, w), align_corners=False)
    ref = F.grid_sample(torch.from_numpy(Pimg.copy())[None].cuda(), grid, align_corners=False)[0].cpu().numpy().astype(np.float64)
    dx_t, dy_t = Win / 2.0 * (gamma(2) + gamma(3)) * S[0], Hin / 2.0 * (gamma(2) + gamma(3)) * S[1]
    allow_t = 2 * gamma(7) * absval + Lx * (2 * coord_delta(ix) + dx_t) + Ly * (2 * coord_delta(iy) + dy_t)
    assert np.all(np.abs(got - ref) <= allow_t), np.max(np.abs(got - ref) - allow_t)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_affine_sample_nonfinite_theta_is_zeros(rf, bad):
    src = _src(9, 40, 56)
    for k in range(6):
        th = np.array([1, 0, 0, 0, 1, 0], dtype=f32)
        th[k] = bad
        out = torch.full((33 * 47, 3), 7.0, device="cuda")
        rf.validation.affine_sample_u8(_dev(th), _dev(src), 33, 47, out=out)
        assert torch.count_nonzero(out).item() == 0, (k, bad)


def test_affine_base_grid_is_torchs():
    """With the identity theta the cuBLAS product is exact, so F.affine_grid returns the base grid itself."""
    for h, w in [(1, 1), (2, 3), (37, 53), (480, 640), (480, 720), (608, 480), (1024, 768)]:
        g = F.affine_grid(torch.eye(2, 3, device="cuda")[None], (1, 3, h, w), align_corners=False)[0].cpu().numpy()
        np.testing.assert_array_equal(g[0, :, 0], affine_base(w))
        np.testing.assert_array_equal(g[:, 0, 1], affine_base(h))


def _fma32(a, b, c):
    """fl32(a * b + c): the fp64 product of two float32 values is exact, and so is its sum with the float32 c here."""
    return f32(np.float64(a) * np.float64(b) + np.float64(c))


@pytest.mark.parametrize("theta", [[[1, 0, 0], [0, 1, 0]], [[0.9, -0.2, 0.05], [0.15, 1.1, -0.08]]])
def test_kernel_affine_grid_is_exact(rf, theta):
    """The kernel's own affine grid points, read back bit for bit.  With a 1 x 1 flowDown8 = v the upsampled flow is v
    exactly, and at keypoint (0, 0) the fine flow is v - 1 (lin11(0) = -1).  For v = (2j + 1) / W with 2j + 1 a multiple
    of W's odd part, v is a float32, v - 1 and the unnormalised coordinate (v W - 1) / 2 = j are exact, so the composition
    samples the affine grid at pixel (jy, jx) with the weights 1, 0, 0, 0: the composed flow flow_out[2:] IS
    affine_grid_point(theta, jy, jx).  It must equal affine_base (which equals torch's base grid, test above) with theta
    applied as one FMA chain.  This pins the base grid's rounding order, not just a sampling bound."""
    th = np.asarray(theta, dtype=f32)
    for H, W in [(480, 640), (480, 720), (608, 480), (64, 64), (37, 53)]:
        def centres(n):
            m = n
            while m % 2 == 0:
                m //= 2
            return [(m * (2 * q + 1) - 1) // 2 for q in range(n) if (m * (2 * q + 1) - 1) // 2 < n]
        jx, jy = centres(W), centres(H)
        probes = min(40, max(len(jx), len(jy)))
        bx, by = affine_base(W), affine_base(H)
        for t in range(probes):
            x, y = jx[t * len(jx) // probes], jy[t * len(jy) // probes]
            v = np.array([(2 * x + 1) / W, (2 * y + 1) / H], dtype=f32)
            _, _, fo = _tail(rf, v.reshape(1, 2, 1, 1), th, (H, W), (H, W), [[0, 0, 0, 0]])
            assert fo[0, 0] == v[0] - 1 and fo[0, 1] == v[1] - 1, (H, W, x, y)
            want = [f32(_fma32(th[r, 1], by[y], f32(th[r, 0] * bx[x])) + th[r, 2]) for r in range(2)]
            assert fo[0, 2] == want[0] and fo[0, 3] == want[1], (H, W, x, y, fo[0, 2:], want)


def _tail(rf, flow8, theta, size_t, size_s, kpts, pair=0, acc=None, want=True):
    n = len(kpts)
    acc = rf.validation.new_counts() if acc is None else acc
    d = torch.full((n,), -1.0, dtype=torch.float64, device="cuda") if want else None
    fo = torch.full((n, 4), 7.0, dtype=torch.float32, device="cuda") if want else None
    kp = _dev(np.asarray(kpts, dtype=np.int32).reshape(-1, 4))
    rf.validation.val_keypoints(_dev(flow8, np.float32), _dev(np.asarray(theta, f32).reshape(-1)), size_t, size_s, kp,
                                _dev(np.array([n], np.int32)), acc, pair, d, fo)
    return acc, (d.cpu().numpy() if want else None), (fo.cpu().numpy() if want else None)


def test_lin11_is_the_cpu_linspace(rf):
    """The grid validation.py:93-95 adds: CPU torch.linspace(-1, 1, n), read back through flow_out with a zero flow."""
    for n in range(16, 2049, 16):
        i = np.arange(n)
        _, _, fo = _tail(rf, np.zeros((1, 2, n // 8, n // 8)), np.eye(2, 3), (n, n), (n, n), np.stack([i, i, i, i], 1))
        want = torch.linspace(-1, 1, n).numpy()
        np.testing.assert_array_equal(fo[:, 0], want, err_msg="n=%d" % n)
        np.testing.assert_array_equal(fo[:, 1], want, err_msg="n=%d" % n)


def tail_ref(flow8, theta, H, W, hA, wA, kpts):
    """fp64 restatement of rf_val_keypoints for in-range keypoints: (flow (n, 2), its allowance, dist, its allowance)."""
    f8 = np.asarray(flow8, dtype=f32)[0]
    h8, w8 = f8.shape[1:]
    k = np.asarray(kpts, dtype=np.int64)
    xb, yb = np.where(k[:, 2] < 0, k[:, 2] + W, k[:, 2]), np.where(k[:, 3] < 0, k[:, 3] + H, k[:, 3])
    rh = f32(h8 - 1) / f32(H - 1) if H > 1 else f32(0)
    rw = f32(w8 - 1) / f32(W - 1) if W > 1 else f32(0)
    h1r, w1r = (rh * yb.astype(f32)).astype(f32), (rw * xb.astype(f32)).astype(f32)
    h1, w1 = h1r.astype(np.int64), w1r.astype(np.int64)
    h1p, w1p = (h1 < h8 - 1).astype(np.int64), (w1 < w8 - 1).astype(np.int64)
    h1l, w1l = (h1r - h1.astype(f32)).astype(f32), (w1r - w1.astype(f32)).astype(f32)
    h0l, w0l = (f32(1) - h1l).astype(f32), (f32(1) - w1l).astype(f32)
    fl, ef = [], []
    for c, (g, pos) in enumerate(((lin11(xb, W), xb), (lin11(yb, H), yb))):
        v = f8[c].astype(np.float64)
        a, b, cc, d = v[h1, w1], v[h1, w1 + w1p], v[h1 + h1p, w1], v[h1 + h1p, w1 + w1p]
        blend = h0l * (w0l * a + w1l * b) + h1l * (w0l * cc + w1l * d)
        ab = h0l * (w0l * abs(a) + w1l * abs(b)) + h1l * (w0l * abs(cc) + w1l * abs(d))
        s = blend + g.astype(np.float64)
        fl.append(np.clip(s, -1, 1))
        ef.append(gamma(4) * ab + U * np.abs(s))
    fx, fy = fl
    P, S = affine_image(theta, H, W)
    ix, iy = unnormalize64(fx, W, False), unnormalize64(fy, H, False)
    val, absval, Lx, Ly, _ = bilinear_zeros(P, ix, iy)
    allow_o = gamma(7) * absval + Lx * (coord_delta(ix) + W / 2.0 * ef[0]) + Ly * (coord_delta(iy) + H / 2.0 * ef[1]) \
        + gamma(2) * S[:, None]
    ex, ey = (val[0] + 1) * 0.5 * (wA - 1), (val[1] + 1) * 0.5 * (hA - 1)
    aex = (wA - 1) / 2.0 * allow_o[0] + gamma(2) * np.abs(ex)
    aey = (hA - 1) / 2.0 * allow_o[1] + gamma(2) * np.abs(ey)
    dist = np.hypot(ex - k[:, 0], ey - k[:, 1])
    return np.stack([fx, fy], 1), np.stack(ef, 1), dist, aex + aey + 1e-12 * (dist + 1)


@pytest.mark.parametrize("theta", [[[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]], [[1.3, 0.05, 0.35], [-0.04, 1.25, -0.3]]])
def test_keypoint_tail_fp64(rf, theta):
    rs = np.random.RandomState(5)
    h8, w8, hA, wA = 15, 19, 104, 136
    H, W = 8 * h8, 8 * w8
    flow8 = rs.uniform(-0.25, 0.25, (1, 2, h8, w8)).astype(f32)
    n = 3000
    kp = np.stack([rs.randint(-5, wA + 5, n), rs.randint(-5, hA + 5, n), rs.randint(-W, W, n), rs.randint(-H, H, n)], 1)
    kp[:4, 2:] = [[W - 1, H - 1], [-1, -1], [-W, -H], [0, 0]]
    acc, d, fo = _tail(rf, flow8, theta, (H, W), (hA, wA), kp)
    fl, ef, dref, adist = tail_ref(flow8, theta, H, W, hA, wA, kp)
    assert np.all(np.abs(fo[:, :2] - fl) <= ef), np.max(np.abs(fo[:, :2] - fl) - ef)
    assert np.all(np.abs(d - dref) <= adist), np.max(np.abs(d - dref) - adist)
    counts, err = rf.validation.read_counts(acc.cpu().numpy())
    thr = rf.validation.PIXEL_GRID.reshape(-1)
    assert err is None and counts[-1] == n
    np.testing.assert_array_equal(counts[:-1], (d[:, None] < thr).sum(0))
    certified = (np.abs(dref[:, None] - thr) > adist[:, None]).all(1)
    assert certified.mean() > 0.99
    np.testing.assert_array_equal((d[certified, None] < thr), (dref[certified, None] < thr))


def test_keypoint_tail_index_rule_and_accumulation(rf):
    rs = np.random.RandomState(6)
    h8, w8 = 6, 8
    H, W = 48, 64
    flow8 = rs.uniform(-0.2, 0.2, (1, 2, h8, w8)).astype(f32)
    theta = [[1, 0, 0], [0, 1, 0]]
    # a negative index wraps once: (-1, -W) reads the same pixel as (H - 1, 0)
    _, d1, _ = _tail(rf, flow8, theta, (H, W), (H, W), [[3, 4, 0, H - 1], [3, 4, -W, -1]])
    assert d1[0] == d1[1]
    # out of range (W, -H - 1, ...): the error word records the first pair; the other keypoints still count
    acc = rf.validation.new_counts()
    _tail(rf, flow8, theta, (H, W), (H, W), [[3, 4, 5, 5], [3, 4, W, 0]], pair=7, acc=acc)
    _tail(rf, flow8, theta, (H, W), (H, W), [[3, 4, 0, -H - 1]], pair=3, acc=acc)
    _tail(rf, flow8, theta, (H, W), (H, W), [[3, 4, 1, 1]], pair=9, acc=acc)
    counts, err = rf.validation.read_counts(acc.cpu().numpy())
    assert err == 3 and counts[-1] == 2
    # zero keypoints: nothing counted
    acc0, _, _ = _tail(rf, flow8, theta, (H, W), (H, W), np.zeros((0, 4)), want=False)
    counts0, err0 = rf.validation.read_counts(acc0.cpu().numpy())
    assert err0 is None and not counts0.any()
    # accumulating over calls equals the sum of separate calls
    kp = np.stack([rs.randint(0, W, 500), rs.randint(0, H, 500), rs.randint(0, W, 500), rs.randint(0, H, 500)], 1)
    both = rf.validation.new_counts()
    parts = []
    for part in (kp[:123], kp[123:]):
        _tail(rf, flow8, theta, (H, W), (H, W), part, acc=both, want=False)
        parts.append(rf.validation.read_counts(_tail(rf, flow8, theta, (H, W), (H, W), part, want=False)[0].cpu().numpy())[0])
    np.testing.assert_array_equal(rf.validation.read_counts(both.cpu().numpy())[0], parts[0] + parts[1])


def test_keypoint_tail_against_torch_composition(rf):
    """validation.py:93-107 and alignmentError as the reference runs them, on the same device flowDown8 and theta."""
    rs = np.random.RandomState(8)
    for (h8, w8, hA, wA, theta) in [(60, 80, 480, 640, [[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]]),
                                    (60, 90, 480, 720, [[1.3, 0.05, 0.35], [-0.04, 1.25, -0.3]])]:
        H, W = 8 * h8, 8 * w8
        flow8 = torch.from_numpy(rs.uniform(-0.05, 0.05, (1, 2, h8, w8)).astype(f32)).cuda()
        th = torch.tensor(theta, dtype=torch.float32, device="cuda")
        n = 2000
        kp = np.stack([rs.randint(0, wA, n), rs.randint(0, hA, n), rs.randint(-W, W, n), rs.randint(-H, H, n)], 1)
        _, d, fo = _tail(rf, flow8.cpu().numpy(), theta, (H, W), (hA, wA), kp)
        with torch.no_grad():
            flowUp = F.interpolate(flow8, scale_factor=8, mode="bilinear", align_corners=True)
            gy = torch.linspace(-1, 1, steps=H).view(1, -1, 1, 1).expand(1, H, W, 1)
            gx = torch.linspace(-1, 1, steps=W).view(1, 1, -1, 1).expand(1, H, W, 1)
            flowCoarse = torch.clamp(flowUp.permute(0, 2, 3, 1) + torch.cat((gx, gy), dim=3).cuda(), min=-1, max=1)
            flowGlobalT = F.affine_grid(th[None], (1, 3, H, W), align_corners=False)
            flowFinal = F.grid_sample(flowGlobalT.permute(0, 3, 1, 2), flowCoarse, align_corners=False).permute(0, 2, 3, 1)
            estimY = (flowFinal[..., 0] + 1) * 0.5 * (wA - 1)
            estimX = (flowFinal[..., 1] + 1) * 0.5 * (hA - 1)
        yb, xb = torch.from_numpy(kp[:, 3]).cuda(), torch.from_numpy(kp[:, 2]).cuda()
        ex, ey = estimY[0, yb, xb].double().cpu().numpy(), estimX[0, yb, xb].double().cpu().numpy()
        fc = flowCoarse[0, yb, xb].cpu().numpy()
        dref = np.sqrt((ex - kp[:, 0]) ** 2 + (ey - kp[:, 1]) ** 2)
        fo = fo[:, :2]
        assert np.all(np.abs(fo - fc) <= 4 * U)                        # the fine flow: torch's upsampling and CPU grid
        print("\n[composition %dx%d] fine flow bit-identical to torch's at %d of %d keypoints" % (H, W, int((fo == fc).all(1).sum()), n))
        P, S = affine_image(theta, H, W)
        ix, iy = unnormalize64(fc[:, 0].astype(np.float64), W, False), unnormalize64(fc[:, 1].astype(np.float64), H, False)
        _, absval, Lx, Ly, _ = bilinear_zeros(P, ix, iy)
        tap = (gamma(2) + gamma(3)) * S[:, None]                      # the two sides' affine grid values
        ao = 2 * gamma(7) * absval + tap + Lx * (2 * coord_delta(ix) + W / 2.0 * 4 * U) + Ly * (2 * coord_delta(iy) + H / 2.0 * 4 * U)
        tol = (wA - 1) / 2.0 * ao[0] + (hA - 1) / 2.0 * ao[1] + gamma(4) * (np.abs(ex) + np.abs(ey)) + 1e-12 * (dref + 1)
        assert np.all(np.abs(d - dref) <= tol), np.max(np.abs(d - dref) - tol)


# --------------------------------------------------------------------------- the whole dataset
@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    """The golden's five pairs as files, CSV rows and thetas, with the oracle's fine flow per pair."""
    g = golden("validation_megadepth")
    root = tmp_path_factory.mktemp("megadepth_val")
    rows, thetas, flows, images = [], [], [], []
    states = {"netFeatCoarse": synth.feature_extractor_state(int(g["feat_seed"])),
              "netFlowCoarse": synth.net_flow_coarse_state(int(g["flow_seed"]))}
    for i in range(int(g["n_pairs"])):
        row = {c: str(g["%s%d" % (c, i)]) for c in ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB")}
        Is, It = pair_images(g["spec%d" % i])
        os.makedirs(root / row["scene"], exist_ok=True)
        Image.fromarray(Is).save(root / row["scene"] / row["source_image"])
        Image.fromarray(It).save(root / row["scene"] / row["target_image"])
        _, f8 = VO.pair_distances(Is, It, g["theta%d" % i], row["XA"], row["YA"], row["XB"], row["YB"], states, with_flow=True)
        rows.append(row)
        thetas.append(g["theta%d" % i])
        flows.append(f8)
        images.append((Is, It))
    import pandas as pd
    return dict(g=g, root=str(root), df=pd.DataFrame(rows, dtype=str), thetas=thetas, flows=flows, images=images)


def _network(rf, flow_seed=1):
    net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7), "netFlowCoarse": rf.model.NetFlowCoarse(7)}
    net["netFeatCoarse"].load_state_dict(synth.feature_extractor_state(0))
    net["netFlowCoarse"].load_state_dict(synth.net_flow_coarse_state(flow_seed))
    for m in net.values():
        m.cuda()
        m.eval()
    return net


# The largest |flowDown8 - reference| an engine may show on the golden's pairs: the fine networks on the exact-FMA engine and
# on the fp32-grade split engine stay within a few 1e-7 of the reference's CPU fp32 flow (bench.py's stage-isolated parity
# reports 3.2e-7 for f16x3 at 480 x 640); 4e-6 leaves a margin of about ten.  A wiring error (a swapped correlation, the
# target normalised, the halves exchanged) moves the flow by 1e-3 or more.
E8_MAX = {"fp32": 4e-6, "f16x3": 4e-6}
MAX_ASIDE = 6                     # 2 % of the golden's 300 keypoints


@pytest.mark.parametrize("engine", ["fp32", "f16x3"])
def test_dataset_matches_the_reference(rf, dataset, engine):
    """Per-keypoint distances within a tolerance derived from a FIXED bound on the engine's flow error, and the precision
    vector equal to the reference's once the (at most MAX_ASIDE) keypoints within that tolerance of a threshold are set
    aside.

    The measured flow error e8 = max |flowDown8 - oracle| of each pair must stay below E8_MAX[engine].  The x8 upsampling is
    a convex combination and the clamp is 1-Lipschitz, so the fine flow at a keypoint moves by at most E8_MAX, i.e.
    E8_MAX W / 2 (E8_MAX H / 2) pixels of the affine grid image, which moves the composed flow by at most Lx (Ly) times
    that, Lx / Ly the image's local Lipschitz constants (geometry_ref.bilinear_zeros, borders included), and the distance by
    (wA - 1) / 2 and (hA - 1) / 2 times the two components.  Twice that, plus 1e-4 px for the fp32 roundings on both sides."""
    V, g = rf.validation, dataset["g"]
    prev = rf.model.get_engine()
    rf.model.set_engine(engine)
    try:
        net = _network(rf)
        prec = V.validation(dataset["df"], dataset["root"], dataset["thetas"], net, None)
        acc = V.new_counts()
        thr = V.PIXEL_GRID.reshape(-1)
        e = E8_MAX[engine]
        keep_gpu, keep_ref, aside, worst, e8max = np.zeros(8), np.zeros(8), 0, 0.0, 0.0
        for i in range(int(g["n_pairs"])):
            Is, It, theta, kp = V.pair_inputs(dataset["df"], i, dataset["root"], dataset["thetas"])
            np.testing.assert_array_equal(kp, g["kpts%d" % i])
            n = len(kp)
            d = torch.empty(n, dtype=torch.float64, device="cuda")
            fo = torch.empty((n, 4), dtype=torch.float32, device="cuda")
            f8 = V.validate_pair(net, Is, It, theta, kp, acc, pair=i, dist_out=d, flow_out=fo)
            e8 = float(np.max(np.abs(f8.cpu().numpy() - dataset["flows"][i])))
            assert e8 <= e, (engine, i, e8)
            e8max = max(e8max, e8)
            d, fo = d.cpu().numpy(), fo.cpu().numpy().astype(np.float64)
            ws, hs = V.resize_min_resolution_size(Is.shape[1], Is.shape[0])
            wt, ht = V.resize_min_resolution_size(It.shape[1], It.shape[0])
            P, _ = affine_image(dataset["thetas"][i], ht, wt)
            _, _, Lx, Ly, _ = bilinear_zeros(P, unnormalize64(fo[:, 0], wt, False), unnormalize64(fo[:, 1], ht, False))
            do = Lx * (wt / 2.0 * e) + Ly * (ht / 2.0 * e)
            tol = 2 * ((ws - 1) / 2.0 * do[0] + (hs - 1) / 2.0 * do[1]) + 1e-4
            gd = g["dist%d" % i]
            assert np.all(np.abs(d - gd) <= tol), (engine, i, e8, np.max(np.abs(d - gd) - tol))
            worst = max(worst, float(np.max(np.abs(d - gd))))
            near = (np.abs(gd[:, None] - thr) <= tol[:, None]).any(1)
            aside += int(near.sum())
            keep_gpu += (d[~near, None] < thr).sum(0)
            keep_ref += (gd[~near, None] < thr).sum(0)
        print("\n[validation %s] max e8 = %.3g, max |d - golden| = %.3g px, keypoints set aside: %d of %d, prec %s, golden %s"
              % (engine, e8max, worst, aside, sum(len(g["dist%d" % i]) for i in range(int(g["n_pairs"]))),
                 prec.tolist(), g["prec"].tolist()))
        assert aside <= MAX_ASIDE, aside
        np.testing.assert_array_equal(keep_gpu, keep_ref)
        counts, err = V.read_counts(acc.cpu().numpy())
        assert err is None
        np.testing.assert_array_equal(prec, counts[:-1] / counts[-1])
        if aside == 0:
            np.testing.assert_array_equal(prec, g["prec"])
    finally:
        rf.model.set_engine(prev)


def test_dataset_loop_does_not_synchronise(rf, dataset):
    V = rf.validation
    net = _network(rf)
    want = V.validation(dataset["df"], dataset["root"], dataset["thetas"], net, None)      # warm: folded weights, programs
    acc = V.new_counts()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        V.queue_validation(dataset["df"], dataset["root"], dataset["thetas"], net, acc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    counts, err = V.read_counts(acc.cpu().numpy())
    assert err is None
    np.testing.assert_array_equal(counts[:-1] / counts[-1], want)


def test_dataset_errors_as_the_reference(rf, dataset):
    V = rf.validation
    net = _network(rf)
    df = dataset["df"].copy()
    df.loc[1, "XB"] = ";".join(["5000"] + df.loc[1, "XB"].split(";")[1:])          # pair 1: column out of range
    with pytest.raises(IndexError, match="pair 1"):
        V.validation(df, dataset["root"], dataset["thetas"], net, None)
    thetas = list(dataset["thetas"])
    thetas[3] = thetas[3].astype(np.float64)
    with pytest.raises(IndexError, match="pair 1"):                               # pair 1's IndexError comes first
        V.validation(df, dataset["root"], thetas, net, None)
    with pytest.raises(RuntimeError, match="same dtype"):
        V.validation(dataset["df"], dataset["root"], thetas, net, None)
    assert np.isnan(V.validation(dataset["df"].iloc[:0], dataset["root"], [], net, None)).all()


def test_cli_picks_the_best_checkpoint(rf, dataset, tmp_path):
    """The documented entry point, ``python -m ransac_flow_b200.validation``, in a process of its own: one line per checkpoint
    with the eight precisions and valPrec@8 (each equal to ``validation`` on the same networks), then the best checkpoint
    by train.py's strict ``>``."""
    import subprocess
    import sys
    V = rf.validation
    csv, pkl = tmp_path / "corr.csv", tmp_path / "coarse.pkl"
    dataset["df"].to_csv(csv, index=False)
    with open(pkl, "wb") as f:
        pickle.dump(dataset["thetas"], f)
    paths, precs = [], []
    engine = "fp32" if rf.model.get_engine() == rf.ops.ENGINE_FP32 else "f16x3"
    for seed in (1, 7):
        p = tmp_path / ("ckpt_%d.pth" % seed)
        torch.save({"netFeatCoarse": synth.feature_extractor_state(0), "netCorr": {},
                    "netFlowCoarse": synth.net_flow_coarse_state(seed), "netMatch": synth.net_matchability_state(2)}, p)
        paths.append(str(p))
        precs.append(V.validation(dataset["df"], dataset["root"], dataset["thetas"], _network(rf, seed), None))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "ransac_flow_b200.validation", "--valImgDir", dataset["root"], "--valCSV", str(csv),
                        "--inPklCoarse", str(pkl), "--resumePth"] + paths + ["--engine", engine],
                       cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "RuntimeWarning" not in r.stderr, r.stderr
    lines = r.stdout.strip().splitlines()
    assert len(lines) == 3, r.stdout
    for line, p, prec in zip(lines, paths, precs):
        assert line.startswith(p) and line.endswith("valPrec@8 : %.9f" % prec[4]), line
        assert line.split("\t")[1].split()[1:] == ["%.6f" % v for v in prec]
    i = 1 if precs[1][4] > precs[0][4] else (0 if precs[0][4] > 0 else None)
    assert lines[2] == ("best\t%s\tvalPrec@8 : %.9f" % (paths[i], precs[i][4]) if i is not None else "best\tnone")


def test_async_resample_tables_stay_on_their_stream(rf):
    """Tables uploaded without a host synchronisation are cached for the uploading stream only: a blocking caller and
    another stream get their own entries, with the same contents."""
    fn, dev = "rf_lanczos_coeffs_host", torch.device("cuda", torch.cuda.current_device())
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        a = rf.ops.resample_coeffs(997, 531, dev, fn, non_blocking=True)
        assert rf.ops.resample_coeffs(997, 531, dev, fn, non_blocking=True)[0].data_ptr() == a[0].data_ptr()
    b = rf.ops.resample_coeffs(997, 531, dev, fn)
    c = rf.ops.resample_coeffs(997, 531, dev, fn, non_blocking=True)
    assert len({a[0].data_ptr(), b[0].data_ptr(), c[0].data_ptr()}) == 3
    side.synchronize()
    torch.cuda.synchronize()
    for x in (a, c):
        assert torch.equal(x[0], b[0]) and torch.equal(x[1], b[1]) and x[2] == b[2]
