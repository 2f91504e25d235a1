"""fp64 reference and truncation band for the warped uint8 target of the training-pair notebook
(train/generate_coarse_aligned_pair.ipynb cell 13: ``ToPILImage(grid_sample(ToTensor(I2), warp_grid(H)))``).

``ToPILImage`` truncates ``255 * v``: wherever 255 v lies farther from an integer than the error of an fp32 evaluation, every
fp32 evaluation (the fused kernel, torch's CPU or CUDA ``grid_sample``) truncates to floor(255 v).  The error bound is
``geometry_ref``'s bilinear sampling bound (gamma_7 |v| + Lx dx + Ly dy) with the coordinate error of an fp32 homography grid,
times 255, plus the rounding of the product by 255."""
import numpy as np

import geometry_ref as G


def grid64(H, h, w):
    """The homography grid of H in fp64 at torch.linspace's fp32 base grid: (h, w) x and y."""
    H = np.asarray(H, dtype=np.float64).reshape(3, 3)
    x = G.lin11(np.arange(w), w).astype(np.float64)[None, :]
    y = G.lin11(np.arange(h), h).astype(np.float64)[:, None]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        pz = H[2, 0] * x + H[2, 1] * y + H[2, 2]
        return (H[0, 0] * x + H[0, 1] * y + H[0, 2]) / pz, (H[1, 0] * x + H[1, 1] * y + H[1, 2]) / pz


def warp_u8_ref(H, src, h, w, grid=None):
    """(255 v (h, w, 3), its fp32 evaluation bound in the same units) for the uint8 (Hin, Win, 3) ``src`` sampled on the grid of
    H (``grid``: a given (gx, gy) instead, e.g. the kernel's exact fp32 grid).  The grid's own fp32 error (four roundings of
    terms up to |H| (|x| + |y| + 1), over |pz|) is covered by a coordinate error of 64 u (|i| + size) pixels."""
    src = np.asarray(src)
    Hin, Win = src.shape[:2]
    P = (src.astype(np.float32) / np.float32(255)).transpose(2, 0, 1)          # ToTensor's fp32 values
    gx, gy = grid if grid is not None else grid64(H, h, w)
    ix, iy = G.unnormalize64(gx, Win, False), G.unnormalize64(gy, Hin, False)
    val, absval, Lx, Ly, outside = G.bilinear_zeros(P, ix, iy)
    with np.errstate(invalid="ignore"):
        dx = 8 * G.U * (np.abs(np.where(outside, 0, ix)) + Win)
        dy = 8 * G.U * (np.abs(np.where(outside, 0, iy)) + Hin)
        allow = G.gamma(7) * absval + Lx * dx + Ly * dy
    allow = np.where(outside[None], 0.0, allow)
    v255 = 255.0 * val.transpose(1, 2, 0)
    return v255, 255.0 * allow.transpose(1, 2, 0) + 2 * 255.0 * G.U * v255


def decided(v255, band):
    """Where every evaluation within ``band`` of 255 v truncates to the same byte."""
    return np.floor(v255 - band) == np.floor(v255 + band)
