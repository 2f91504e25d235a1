"""Bit-exact restatements of the exact-FMA SIMT kernels (csrc/gemm_simt.cu), helper of the engine-0 tests, not a test module.

Every output element of ``conv_kernel`` is one fp32 FMA chain ``acc = fmaf(a_k, b_k, acc)``: acc starts at +0, k runs over
0 .. K - 1 in (r, s, c) order (the loader's ``tap = k / Cin, r = tap / S, s = tap % S`` and the [R*S*Cin][Cout] weight packing),
then the epilogue adds the bias and the residual in fp32, applies fmaxf(., 0) and, with ``round_out``, cvt.rna.tf32.  Every
score of ``corr_argmax_kernel`` is the same kind of chain over the C channels.  The library is built without fast-math, so
there is no flush to zero and no reassociation: the results are fully determined and are restated here bit for bit, with
fp64 tensor arithmetic that runs on the device (tests/test_fma_ref.py holds this module to exact rational arithmetic).

fl32(a * b + c) of fp32 values a, b, c: the product is exact in fp64 (48 significand bits, exponents far inside fp64's
range), TwoSum gives s = fl64(p + c) and its exact error e, and s is moved to its odd neighbour towards p + c when it is
inexact and even (round to odd).  One rounding of that to fp32 is the correctly rounded fp32 result, because 53 >= 24 + 2
(Boldo and Melquiond, "Emulation of a FMA and correctly-rounded sums: proved algorithms using rounding to odd", 2008).
"""
import numpy as np
import torch

import wgmma_ref as R

_INF = float("inf")


def fma32(a, b, c):
    """fl32(a * b + c), rounded to nearest even, of fp64 tensors holding fp32 values (broadcasting; CPU or CUDA).  Returns an
    fp64 tensor holding the fp32 results."""
    p = a * b                                       # exact
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                   # TwoSum: s + e == p + c exactly
    even = (s.contiguous().view(torch.int64) & 1) == 0
    toward = torch.where(e > 0, torch.full_like(s, _INF), torch.full_like(s, -_INF))
    s = torch.where((e != 0) & even, torch.nextafter(s, toward), s)
    return s.float().double()


def add32(a, b):
    """fl32(a + b) of fp64 tensors holding fp32 values (a * 1 is exact, so this is fma32 with one operand 1)."""
    return fma32(a, torch.ones((), dtype=torch.float64, device=a.device), b)


def conv_rows(x, k, stride, pad):
    """[Ho * Wo, k * k * Cin] fp64 patch rows of a (1, Cin, H, W) image in (r, s, c) order (wgmma_ref.im2col_ref)."""
    return R.im2col_ref(x.double(), k, stride, pad, k * k * x.shape[1])


def packed_weights(w):
    """(Cout, Cin, k, k) -> [k * k * Cin, Cout] in (r, s, c) order, the SIMT kernel's weight layout (fp32, same device)."""
    cout, cin, k, _ = w.shape
    return w.float().permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous()


def chain(col, wk, acc=None):
    """acc = fma32(col[:, k], wk[k], acc) for k = 0 .. K - 1 over [P, Cout], acc starting at +0.  col [P, K] and wk [K, Cout]
    fp64 holding fp32 values."""
    wk = wk.double()
    if acc is None:
        acc = torch.zeros((col.shape[0], wk.shape[1]), dtype=torch.float64, device=col.device)
    for kk in range(col.shape[1]):
        acc = fma32(col[:, kk:kk + 1], wk[kk:kk + 1], acc)
    return acc


def epilogue(acc, bias=None, residual=None, relu=False, round_out=False):
    """conv_kernel's epilogue on fp64-held fp32 accumulators [P, Cout]: + bias, + residual (each an fp32 add), fmaxf(., 0),
    cvt.rna.tf32.  Returns fp32."""
    if bias is not None:
        acc = add32(acc, bias.double().view(1, -1))
    if residual is not None:
        acc = add32(acc, residual.double())
    if relu:
        acc = torch.where(acc > 0, acc, torch.zeros_like(acc))       # fmaxf(v, 0): +0 for every v <= 0
    out = acc.float()
    return R.tf32_rna(out) if round_out else out


def conv_chain(x, w, bias=None, residual=None, stride=1, pad=0, relu=False, round_out=False):
    """The SIMT convolution's output for one image, bit for bit: x (1, Cin, H, W) fp32, w (Cout, Cin, k, k) fp32, bias
    (Cout,) or None, residual [Ho * Wo, Cout] rows or (1, Cout, Ho, Wo) or None; all on one device.  Returns [Ho * Wo, Cout]
    fp32 rows (NHWC), the layout the kernel writes.

    The chain includes the out-of-image taps, which the kernel skips, and stops at K, where the kernel runs on through the
    zero tail of its last 16-wide K slice: both are the same, because fma(0, w, acc) == acc for every acc != -0 and acc is
    never -0 (it starts at +0, and an exact cancellation rounds to +0)."""
    k = w.shape[2]
    acc = chain(conv_rows(x, k, stride, pad), packed_weights(w))
    if residual is not None and residual.dim() == 4:
        residual = residual[0].permute(1, 2, 0).reshape(-1, residual.shape[1])
    return epilogue(acc, bias, residual, relu, round_out)


def conv_chain_images(xs, w, bias=None, residuals=None, stride=1, pad=0, relu=False, round_out=False):
    """conv_chain of every image of a batch in one chain (their patch rows stacked): [sum Ho * Wo, Cout] fp32, the layout of
    the kernel's ragged output."""
    k = w.shape[2]
    col = torch.cat([conv_rows(x, k, stride, pad) for x in xs], 0)
    acc = chain(col, packed_weights(w))
    res = None
    if residuals is not None:
        res = torch.cat([r[0].permute(1, 2, 0).reshape(-1, r.shape[1]) if r.dim() == 4 else r for r in residuals], 0)
    return epilogue(acc, bias, res, relu, round_out)


def scores(A, B, rows=None):
    """fp32 correlation scores A[rows] . B^T as C-step fma32 chains (corr_argmax_kernel), fp64 holding fp32: A [NA, C],
    B [NB, C] fp32."""
    a = (A if rows is None else A[rows]).double()
    return chain(a, B.double().t())


def corr_keys(A, B, block_elems=1 << 23):
    """The correlation's arg-max keys and mutual pairs (rf_corr_mutual_nn at precision 0), bit for bit.  A [NA, C], B [NB, C]
    fp32 on one device.  Scores are computed in row blocks of at most ``block_elems`` elements (about 1 GB of fp64
    temporaries at the default).  Returns numpy (row keys uint64 [NA], column keys uint64 [NB], idx1, idx2): each key is
    wgmma_ref.encode_key(best score, its index), the smallest index on ties; the pairs are the mutual ones whose score v has
    fp32 v * v > 0 (``__fmul_rn(v, v) > 0``), in row order."""
    NA, NB = A.shape[0], B.shape[0]
    if NA == 0 or NB == 0:
        z = np.zeros(0, np.int64)
        return np.zeros(NA, np.uint64), np.zeros(NB, np.uint64), z, z
    dev = A.device
    rbest = torch.empty(NA, dtype=torch.float32, device=dev)
    ridx = torch.empty(NA, dtype=torch.int64, device=dev)
    cbest = torch.full((NB,), -_INF, dtype=torch.float32, device=dev)
    cidx = torch.zeros(NB, dtype=torch.int64, device=dev)
    step = max(1, block_elems // NB)
    for r0 in range(0, NA, step):
        s = scores(A, B, slice(r0, r0 + step)).float()
        ri = s.argmax(1)                                          # the first maximum: the smallest column on ties
        rbest[r0:r0 + step] = s.gather(1, ri[:, None])[:, 0]
        ridx[r0:r0 + step] = ri
        ci = s.argmax(0)                                          # the smallest row of this block on ties
        cv = s.gather(0, ci[None])[0]
        better = cv > cbest                                       # strict: an earlier block keeps its (smaller) row on ties
        cbest = torch.where(better, cv, cbest)
        cidx = torch.where(better, ci + r0, cidx)
    rv, ri, cv, ci = (t.cpu().numpy() for t in (rbest, ridx, cbest, cidx))
    rowk, colk = R.encode_key(rv, ri), R.encode_key(cv, ci)
    mutual = ci[ri] == np.arange(NA)
    keep = mutual & (rv * rv > np.float32(0))                     # fp32 square: underflows to 0 below 2^-75
    i1 = np.nonzero(keep)[0].astype(np.int64)
    return rowk, colk, i1, ri[keep].astype(np.int64)
