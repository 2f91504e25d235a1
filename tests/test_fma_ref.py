"""The fp32 FMA-chain restatements of tests/fma_ref.py against exact rational arithmetic, and proof that the bit comparison of
tests/test_gpu_simt_exact.py rejects subtly wrong kernels (CPU only)."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import fma_ref as FR
import wgmma_ref as R
from test_gpu_simt_exact import CASES, case_id, case_inputs, ohw_of, tie_inputs


# ------------------------------------------------------------------ exact fp32 rounding of a rational
def fl32(q, negative_zero=False):
    """The fp32 value nearest to the Fraction q (ties to even), with subnormals and overflow to infinity, as np.float32.  A
    zero q gives -0 when ``negative_zero``; a nonzero q that rounds to zero keeps its sign."""
    if q == 0:
        return np.float32(-0.0 if negative_zero else 0.0)
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if q < Fraction(2) ** e:
        e -= 1                                                  # 2^e <= q < 2^(e + 1)
    quantum = Fraction(2) ** (max(e, -126) - 23)
    n = q / quantum
    m = n.numerator // n.denominator
    rem = n - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m % 2 == 1):
        m += 1
    v = m * quantum
    if v >= Fraction(2) ** 128:
        return np.float32(sign * np.inf)
    return np.float32(sign * float(v)) if m else np.float32(-0.0 if sign < 0 else 0.0)


def fma_exact(a, b, c):
    """fl32(a * b + c) of np.float32 values by rational arithmetic, with IEEE's zero signs (an exact zero sum is +0 unless
    both the product and c are -0)."""
    q = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    neg_zero = (a == 0 or b == 0) and c == 0 and (np.signbit(a) != np.signbit(b)) and np.signbit(c)
    return fl32(q, neg_zero)


def fma_exact_chain(a, b):
    """fl32 FMA chain over the pairs of a and b, acc starting at +0, by rational arithmetic."""
    acc = np.float32(0)
    for x, y in zip(a, b):
        acc = fma_exact(x, y, acc)
    return float(acc)


def f32(v):
    return np.asarray(v, dtype=np.float64).astype(np.float32)


def triples(rs):
    """>= 20 000 fp32 (a, b, c) triples: random with exponent gaps between a * b and c up to +-120, exact cancellations, exact
    fp32 midpoints in both tie directions (and a tiny c beside a midpoint product, where rounding fp64 then fp32 would fail),
    subnormal results and signed zeros."""
    out = []
    n = 6000
    a = f32(rs.randn(n) * 2.0 ** rs.randint(-20, 21, n))
    b = f32(rs.randn(n) * 2.0 ** rs.randint(-20, 21, n))
    gap = rs.randint(-120, 121, n)
    gap[:4] = [120, -120, 119, -119]
    eab = np.frexp(a.astype(np.float64) * b.astype(np.float64))[1]
    c = f32(rs.randn(n) * 2.0 ** np.clip(eab + gap, -140, 120))
    out.append((a, b, c))
    # exact cancellations: a * b exact in fp32 (12-bit significands), c = -a * b  -> +0
    n = 2000
    a = f32(rs.randint(1, 4096, n) * 2.0 ** rs.randint(-30, 30, n) * rs.choice([-1, 1], n))
    b = f32(rs.randint(1, 4096, n) * 2.0 ** rs.randint(-30, 30, n) * rs.choice([-1, 1], n))
    out.append((a, b, f32(-(a.astype(np.float64) * b.astype(np.float64)))))
    # near cancellations: c = -fl32(a * b), the result is the product's rounding error
    a, b = f32(rs.randn(n)), f32(rs.randn(n) * 2.0 ** rs.randint(-10, 10, n))
    out.append((a, b, -(a * b)))
    # exact midpoints: c = fp32 m (either parity), a * b = (2j + 1) * ulp(m) / 2
    n = 4000
    m = f32(rs.uniform(1, 2, n) * 2.0 ** rs.randint(-100, 100, n) * rs.choice([-1, 1], n))
    ulp = np.spacing(np.abs(m)).astype(np.float64)
    a = f32(2 * rs.randint(0, 200, n) + 1)
    b = f32(ulp / 2 * rs.choice([-1, 1], n))
    out.append((a, b, m))
    # products that are midpoints themselves (odd 25-bit integers times 2^k), c = 0 or a tiny nudge either way
    p1, p2 = 2 * rs.randint(2 ** 11, 2 ** 12, n) + 1, 2 * rs.randint(2 ** 11, 2 ** 12, n) + 1
    sc = rs.randint(-60, 60, n)
    a, b = f32(p1 * 2.0 ** sc), f32(p2 * 2.0 ** -sc)
    tiny = f32(rs.choice([0.0, 1.0, -1.0], n) * 2.0 ** rs.randint(-100, -60, n))
    out.append((a * f32(rs.choice([-1, 1], n)), b, tiny))
    # subnormal results, and half the smallest subnormal (a tie that rounds to a signed zero)
    n = 2000
    a = f32(rs.randn(n) * 2.0 ** rs.randint(-78, -65, n))
    b = f32(rs.randn(n) * 2.0 ** rs.randint(-78, -65, n))
    c = f32(rs.choice([0.0, 1.0], n) * rs.randint(-2 ** 22, 2 ** 22, n) * 2.0 ** -149)
    out.append((a, b, c))
    a = f32(rs.choice([-1, 1], 200) * 2.0 ** -75)
    out.append((a, f32(np.full(200, 2.0 ** -75)), f32(rs.choice([0.0, -0.0], 200))))
    # subnormal results from normal operands: c = -+2^-126 (1 + small), a * b near it
    a, b = f32(rs.uniform(1, 2, n) * 2.0 ** -63), f32(rs.uniform(1, 2, n) * 2.0 ** -63)
    out.append((a, b, f32(-(a.astype(np.float64) * b.astype(np.float64)) * (1 + rs.randint(-8, 9, n) * 2.0 ** -22))))
    # signed zeros
    z = f32(rs.choice([0.0, -0.0], 400))
    out.append((z, f32(rs.randn(400)), f32(rs.choice([0.0, -0.0], 400))))
    return [np.concatenate(t) for t in zip(*out)]


def test_fma32_matches_rational_arithmetic():
    a, b, c = triples(np.random.RandomState(0))
    assert len(a) >= 20000
    got = FR.fma32(torch.from_numpy(a).double(), torch.from_numpy(b).double(), torch.from_numpy(c).double()).float().numpy()
    exp = np.array([fma_exact(x, y, z) for x, y, z in zip(a, b, c)], dtype=np.float32)
    bad = got.view(np.uint32) != exp.view(np.uint32)
    assert not bad.any(), [(a[i], b[i], c[i], got[i], exp[i]) for i in np.nonzero(bad)[0][:5]]
    # the kinds of result the triples were built to reach
    s = np.abs(exp)
    assert np.sum((s > 0) & (s < 2.0 ** -126)) > 500                     # subnormal
    assert np.sum(exp.view(np.uint32) == 0x80000000) > 50                 # -0
    assert np.sum(exp.view(np.uint32) == 0) > 2000                        # +0, most of them exact cancellations
    # ties in both directions: results of the midpoint block that rounded down and up from m
    fl_sum = a[10000:14000].astype(np.float64) * b[10000:14000] + c[10000:14000]
    d = exp[10000:14000].astype(np.float64) - fl_sum
    assert np.sum(d > 0) > 1000 and np.sum(d < 0) > 1000
    # the double-rounding trap: plain fp64 then fp32 rounding gets some of these wrong
    naive = (torch.from_numpy(a).double() * torch.from_numpy(b).double() + torch.from_numpy(c).double()).float().numpy()
    assert np.sum(naive.view(np.uint32) != exp.view(np.uint32)) > 100


# ------------------------------------------------------------------ conv_chain against a literal loop of exact FMAs
def conv_literal(x, w, bias, res, stride, pad, relu, round_out):
    """Per output element: acc = +0, then fma_exact over the in-image taps in (r, s, c) order, + bias, + residual (each
    rounded to fp32), max(., 0), cvt.rna.tf32.  x (1, Cin, H, W), w (Cout, Cin, k, k), res (1, Cout, Ho, Wo) fp32."""
    x, w = x.numpy(), w.numpy()
    _, cin, h, wd = x.shape
    cout, _, k, _ = w.shape
    ho, wo = R.out_hw(h, wd, k, stride, pad)
    out = np.zeros((ho * wo, cout), np.float32)
    for oy in range(ho):
        for ox in range(wo):
            for o in range(cout):
                acc = np.float32(0.0)
                for r in range(k):
                    for s in range(k):
                        iy, ix = oy * stride - pad + r, ox * stride - pad + s
                        if 0 <= iy < h and 0 <= ix < wd:
                            for ci in range(cin):
                                acc = fma_exact(x[0, ci, iy, ix], w[o, ci, r, s], acc)
                if bias is not None:
                    acc = fma_exact(np.float32(1), acc, bias[o].numpy())
                if res is not None:
                    acc = fma_exact(np.float32(1), acc, res[0, o, oy, ox].numpy())
                if relu:
                    acc = max(acc, np.float32(0))
                if round_out:
                    acc = np.array([(np.array([acc], np.float32).view(np.int32)[0] + 0x1000) & ~0x1FFF], np.int32).view(np.float32)[0]
                out[oy * wo + ox, o] = acc
    return out


def test_conv_chain_equals_literal_exact_loop():
    g = torch.Generator().manual_seed(3)
    sizes, cout = [(5, 4), (3, 6)], 5
    xs = [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, 3, 3, 3, generator=g)
    bias = torch.randn(cout, generator=g)
    rs = [torch.randn(1, cout, ho, wo, generator=g) for ho, wo in ohw_of(sizes, 3, 2, 1)]
    got = FR.conv_chain_images(xs, w, bias, rs, 2, 1, True, True)
    exp = np.concatenate([conv_literal(x, w, bias, r, 2, 1, True, True) for x, r in zip(xs, rs)])
    assert np.array_equal(got.numpy().view(np.uint32), exp.view(np.uint32))
    assert (exp == 0).any() and (exp > 0).any()
    one = FR.conv_chain(xs[1], w, bias, rs[1], 2, 1, True, True)
    assert torch.equal(one, got[6:])


@pytest.mark.parametrize("cin,cout,k,stride,pad,sizes", [(3, 8, 3, 2, 1, [(9, 7)]), (40, 6, 5, 1, 2, [(6, 5), (1, 1)]),
                                                         (256, 4, 1, 1, 0, [(7, 3)])])
def test_conv_chain_is_a_convolution(cin, cout, k, stride, pad, sizes):
    """Within gamma_{K+2} absref of the fp64 convolution + bias + residual (+ ReLU)."""
    g = torch.Generator().manual_seed(cin)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, k, k, generator=g)
    bias = torch.randn(cout, generator=g)
    rs = [torch.randn(1, cout, ho, wo, generator=g) for ho, wo in ohw_of(sizes, k, stride, pad)]
    got = FR.conv_chain_images(xs, w, bias, rs, stride, pad, True)
    refs = [R.conv_ref(x, w, bias, r, stride, pad, True) for x, r in zip(xs, rs)]
    ref = torch.cat([a[0].permute(1, 2, 0).reshape(-1, cout) for a, _ in refs])
    absref = torch.cat([b[0].permute(1, 2, 0).reshape(-1, cout) for _, b in refs])
    err = (got.double() - ref).abs()
    assert bool((err <= R.gamma(k * k * cin + 2) * absref).all())
    assert float(err.max()) > 0                                     # fp32 rounding happened


# ------------------------------------------------------------------ mutations: wrong kernels the bit comparison rejects
def mut_unfused(x, w, b, r, stride, pad, relu):
    k = w.shape[2]
    col, wk = FR.conv_rows(x, k, stride, pad).float(), FR.packed_weights(w)
    acc = torch.zeros(col.shape[0], wk.shape[1])
    for kk in range(col.shape[1]):
        acc = acc + col[:, kk:kk + 1] * wk[kk:kk + 1]             # two fp32 roundings
    return FR.epilogue(acc.double(), b, r, relu)


def mut_channel_major(x, w, b, r, stride, pad, relu):
    k, cin = w.shape[2], w.shape[1]
    col = FR.conv_rows(x, k, stride, pad)
    perm = torch.arange(k * k * cin).view(k * k, cin).t().reshape(-1)          # (c, r, s) order
    return FR.epilogue(FR.chain(col[:, perm], FR.packed_weights(w)[perm]), b, r, relu)


def mut_bias_first(x, w, b, r, stride, pad, relu):
    col, wk = FR.conv_rows(x, w.shape[2], stride, pad), FR.packed_weights(w)
    acc0 = b.double().view(1, -1).expand(col.shape[0], -1).clone() if b is not None else None
    return FR.epilogue(FR.chain(col, wk, acc0), None, r, relu)


def mut_residual_after_relu(x, w, b, r, stride, pad, relu):
    acc = FR.chain(FR.conv_rows(x, w.shape[2], stride, pad), FR.packed_weights(w))
    out = FR.epilogue(acc, b, None, relu).double()
    return FR.add32(out, r.double()).float() if r is not None else out.float()


def mut_drop_last_slice(x, w, b, r, stride, pad, relu):
    col, wk = FR.conv_rows(x, w.shape[2], stride, pad), FR.packed_weights(w)
    K = col.shape[1] // 16 * 16
    if K == 0:
        return FR.epilogue(torch.zeros(col.shape[0], wk.shape[1], dtype=torch.float64), b, r, relu)
    return FR.epilogue(FR.chain(col[:, :K], wk[:K]), b, r, relu)


def mut_border(x, w, b, r, stride, pad, relu):
    """ix < W - 1 instead of ix < W: the image's last column is read as outside."""
    x = x.clone()
    x[..., -1] = 0
    return FR.conv_chain(x, w, b, r, stride, pad, relu)


MUTANTS = {"unfused": mut_unfused, "channel_major": mut_channel_major, "bias_first": mut_bias_first,
           "residual_after_relu": mut_residual_after_relu, "drop_last_slice": mut_drop_last_slice, "border": mut_border}


def cheap_cases(budget=400_000):
    """The GPU test's cases whose chains are cheap on the CPU (output elements x K below ``budget``)."""
    out = []
    for c in CASES:
        cin, cout, k, stride, pad, sizes = c[:6]
        P = sum(h * w for h, w in ohw_of(sizes, k, stride, pad))
        if P * cout * k * k * cin <= budget:
            out.append(c)
    return out


@pytest.fixture(scope="module")
def cheap():
    """(case, inputs, conv_chain rows) of the cheap cases."""
    out = []
    for c in cheap_cases():
        xs, w, b, rs = case_inputs(c)
        ref = FR.conv_chain_images(xs, w, b, rs, c[3], c[4], c[8])
        out.append((c, (xs, w, b, rs), ref))
    return out


def test_cheap_cases_span_the_instances():
    from test_gpu_simt_exact import instance
    cs = cheap_cases()
    assert len(cs) >= 12
    assert {instance(c[0], c[1]) for c in cs} == {(4, False), (4, True), (8, False), (8, True)}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_bit_comparison_rejects_mutant(cheap, mutant):
    """The mutant differs from the FMA chain in at least one output bit on at least one of the GPU test's cases: the GPU test
    would fail on a kernel that computed it."""
    f = MUTANTS[mutant]
    caught = []
    for c, (xs, w, b, rs), ref in cheap:
        stride, pad, relu = c[3], c[4], c[8]
        rows = [rr[0].permute(1, 2, 0).reshape(-1, rr.shape[1]) for rr in rs] if rs is not None else [None] * len(xs)
        got = torch.cat([f(x, w, b, r, stride, pad, relu) for x, r in zip(xs, rows)])
        if not torch.equal(got.view(torch.int32), ref.view(torch.int32)):
            caught.append(case_id(c))
    print("%s: caught by %d of %d cases" % (mutant, len(caught), len(cheap)))
    assert caught


def test_bit_comparison_rejects_tf32_ties_to_even():
    """On the constructed ties of the engine-1 fallback test, nearest-even TF32 rounding differs from cvt.rna."""
    xs, w, b, rs = tie_inputs()
    plain = FR.conv_chain_images(xs, w, b, rs, 1, 0, True)
    rna = FR.conv_chain_images(xs, w, b, rs, 1, 0, True, round_out=True)
    ties = (plain.view(torch.int32) & 0x1FFF) == 0x1000
    assert int(ties.sum()) > 100
    assert not torch.equal(R.tf32_round(plain).view(torch.int32), rna.view(torch.int32))
    assert bool((R.tf32_round(plain)[ties] < rna[ties]).any())


# ------------------------------------------------------------------ corr_keys on hand-made cases
def test_corr_keys_tie_breaks():
    """Equal scores: the smallest index wins, on rows and columns, inside one row block and across blocks."""
    A = torch.tensor([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [1.0, 0, 0, 0], [0, 0, 1.0, 0]])
    B = torch.tensor([[0, 1.0, 0, 0], [1.0, 0, 0, 0], [1.0, 0, 0, 0], [0, 0, 0, 1.0]])
    for block in (1 << 20, 4, 8):                                  # one block, one row per block, two rows per block
        rowk, colk, i1, i2 = FR.corr_keys(A, B, block_elems=block)
        rs, ri = R.decode_key(rowk)
        cs, ci = R.decode_key(colk)
        assert ri.tolist() == [1, 0, 1, 0] and rs.tolist() == [1, 1, 1, 0]    # row 3 scores 0 everywhere: column 0
        assert ci.tolist() == [1, 0, 0, 0] and cs.tolist() == [1, 1, 1, 0]
        assert i1.tolist() == [0, 1] and i2.tolist() == [1, 0]
        assert np.array_equal(rowk, R.encode_key(rs, ri))


def test_corr_keys_square_underflow():
    """A mutual pair is kept only if the fp32 square of its score is > 0: 2^-80 (square 0) is dropped, 2^-70 (square
    2^-140, subnormal) and 2^-60 are kept; negative maxima are kept too."""
    from test_gpu_simt_exact import underflow_features
    A, B = underflow_features()
    _, _, i1, i2 = FR.corr_keys(A, B)
    assert i1.tolist() == [1, 2] and i2.tolist() == [2, 3]
    A = torch.tensor([[-1.0, 0, 0, 0], [0, -2.0, 0, 0]])
    B = torch.tensor([[1.0, 0, 0, 0], [0, 1.0, 0, 0]])
    rowk, colk, i1, i2 = FR.corr_keys(A, B)
    rs, ri = R.decode_key(rowk)
    assert ri.tolist() == [1, 0] and rs.tolist() == [0, 0]        # -1 / -2 lose to the 0 of the other column
    A = torch.tensor([[-1.0, 0, 0, 0]])
    _, _, i1, i2 = FR.corr_keys(A, B[:1])
    assert i1.tolist() == [0] and i2.tolist() == [0]              # score -1: (-1)^2 > 0


def test_corr_keys_scores_are_fma_chains():
    """Scores are fp32 FMA chains over C in channel order, not fp32 dot products of another order."""
    rs = np.random.RandomState(1)
    A = torch.from_numpy(rs.randn(40, 36).astype(np.float32))
    B = torch.from_numpy(rs.randn(30, 36).astype(np.float32))
    s = FR.scores(A, B).float()
    row = [fma_exact_chain(A[i].numpy(), B[j].numpy()) for i, j in ((0, 0), (5, 7), (39, 29))]
    assert [s[0, 0].item(), s[5, 7].item(), s[39, 29].item()] == row
    rowk, colk, _, _ = FR.corr_keys(A, B)
    sc, idx = R.decode_key(rowk)
    assert np.array_equal(idx, s.argmax(1).numpy()) and np.array_equal(sc, s.max(1).values.numpy())


def test_fl32_rounding_helper():
    assert fl32(Fraction(1) + Fraction(1, 2 ** 24)) == np.float32(1.0)                  # tie to even (down)
    assert fl32(Fraction(1) + Fraction(3, 2 ** 24)) == np.float32(1 + 2.0 ** -22)        # tie to even (up)
    assert fl32(Fraction(1, 2 ** 150)) == 0 and not np.signbit(fl32(Fraction(1, 2 ** 150)))
    assert np.signbit(fl32(-Fraction(1, 2 ** 150)))
    assert fl32(Fraction(3, 2 ** 151)) == np.float32(2.0 ** -149)
    assert fl32(Fraction(2) ** 128) == np.inf
