"""Engine 0, the exact-FMA SIMT engine (csrc/gemm_simt.cu), bit for bit against the fp32 restatements of its FMA chains in
tests/fma_ref.py: the convolution (all four conv_kernel instances, TN 4 / 8 x VEC or not), engine 1's fallback to it (with
the cvt.rna.tf32 rounding of ReLU'd outputs), the layer runner on engine 0, and the correlation's arg-max keys and mutual
pairs at precision 0.  Outputs are NaN-filled with a guard region after them; an element passes only if its int32 bits
equal the restatement's (so -0 against +0 fails too).  Plus the invariants that need no reference, the alignment and
residual-shape checks, and a CPU test that the case list covers the shapes it claims to."""
import numpy as np
import pytest
import torch

import fma_ref as FR
import wgmma_ref as R
from conftest import golden
from test_gpu_wgmma_edges import corr_call, corr_data

GUARD = 4096

# ------------------------------------------------------------------ cases
# (cin, cout, k, stride, pad, sizes, bias, res, relu)
RAG = [(5, 7), (9, 13), (1, 1), (11, 4)]                      # 197 pixels at 3x3 / stride 1 / pad 1: tiles straddle images
# sixteen images (RF_MAX_IMGS); at 3x3 / stride 1 / pad 1 the first 128-pixel tile spans 11 of them, at stride 2 all 16
SIXTEEN = [(2, 3), (1, 5), (4, 4), (3, 3), (1, 1), (2, 2), (5, 1), (3, 4), (2, 5), (6, 7), (9, 9), (1, 1), (4, 6), (13, 11), (2, 2),
           (7, 3)]
# the shapes torch-CPU checked within 2e-5 * max|ref| before, each with (relu, res) = (on, off), (on, on), (off, off)
LEGACY = [(3, 64, 3, 1, 1, [(20, 28)]), (3, 64, 7, 2, 3, [(32, 48), (18, 22)]), (64, 64, 3, 1, 1, [(24, 32), (9, 7)]),
          (64, 128, 3, 2, 1, [(24, 32)]), (64, 256, 1, 1, 0, [(13, 17), (6, 5), (1, 1)]), (256, 512, 1, 2, 0, [(14, 18)]),
          (128, 128, 3, 1, 1, [(16, 16), (16, 16)]), (49, 512, 3, 1, 1, [(6, 8)]), (128, 49, 3, 1, 1, [(6, 8)]),
          (128, 1, 3, 1, 1, [(6, 8), (6, 8)]), (1024, 256, 1, 1, 0, [(15, 20), (30, 40)]), (16, 20, 3, 1, 1, [(5, 5)])]
CASES = [c[:5] + (c[5], True, res, relu) for c in LEGACY for relu, res in ((True, False), (True, True), (False, False))] + [
    (1, 2, 1, 1, 0, [(1, 1), (1, 37), (29, 1)], True, True, True),         # K = 1; 1 x 1, 1 x W, H x 1 images
    (1, 65, 3, 1, 1, [(1, 1), (1, 9), (7, 1)], True, False, True),
    (3, 63, 3, 2, 1, RAG, False, True, False),                             # Cout % 4 != 0 with a residual, no bias
    (15, 127, 3, 1, 1, RAG, True, True, False),                            # Cout % 4 != 0 with bias and residual
    (16, 129, 3, 1, 0, [(5, 7), (9, 13), (3, 3), (11, 4)], True, True, True),
    (17, 200, 5, 1, 2, [(2, 3), (6, 9), (1, 1)], True, False, True),       # images smaller than the kernel
    (32, 49, 7, 2, 3, [(3, 2), (13, 11), (1, 1)], True, True, True),
    (49, 64, 3, 1, 2, [(4, 5), (1, 1)], True, True, False),
    (64, 65, 1, 2, 0, [(37, 53), (1, 1), (5, 131)], True, True, True),
    (256, 64, 3, 1, 1, [(60, 80)], True, True, True),
    (1024, 128, 3, 1, 1, [(3, 4), (1, 1)], True, False, True),             # K = 9216
    (1024, 2, 1, 1, 0, [(7, 19)], False, False, False),                    # 133 pixels, bare chain
    (16, 128, 1, 1, 0, [(127, 1)], False, True, True),                     # 127 pixels
    (15, 64, 1, 1, 0, [(8, 16)], True, False, False),                      # 128 pixels
    (64, 63, 3, 1, 1, [(3, 43)], True, True, True),                        # 129 pixels
    (3, 512, 3, 1, 1, SIXTEEN, True, True, True),
    (32, 1, 3, 2, 1, SIXTEEN, True, False, True),
    (17, 2, 1, 1, 1, [(4, 6), (1, 1)], True, True, True),                  # pad > k - 1: the border outputs have no tap
    (15, 129, 3, 1, 3, [(2, 2), (5, 3)], True, False, False),              # (bias / residual only)
    (64, 200, 5, 1, 2, [(9, 7), (1, 2)], False, True, True),
    (49, 127, 3, 1, 1, [(6, 8), (15, 20)], False, False, True),
    (256, 65, 1, 1, 0, RAG, True, True, True),
    (32, 64, 3, 2, 1, [(128, 3), (3, 128)], True, True, False),
    (1, 1, 7, 2, 3, [(9, 9), (2, 1)], True, True, True),
    (3, 128, 1, 2, 0, [(1, 1), (6, 5)], False, True, True),
]


def case_id(c):
    cin, cout, k, stride, pad, sizes, bias, res, relu = c
    return "%d-%d-k%ds%dp%d-%s-%s%s%s" % (cin, cout, k, stride, pad, "_".join("%dx%d" % s for s in sizes[:3]) + ("_x%d" % len(sizes) if len(sizes) > 3 else ""),
                                        "b" if bias else "", "r" if res else "", "R" if relu else "")


def instance(cin, cout):
    """(TN, VEC) of the conv_kernel instance rf_conv2d_nhwc launches."""
    return (8 if cout >= 128 else 4), cin % 16 == 0


def ohw_of(sizes, k, stride, pad):
    return [R.out_hw(h, w, k, stride, pad) for h, w in sizes]


def images_per_tile(ohw):
    """The largest number of images whose output pixels share one 128-pixel tile."""
    ends = np.cumsum([0] + [h * w for h, w in ohw])
    tiles = (ends[-1] + 127) // 128
    return max(sum(1 for i in range(len(ohw)) if ends[i] < 128 * (t + 1) and ends[i + 1] > 128 * t) for t in range(tiles))


def tapless_outputs(h, w, k, stride, pad):
    """Number of output pixels of an h x w image none of whose taps is inside the image."""
    ho, wo = R.out_hw(h, w, k, stride, pad)
    rows = sum(1 for oy in range(ho) if all(not (0 <= oy * stride - pad + r < h) for r in range(k)))
    cols = sum(1 for ox in range(wo) if all(not (0 <= ox * stride - pad + s < w) for s in range(k)))
    return ho * wo - (ho - rows) * (wo - cols)


def inputs(seed, cin, cout, k, stride, pad, sizes, bias, res):
    """Seeded fp32 CPU inputs: images (1, Cin, H, W), weights / sqrt(fan-in), bias or None, residuals (1, Cout, Ho, Wo) or None."""
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, k, k, generator=g) / float(np.sqrt(cin * k * k))
    b = torch.randn(cout, generator=g) if bias else None
    rs = [torch.randn(1, cout, ho, wo, generator=g) for ho, wo in ohw_of(sizes, k, stride, pad)] if res else None
    return xs, w, b, rs


def case_inputs(c):
    cin, cout, k, stride, pad, sizes, bias, res, _ = c
    return inputs(CASES.index(c) + 1000 * k + cin, cin, cout, k, stride, pad, sizes, bias, res)


def tie_inputs():
    """A 1 x 1 convolution (Cin 3, not a tensor-core shape) whose even output channels are exact TF32 midpoints: channel 0
    of x is a power of two, the weights of channels 1 and 2 are 0, and w[o, 0] = 1 + (2 m + 1) 2^-11 (12 significant bits,
    the last one set).  cvt.rna rounds them away from zero, round-to-nearest-even down for even m."""
    g = torch.Generator().manual_seed(7)
    sizes = [(4, 5), (3, 3)]
    xs = [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]
    for x in xs:
        x[0, 0] = torch.pow(2.0, torch.randint(-3, 4, (x.shape[2], x.shape[3]), generator=g).float())
    w = torch.randn(72, 3, 1, 1, generator=g)
    m = torch.randint(0, 1024, (36,), generator=g).float()
    w[0::2, 0, 0, 0] = 1 + (2 * m + 1) * 2.0 ** -11
    w[0::2, 1:] = 0
    return xs, w, None, None


# ------------------------------------------------------------------ running the library and the restatement
def nhwc_cuda(ts):
    return R.nhwc(ts).cuda()


def run(rf, xs, w, bias, rs, k, stride, pad, relu, engine=0, w_tc=None):
    """rf_conv2d_nhwc on a NaN-filled output with GUARD floats after it.  Returns (output [P, Cout] fp32, guard view)."""
    cout, cin = w.shape[0], xs[0].shape[1]
    hw = [(x.shape[2], x.shape[3]) for x in xs]
    P = sum(h * ww for h, ww in ohw_of(hw, k, stride, pad))
    flat = torch.full((P * cout + GUARD,), 1234.0, dtype=torch.float32, device="cuda")
    flat[:P * cout] = float("nan")
    y = flat[:P * cout].view(P, cout)
    R.conv_call(rf, nhwc_cuda(xs), hw, cin, FR.packed_weights(w).cuda(), w_tc, bias.cuda() if bias is not None else None,
                nhwc_cuda(rs) if rs is not None else None, cout, k, stride, pad, relu, engine, y)
    torch.cuda.synchronize()
    return y, flat[P * cout:]


def reference(xs, w, bias, rs, stride, pad, relu, round_out=False):
    return FR.conv_chain_images([x.cuda() for x in xs], w.cuda(), bias.cuda() if bias is not None else None,
                                [r.cuda() for r in rs] if rs is not None else None, stride, pad, relu, round_out)


def bits(t):
    return t.contiguous().view(torch.int32)


def assert_bits(got, ref, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = bits(got) != bits(ref)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements differ in bits from the FMA chain; first at %s: got %r (0x%08x) chain %r (0x%08x)"
                             % (what, int(bad.sum()), bad.numel(), i, got[i].item(), bits(got)[i].item() & 0xFFFFFFFF, ref[i].item(),
                                bits(ref)[i].item() & 0xFFFFFFFF))


def assert_guard(guard):
    assert bool((guard == 1234.0).all()), "the convolution wrote past its output"


# ------------------------------------------------------------------ the case list covers what it claims (CPU)
def test_case_list_coverage():
    cins, couts = {c[0] for c in CASES}, {c[1] for c in CASES}
    assert {1, 3, 15, 16, 17, 32, 49, 64, 256, 1024} <= cins
    assert {1, 2, 49, 63, 64, 65, 127, 128, 129, 200, 512} <= couts
    assert {c[2:5] for c in CASES} >= {(1, 1, 0), (1, 2, 0), (3, 1, 1), (3, 2, 1), (3, 1, 0), (5, 1, 2), (7, 2, 3), (3, 1, 2)}
    assert {instance(c[0], c[1]) for c in CASES} == {(4, False), (4, True), (8, False), (8, True)}
    Ks = [c[2] * c[2] * c[0] for c in CASES]
    assert min(Ks) == 1 and max(Ks) == 9216 and any(K % 16 == 0 for K in Ks) and any(K % 16 for K in Ks)
    for j in (6, 7, 8):                                            # bias, residual, ReLU: each on and off
        assert {c[j] for c in CASES} == {True, False}
    assert any(c[1] % 4 and c[6] and c[7] for c in CASES)           # scalar B loads and the scalar epilogue, bias + residual
    sizes = [s for c in CASES for s in c[5]]
    assert (1, 1) in sizes and any(h == 1 and w > 1 for h, w in sizes) and any(w == 1 and h > 1 for h, w in sizes)
    assert any(min(h, w) < c[2] for c in CASES for h, w in c[5])    # images smaller than the kernel
    totals = {sum(h * w for h, w in ohw_of(c[5], *c[2:5])) for c in CASES}
    assert {127, 128, 129} <= totals
    per_tile = [images_per_tile(ohw_of(c[5], *c[2:5])) for c in CASES]
    assert any(len(c[5]) == 16 and n >= 8 for c, n in zip(CASES, per_tile))
    assert sum(1 for n in per_tile if n >= 2) >= 10                  # ragged batches whose tiles straddle images
    assert any(c[0] == 256 and (60, 80) in c[5] for c in CASES)
    assert any(tapless_outputs(h, w, *c[2:5]) for c in CASES for h, w in c[5])     # outputs that are bias / residual only
    assert len({case_id(c) for c in CASES}) == len(CASES)


# ------------------------------------------------------------------ engine 0 against the FMA chains
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_engine0_bits(rf, case):
    cin, cout, k, stride, pad, sizes, bias, res, relu = case
    xs, w, b, rs = case_inputs(case)
    y, guard = run(rf, xs, w, b, rs, k, stride, pad, relu)
    assert_bits(y, reference(xs, w, b, rs, stride, pad, relu), case_id(case))
    assert_guard(guard)


@pytest.mark.gpu
def test_cout127_equals_first_channels_of_cout128(rf):
    """Cout 127 (TN 4, scalar weight loads and epilogue) == the first 127 channels of Cout 128 (TN 8, float4 paths)."""
    xs, w, b, rs = inputs(1, 64, 128, 3, 1, 1, RAG, True, True)
    y128, _ = run(rf, xs, w, b, rs, 3, 1, 1, True)
    y127, g = run(rf, xs, w[:127].contiguous(), b[:127].contiguous(), [r[:, :127].contiguous() for r in rs], 3, 1, 1, True)
    assert instance(64, 127) == (4, True) and instance(64, 128) == (8, True)
    assert torch.equal(bits(y127), bits(y128[:, :127].contiguous()))
    assert_guard(g)


@pytest.mark.gpu
def test_cin15_equals_cin16_with_zero_channel(rf):
    """Cin 15 (the scalar A loader, K slices straddling taps) == Cin 16 with a zero 16th channel and zero weights (the float4
    loader)."""
    xs, w, b, rs = inputs(2, 15, 72, 3, 1, 1, RAG, True, True)
    xs16 = [torch.cat([x, torch.zeros_like(x[:, :1])], 1) for x in xs]
    w16 = torch.cat([w, torch.zeros_like(w[:, :1])], 1)
    y15, _ = run(rf, xs, w, b, rs, 3, 1, 1, True)
    y16, _ = run(rf, xs16, w16, b, rs, 3, 1, 1, True)
    assert instance(15, 72) == (4, False) and instance(16, 72) == (4, True)
    assert torch.equal(bits(y15), bits(y16))


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [72, 136])
def test_sixteen_image_batch_equals_images_alone(rf, cout):
    """Each image of a sixteen-image batch equals that image run alone, two calls give identical bits, and a seventeenth
    image is refused."""
    xs, w, b, rs = inputs(3, 32, cout, 3, 1, 1, SIXTEEN, True, True)
    y, _ = run(rf, xs, w, b, rs, 3, 1, 1, True)
    y2, _ = run(rf, xs, w, b, rs, 3, 1, 1, True)
    assert not bool(torch.isnan(y).any())
    assert torch.equal(bits(y), bits(y2))
    o = np.cumsum([0] + [h * ww for h, ww in SIXTEEN])
    for i in range(16):
        alone, _ = run(rf, xs[i:i + 1], w, b, rs[i:i + 1], 3, 1, 1, True)
        assert torch.equal(bits(y[o[i]:o[i + 1]]), bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        run(rf, xs + xs[:1], w, b, rs + rs[:1], 3, 1, 1, True)


# ------------------------------------------------------------------ engine 1's fallback to conv_kernel (round_out after ReLU)
# (cin, cout, k, stride, pad, sizes, bias, res, pass w_tc): shapes the TF32 wgmma kernel does not take, and a supported one
# passed without tensor-core weights; "tie" is tie_inputs()
FALLBACK = [(3, 64, 7, 2, 3, [(16, 16), (9, 5)], True, False, True), (3, 65, 5, 1, 2, [(6, 7), (1, 1)], True, True, True),
            (49, 64, 3, 1, 1, [(6, 8), (15, 20)], True, True, True), (49, 128, 5, 1, 2, [(5, 6)], False, True, True),
            (64, 128, 5, 1, 2, [(7, 9)], True, False, True), (64, 136, 3, 1, 1, [(9, 11), (2, 3)], True, True, False), "tie"]


def fallback_id(c):
    return "tie" if c == "tie" else "%d-%d-k%ds%dp%d%s%s" % (c[:5] + ("-res" if c[7] else "", "" if c[8] else "-no_w_tc"))


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("case", FALLBACK, ids=fallback_id)
def test_tf32_engine_fallback_bits(rf, case, relu):
    """Engine 1 on shapes it runs on the SIMT kernel: with ReLU the outputs are tf32_rna of the FMA chain (and TF32 values),
    without ReLU the chain itself, unrounded."""
    if case == "tie":
        xs, w, b, rs = tie_inputs()
        k, stride, pad, with_tc = 1, 1, 0, True
    else:
        cin, cout, k, stride, pad, sizes, bias, res, with_tc = case
        xs, w, b, rs = inputs(11 + cin + k, cin, cout, k, stride, pad, sizes, bias, res)
    w_tc = R.tf32_round(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)).contiguous().cuda() if with_tc else None
    y, guard = run(rf, xs, w, b, rs, k, stride, pad, relu, engine=1, w_tc=w_tc)
    ref = reference(xs, w, b, rs, stride, pad, relu, round_out=relu)
    assert_bits(y, ref, "engine 1 fallback %s relu %s" % (fallback_id(case), relu))
    assert_guard(guard)
    if relu:
        assert bool(R.is_tf32(y).all())
    else:
        assert not bool(R.is_tf32(y).all())
    if case == "tie" and relu:
        plain = reference(xs, w, b, rs, stride, pad, True)
        assert bool((R.tf32_round(plain) != y).any()), "no tie where nearest-even and cvt.rna differ"


# ------------------------------------------------------------------ the layer runner on engine 0
def random_bn(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                n = m.num_features
                m.weight.copy_(torch.rand(n, generator=g) + 0.5)
                m.bias.copy_(torch.randn(n, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(n, generator=g) + 0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["NetFlowCoarse", "NetMatchability"])
def test_head_program_on_engine0_bits(rf, net):
    """The head's layer program (four 3x3 convolutions 64 (49 + 15 zero channels) -> 512 -> 256 -> 128 -> 49 / 1) through
    rf_run_layers on engine 0 == the FMA chains of its folded layers, one after the other, on a ragged pair."""
    torch.manual_seed(5)
    m = getattr(rf.model, net)(7)
    random_bn(m, 6)
    m = m.cuda().eval()
    prog = m._folded(0)
    hw = [(6, 8), (15, 20)]
    g = torch.Generator().manual_seed(8)
    P = sum(h * w for h, w in hw)
    data = torch.zeros(P, 64)
    data[:, :49] = torch.rand(P, 49, generator=g) * 2 - 1
    out, ohw = prog.run(rf.ops.Ragged(data.cuda(), hw), 0)
    torch.cuda.synchronize()
    assert ohw == hw
    x = [t.cuda() for t in R.images(data, hw)]
    for op in prog.ops:
        fc = op[9]
        w = fc.w.view(fc.k, fc.k, fc.cin, fc.cout).permute(3, 2, 0, 1)
        y = FR.conv_chain_images(x, w, fc.bias, None, fc.stride, fc.pad, bool(op[8]))
        x = [t.cuda() for t in R.images(y.cpu(), hw)]
    assert tuple(out.shape) == (P, 49 if net == "NetFlowCoarse" else 1)
    assert_bits(out.float(), y, net)


# ------------------------------------------------------------------ correlation, precision 0
def random_features(C, NA, NB, seed):
    """test_gpu_matching.test_random_features' features as [N, C] rows."""
    rs = np.random.RandomState(seed)
    A = np.abs(rs.randn(C, NA)).astype(np.float32)
    B = np.abs(rs.randn(C, NB)).astype(np.float32)
    n = min(NA, NB) // 2
    B[:, :n] = A[:, rs.permutation(NA)[:n]] + 0.1 * np.abs(rs.randn(C, n)).astype(np.float32)
    A /= np.linalg.norm(A, axis=0, keepdims=True)
    B /= np.linalg.norm(B, axis=0, keepdims=True)
    if NB > 2:
        B[:, 1] = 0
    return torch.from_numpy(np.ascontiguousarray(A.T)), torch.from_numpy(np.ascontiguousarray(B.T))


def underflow_features():
    """Three mutual pairs with scores 2^-80 (fp32 v * v underflows to 0: dropped), 2^-70 (v * v = 2^-140, subnormal: kept
    without flush to zero) and 2^-60 (kept); every other score is 0."""
    A = torch.zeros(4, 8)
    B = torch.zeros(5, 8)
    for i, (j, e) in enumerate(((0, -40), (2, -35), (3, -30))):
        A[i, i] = 2.0 ** e
        B[j, i] = 2.0 ** e
    return A, B


CORR = ["golden", "ties", "negative", "row1", "col1", "NA51200", "NA51201", "NA0", "NB0", "underflow"] + \
       ["random%d" % i for i in range(7)]
RANDOM = [(1024, 13065, 1200, 0), (1024, 2107, 300, 1), (64, 129, 127, 2), (16, 5, 3, 3), (256, 1, 1, 4), (1024, 300, 1200, 5),
          (36, 500, 260, 6)]


def corr_features(case):
    if case == "golden":
        g = golden("mutual_matching")
        return torch.from_numpy(np.ascontiguousarray(g["featA"].T)), torch.from_numpy(np.ascontiguousarray(g["featB"].T))
    if case.startswith("random"):
        return random_features(*RANDOM[int(case[6:])])
    if case.startswith("NA5"):
        rs = np.random.RandomState(12)
        A, B = rs.randn(int(case[2:]), 64).astype(np.float32), rs.randn(300, 64).astype(np.float32)
        return torch.from_numpy(A), torch.from_numpy(B)
    if case == "NA0":
        return torch.zeros(0, 64), torch.randn(30, 64)
    if case == "NB0":
        return torch.randn(30, 64), torch.zeros(0, 64)
    if case == "underflow":
        return underflow_features()
    return corr_data(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CORR)
def test_corr_precision0_bits(rf, case):
    """The row and column keys in the workspace bit-equal to the FMA-chain keys, and idx1, idx2 and count exactly the mutual
    pairs.  NA 51200 / 51201 are the last size the column-driven compaction takes and the first the row-driven one does."""
    A, B = corr_features(case)
    rowk, colk, i1, i2 = corr_call(rf, A, B, 0)
    ref_r, ref_c, r1, r2 = FR.corr_keys(A.cuda(), B.cuda())
    assert np.array_equal(rowk, ref_r), (case, "row keys", int(np.sum(rowk != ref_r)))
    assert np.array_equal(colk, ref_c), (case, "column keys", int(np.sum(colk != ref_c)))
    assert np.array_equal(i1, r1) and np.array_equal(i2, r2), (case, len(i1), len(r1))
    if case in ("NA0", "NB0"):
        assert len(i1) == 0
    if case == "underflow":
        assert i1.tolist() == [1, 2] and i2.tolist() == [2, 3]
    print("correlation %s: %d pairs" % (case, len(i1)))


# ------------------------------------------------------------------ argument checks
@pytest.mark.gpu
@pytest.mark.parametrize("engine", [0, 1])
@pytest.mark.parametrize("which", ["bias", "residual"])
def test_misaligned_bias_or_residual_refused(rf, engine, which):
    """A bias or residual 4 bytes off 16-byte alignment is refused before any launch (the SIMT epilogue reads them as float4
    when Cout % 4 == 0); engine 1 takes this 7x7 shape on the SIMT kernel too."""
    xs, w, b, rs = inputs(4, 3, 64, 7, 2, 3, [(16, 16)], True, True)
    hw = [(16, 16)]
    P = 8 * 8
    bias, res = b.cuda(), nhwc_cuda(rs)
    if which == "bias":
        bias = torch.cat([torch.zeros(1), b]).cuda()[1:]
    else:
        res = torch.cat([torch.zeros(1), R.nhwc(rs).reshape(-1)]).cuda()[1:].view(P, 64)
    w_tc = w.permute(0, 2, 3, 1).reshape(64, -1).contiguous().cuda() if engine == 1 else None
    y = torch.full((P, 64), float("nan"), device="cuda")
    torch.cuda.synchronize()
    n0 = rf._lib.launch_count()
    with pytest.raises(rf._lib.RFError):
        R.conv_call(rf, nhwc_cuda(xs), hw, 3, FR.packed_weights(w).cuda(), w_tc, bias, res, 64, 7, 2, 3, True, engine, y)
    assert rf._lib.launch_count() == n0
    assert bool(torch.isnan(y).all())


@pytest.mark.gpu
def test_residual_of_wrong_size_refused(rf):
    x = rf.ops.Ragged(torch.randn(48, 16).cuda(), [(6, 8)])
    w = torch.randn(9 * 16, 32).cuda()
    bias = torch.randn(32).cuda()
    rf.ops.conv2d(x, w, bias, 32, 3, 1, 1, True, rf.ops.Ragged(torch.randn(48, 32).cuda(), [(6, 8)]), 0)
    with pytest.raises(AssertionError):
        rf.ops.conv2d(x, w, bias, 32, 3, 1, 1, True, rf.ops.Ragged(torch.randn(42, 32).cuda(), [(6, 7)]), 0)
    with pytest.raises(AssertionError):
        rf.ops.conv2d(x, w, bias, 32, 3, 1, 1, True, rf.ops.Ragged(torch.randn(48, 36).cuda(), [(6, 8)]), 0)
    with pytest.raises(AssertionError):
        rf.ops.conv2d(x, w, bias, 32, 3, 2, 1, True, rf.ops.Ragged(torch.randn(48, 32).cuda(), [(6, 8)]), 0)
