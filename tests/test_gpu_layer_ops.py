"""The kernels rf_run_layers runs between the convolutions (max-pool, blur, pool + blur, im2col), the L2 normalisation that
writes the correlation's operands, and the flow / matchability head epilogues, against fp64 references of the values they
read (tests/wgmma_ref.py), element by element, into outputs filled with NaN first.

These are SIMT kernels with fixed fp32 arithmetic, so every allowance follows from the code (u = 2^-24, gamma_n =
n u / (1 - n u)); none is measured.  Apart from the rounding of fp16 and TF32 outputs, every allowance is at least 30x below
2^-11, so a split kernel that loses its lo plane fails.  The layer ops run as one-op LayerPrograms on engines 0 (fp32),
1 (fp32, outputs rounded to TF32), 2 (fp16) and 4 (split), the way the networks run them."""
import numpy as np
import pytest
import torch

import wgmma_ref as R
from test_gpu_wgmma_edges import SIXTEEN, _bits, _slice

pytestmark = pytest.mark.gpu

ENGINES = (0, 1, 2, 4)
KIND = {0: "f32", 1: "f32", 2: "f16", 4: "split"}
OUT = {0: (0.0, 0.0), 1: (R.R_TF32, 0.0), 2: (R.R_F16, R.ATOL["f16"]), 4: (R.R_SPLIT, R.ATOL["split"])}   # (r_out, atol)
CHANNELS = {0: (4, 64, 128, 132), 1: (4, 64, 128, 132), 2: (8, 64, 128, 264), 4: (8, 64, 128, 264)}   # 132 / 264: 33 vectors
assert R.gamma(9) * 30 <= R.ELEVEN_BIT and (R.gamma(264) / 2 + 2 * R.U) * 30 <= R.ELEVEN_BIT


# ------------------------------------------------------------------ inputs and one-op programs
def layer_images(seed, c, sizes, style):
    """Seeded fp32 (1, C, H, W) CPU images.  "ties": few distinct values (duplicate maxima in every window); "negative":
    every value < 0 (the padding must never win a max); "tiny": a third of the values below 2^-14 (fp16 subnormals, subnormal
    hi planes)."""
    g = torch.Generator().manual_seed(seed)
    xs = []
    for h, w in sizes:
        x = torch.randn(1, c, h, w, generator=g)
        if style == "ties":
            x = torch.randint(-2, 3, (1, c, h, w), generator=g).float() * 0.75
        elif style == "negative":
            x = -(x.abs() + 0.5)
        elif style == "tiny":
            x = torch.where(torch.rand(1, c, h, w, generator=g) < 0.33, x * 2.0 ** -18, x)
        xs.append(x)
    return xs


def build(op, cin):
    from ransac_flow_b200.program import LayerProgram
    P = LayerProgram(cin)
    if op[0] == "maxpool":
        P.maxpool(0, *op[1:])
    elif op[0] == "blur":
        P.blur(0, op[1])
    elif op[0] == "poolblur":
        P.poolblur(0)
    else:
        P.im2col(0, *op[1:])
    return P


def out_size(op, h, w):
    if op[0] == "maxpool":
        return R.out_hw(h, w, *op[1:])
    if op[0] == "blur":
        return R.out_hw(h, w, 3, op[1], 1)
    if op[0] == "poolblur":
        return R.out_hw(h, w, 4, 2, 1)
    return R.out_hw(h, w, op[1], op[2], op[3])


def run_op(rf, P, xd, hw, engine):
    """Runs the program twice, the second time into its output buffer filled with NaN; returns (output view, out hw)."""
    x = rf.ops.Ragged(xd, hw)
    out, ohw = P.run(x, engine)
    out.fill_(float("nan"))
    out, ohw = P.run(x, engine)
    torch.cuda.synchronize()
    return out, ohw


def layer_run(rf, engine, op, xs):
    """One pool / blur / pool + blur op on ``engine``: (raw output, out hw, fp64 outputs per image, fp64 operand images)."""
    hw = [(x.shape[2], x.shape[3]) for x in xs]
    xd, xq = R.operand(R.nhwc(xs), KIND[engine])
    out, ohw = run_op(rf, build(op, xs[0].shape[1]), xd.contiguous().cuda(), hw, engine)
    assert ohw == [out_size(op, h, w) for h, w in hw]
    assert out.dim() == (3 if engine == 4 else 2)
    got = R.images(R.from_split(out) if engine == 4 else out.double(), ohw)
    return out, ohw, got, R.images(xq.cuda(), hw)


def layer_check(rf, engine, op, xs, what):
    """max-pool: equal to the fp64 max of the operands (fp32 / fp16 bit-equal; split: from_split(out) within ATOL["split"],
    values not planes: re-splitting a tie may flip hi / lo).  blur / pool + blur: r_out |ref| + gamma_9 absref + atol (nine
    fp32 FMAs with exact weights, then the output rounding, whose relative error also applies to the sum's error: gamma_9
    (1 + r_out)); engine 1: every output TF32-representable.  Returns the worst
    error / allowance ratio and the raw output."""
    out, ohw, got, xq = layer_run(rf, engine, op, xs)
    r_out, atol = OUT[engine]
    worst = 0.0
    for i, xi in enumerate(xq):
        name = "%s engine %d image %d" % (what, engine, i)
        if op[0] == "maxpool":
            ref = R.maxpool_ref(xi, *op[1:])
            assert got[i].shape == ref.shape, name
            err = (got[i] - ref).abs()
            assert not bool(err.isnan().any()), name
            assert float(err.max()) <= (R.ATOL["split"] if engine == 4 else 0.0), (name, float(err.max()))
        else:
            ref, absref = R.blur_ref(xi, op[1]) if op[0] == "blur" else R.poolblur_ref(xi)
            worst = max(worst, R.check(got[i], ref, absref, r_out, R.gamma(9) * (1 + r_out), atol, name))
    if engine == 1 and op[0] != "maxpool":
        tf = R.is_tf32(out)
        assert bool(tf.all()), "%s: %d engine-1 outputs are not TF32-rounded" % (what, int((~tf).sum()))
    print("%s engine %d: worst error / allowance %.3g" % (what, engine, worst))
    return worst, out


# ------------------------------------------------------------------ max-pool, blur, pool + blur
POOL_CASES = [("min", [(1, 1)], "randn"), ("1xW", [(1, 37)], "ties"), ("Hx1", [(29, 1)], "negative"),
              ("odd_even", [(17, 23), (8, 6)], "ties"), ("ragged", [(33, 47), (2, 3), (12, 5), (5, 64)], "tiny"),
              ("negative", [(9, 11), (4, 4), (3, 8)], "negative")]


@pytest.mark.parametrize("name,sizes,style", POOL_CASES, ids=[c[0] for c in POOL_CASES])
@pytest.mark.parametrize("ci", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["3/2/1", "2/1/0"])
@pytest.mark.parametrize("engine", ENGINES)
def test_maxpool_equals_fp64_max(rf, engine, kind, ci, name, sizes, style):
    """nn.MaxPool2d(3, 2, 1) (the ResNet trunk) and (2, 1, 0): the maximum of the in-image window, exactly.  Windows with
    duplicate maxima, all-negative windows at the padded border, single pixels, single rows and columns."""
    k, s, p = map(int, kind.split("/"))
    sizes = [(max(h, k - 2 * p), max(w, k - 2 * p)) for h, w in sizes]
    c = CHANNELS[engine][ci]
    layer_check(rf, engine, ("maxpool", k, s, p), layer_images(ci * 7 + k, c, sizes, style), "maxpool %s C %d %s" % (kind, c, name))


BLUR_CASES = [("min", [(2, 2)], "randn"), ("2xW", [(2, 37)], "randn"), ("Hx2", [(29, 2)], "negative"),
              ("odd", [(17, 23), (9, 5)], "tiny"), ("even", [(16, 24), (8, 6)], "randn"),
              ("ragged", [(33, 47), (2, 3), (12, 5), (6, 64), (21, 30), (8, 9)], "tiny")]


@pytest.mark.parametrize("name,sizes,style", BLUR_CASES, ids=[c[0] for c in BLUR_CASES])
@pytest.mark.parametrize("ci", [0, 1, 2, 3])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("engine", ENGINES)
def test_blur_vs_fp64(rf, engine, stride, ci, name, sizes, style):
    """The anti-aliased blur (ReflectionPad2d(1) + [1 2 1]^2 / 16) at strides 1 and 2: the smallest size it allows (2 x 2),
    two-pixel rows and columns, odd and even sizes, ragged batches."""
    c = CHANNELS[engine][ci]
    layer_check(rf, engine, ("blur", stride), layer_images(ci * 5 + stride, c, sizes, style), "blur stride %d C %d %s" % (stride, c, name))


POOLBLUR_CASES = [("min", [(3, 3)], "randn"), ("3xW", [(3, 37)], "ties"), ("Hx3", [(29, 3)], "negative"),
                  ("odd", [(17, 23), (9, 5)], "tiny"), ("even", [(16, 24), (8, 6)], "randn"),
                  ("ragged", [(33, 47), (3, 4), (12, 5), (6, 64), (21, 30), (8, 9)], "tiny")]


@pytest.mark.parametrize("name,sizes,style", POOLBLUR_CASES, ids=[c[0] for c in POOLBLUR_CASES])
@pytest.mark.parametrize("ci", [0, 1, 2, 3])
@pytest.mark.parametrize("engine", ENGINES)
def test_poolblur_vs_fp64(rf, engine, ci, name, sizes, style):
    """FeatureExtractor's stem tail, MaxPool2d(2, 1) + the stride-2 blur fused: the smallest size (3 x 3), three-pixel rows
    and columns, odd and even sizes, ragged batches."""
    c = CHANNELS[engine][ci]
    layer_check(rf, engine, ("poolblur",), layer_images(ci * 3 + 1, c, sizes, style), "poolblur C %d %s" % (c, name))


def test_feature_extractor_stem_tail_pair_size(rf):
    """The pool + blur as a pair runs it: two 480 x 640 images, C = 64, split."""
    layer_check(rf, 4, ("poolblur",), layer_images(11, 64, [(480, 640), (480, 640)], "randn"), "poolblur 2 x 480x640 C 64")


def trunk_pool_sizes():
    """The max-pool input sizes of the 8-image ResNet trunk batch at config 2 (7 scales with scaleR 2 of a 640 x 480 source
    plus the target): the stem outputs of the resized images."""
    from ransac_flow_b200 import coarseAlignFeatMatch as ca
    a = ca.CoarseAlignA.__new__(ca.CoarseAlignA)
    a.strideNet = 16
    sizes = [a._target_size(640, 480, int(480 * s)) for s in ca.scale_list(7, 2)] + [a._target_size(640, 480, 480)]
    return [R.out_hw(h, w, 7, 2, 3) for w, h in sizes]


@pytest.mark.parametrize("engine", ENGINES)
def test_trunk_maxpool_config2_sizes(rf, engine):
    sizes = trunk_pool_sizes()
    assert len(sizes) == 8 and sizes[0] == (480, 640) and sizes[-1] == (240, 320)
    layer_check(rf, engine, ("maxpool", 3, 2, 1), layer_images(2, 64, sizes, "randn"), "trunk maxpool")


# ------------------------------------------------------------------ im2col (the stems)
# engine -> {name: (k, stride, pad, Kpad)}; the smem kernels (ResNet stem: TPX 64 output pixels per CTA row segment,
# FeatureExtractor stem: TPX 128) and, on engines 0 / 1, the three generic instances <7,3,160>, <3,3,32> and <0,0,0>
IM2COL_SHAPES = {
    0: {"resnet": (7, 2, 3, 160), "fe": (3, 1, 1, 32), "7x7s1": (7, 1, 3, 160), "3x3s2": (3, 2, 1, 32), "5x5": (5, 1, 2, 80)},
    2: {"resnet": (7, 2, 3, 192), "fe": (3, 1, 1, 64)},
    4: {"fe": (3, 1, 1, 64)}}
IM2COL_SHAPES[1] = IM2COL_SHAPES[0]
# output widths below, at and above both segments (ResNet stem: Wo = (W - 1) // 2 + 1; FeatureExtractor stem: Wo = W), a
# last segment that is partial, and images of different widths in one batch
IM2COL_SIZES = {"1x1": [(1, 1)], "below": [(3, 63), (2, 125)], "at": [(2, 64), (3, 127), (2, 128)],
                "above": [(3, 65), (2, 129), (4, 259)], "mixed": [(5, 129), (1, 1), (9, 300), (7, 127), (1, 2)]}
IM2COL_CASES = [(e, s, z) for e in ENGINES for s in IM2COL_SHAPES[e] for z in IM2COL_SIZES]


def stem_images(seed, sizes):
    """3-channel fp32 images: half the values with low 13 mantissa bits exactly 0x1000 (a TF32 tie: ties-away and ties-to-even
    differ), some beyond the fp16 range (the split planes saturate at +-65504) and some below 2^-14 (subnormal hi)."""
    g = torch.Generator().manual_seed(seed)
    xs = []
    for h, w in sizes:
        x = torch.randn(1, 3, h, w, generator=g)
        u = torch.rand(1, 3, h, w, generator=g)
        b = x.view(torch.int32)
        x = torch.where(u < 0.5, ((b & ~0x1FFF) | 0x1000).view(torch.float32), x)
        x = torch.where(u > 0.95, x.sign() * 1e5, torch.where(u > 0.9, x * 2.0 ** -20, x))
        xs.append(x)
    return xs


def im2col_expected(engine, patch):
    """What the kernel must store for the fp32 patch rows: the values (engine 0), their TF32 rounding with ties away from
    zero (engine 1), fp16 (engine 2), split planes (engine 4)."""
    return {0: patch, 1: R.tf32_rna(patch), 2: patch.half(), 4: R.to_split(patch)}[engine]


def im2col_run(rf, engine, shape, xs):
    k, s, p, kpad = shape
    hw = [(x.shape[2], x.shape[3]) for x in xs]
    out, ohw = run_op(rf, build(("im2col", k, s, p, kpad), 3), R.nhwc(xs).cuda(), hw, engine)
    assert ohw == [R.out_hw(h, w, k, s, p) for h, w in hw]
    exp = im2col_expected(engine, torch.cat([R.im2col_ref(x.cuda(), k, s, p, kpad) for x in xs], 0))
    return out, exp


@pytest.mark.parametrize("engine,shape,sizes", IM2COL_CASES, ids=["e%d-%s-%s" % c for c in IM2COL_CASES])
def test_im2col_bit_exact(rf, engine, shape, sizes):
    """im2col's rows are copies: the k x k patch in (r, s, c) order, zero outside the image and in the Kpad columns, bit for
    bit in the engine's element type."""
    xs = stem_images(len(sizes) * 13 + engine, IM2COL_SIZES[sizes])
    out, exp = im2col_run(rf, engine, IM2COL_SHAPES[engine][shape], xs)
    assert out.shape == exp.shape and out.dtype == exp.dtype
    same = _bits(out) == _bits(exp)
    assert bool(same.all()), "%d of %d elements differ; first at %s" % (int((~same).sum()), same.numel(), tuple((~same).nonzero()[0].tolist()))


# ------------------------------------------------------------------ sixteen-image ragged batches
SIXTEEN3 = [(max(h, 3), max(w, 3)) for h, w in SIXTEEN]
SIXTEEN_OPS = {"maxpool": (("maxpool", 3, 2, 1), SIXTEEN), "blur2": (("blur", 2), SIXTEEN3), "blur1": (("blur", 1), SIXTEEN3),
               "poolblur": (("poolblur",), SIXTEEN3)}


def sixteen_check(rf, engine, run_batch):
    """run_batch(list of image indices) -> (raw output, out hw).  Each image of the sixteen equals that image run alone, bit
    for bit; a seventeenth image is refused."""
    y, ohw = run_batch(list(range(16)))
    y = y.clone()
    o = np.cumsum([0] + [h * w for h, w in ohw])
    for i in range(16):
        alone, _ = run_batch([i])
        assert torch.equal(_bits(_slice(y, o, i)), _bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        run_batch(list(range(16)) + [0])


@pytest.mark.parametrize("op", list(SIXTEEN_OPS))
@pytest.mark.parametrize("engine", ENGINES)
def test_sixteen_image_batch_equals_images_alone(rf, engine, op):
    spec, sizes = SIXTEEN_OPS[op]
    c = CHANNELS[engine][1]
    xs = layer_images(16 + engine, c, sizes, "tiny")
    layer_check(rf, engine, spec, xs, "%s sixteen images" % op)
    P = build(spec, c)

    def run_batch(idx):
        sel = [xs[i] for i in idx]
        xd, _ = R.operand(R.nhwc(sel), KIND[engine])
        return run_op(rf, P, xd.contiguous().cuda(), [(x.shape[2], x.shape[3]) for x in sel], engine)
    sixteen_check(rf, engine, run_batch)


@pytest.mark.parametrize("engine", ENGINES)
def test_im2col_sixteen_image_batch_equals_images_alone(rf, engine):
    shape = IM2COL_SHAPES[engine]["fe" if engine == 4 else "resnet"]
    xs = stem_images(160 + engine, SIXTEEN)
    out, exp = im2col_run(rf, engine, shape, xs)
    assert torch.equal(_bits(out), _bits(exp))
    k, s, p, kpad = shape
    P = build(("im2col", k, s, p, kpad), 3)

    def run_batch(idx):
        sel = [xs[i] for i in idx]
        return run_op(rf, P, R.nhwc(sel).cuda(), [(x.shape[2], x.shape[3]) for x in sel], engine)
    sixteen_check(rf, engine, run_batch)


# ------------------------------------------------------------------ refusals
REFUSALS = [(0, ("maxpool", 3, 2, 1), 6, (8, 8)), (1, ("blur", 2), 6, (8, 8)), (0, ("poolblur",), 2, (8, 8)),
            (2, ("maxpool", 3, 2, 1), 12, (8, 8)), (4, ("blur", 1), 4, (8, 8)), (2, ("poolblur",), 4, (8, 8)), (4, ("maxpool", 2, 1, 0), 20, (8, 8)),
            (0, ("blur", 2), 4, (1, 8)), (2, ("blur", 1), 8, (8, 1)), (4, ("blur", 2), 8, (1, 1)),
            (1, ("poolblur",), 4, (2, 8)), (2, ("poolblur",), 8, (8, 2)), (4, ("poolblur",), 8, (2, 2)),
            (2, ("im2col", 7, 2, 3, 160), 3, (16, 16)), (2, ("im2col", 3, 1, 1, 32), 3, (16, 16)), (2, ("im2col", 5, 1, 2, 80), 3, (16, 16)),
            (4, ("im2col", 7, 2, 3, 192), 3, (16, 16)), (4, ("im2col", 3, 2, 1, 64), 3, (16, 16))]


@pytest.mark.parametrize("engine,op,c,size", REFUSALS)
def test_layer_op_refusals_launch_nothing(rf, engine, op, c, size):
    """fp32 C % 4 != 0, fp16 / split C % 8 != 0, blur below 2 x 2, pool + blur below 3 x 3, fp16 / split im2col outside the
    two stems: an RFError before any launch."""
    P = build(op, c)
    xs = layer_images(0, c, [size], "randn")
    xd = R.nhwc(xs) if op[0] == "im2col" else R.operand(R.nhwc(xs), KIND[engine])[0]
    x = rf.ops.Ragged(xd.contiguous().cuda(), [size])
    torch.cuda.synchronize()
    n0 = rf._lib.launch_count()
    with pytest.raises(rf._lib.RFError):
        P.run(x, engine)
    assert rf._lib.launch_count() == n0


def engine_only_program(op):
    """One-op programs whose ops the library runs on some activation formats only; the Python-side guards are switched off so
    that the library's own check is the one exercised."""
    from ransac_flow_b200.model import FoldedConv
    from ransac_flow_b200.program import LayerProgram
    g = torch.Generator().manual_seed(5)
    if op == "maxpool":
        return build(("maxpool", 3, 2, 1), 8), 8
    if op == "conv_dual":
        fa, fb = (FoldedConv(torch.randn(64, 64, 1, 1, generator=g) / 8, None, 1, pad=0, device="cuda") for _ in range(2))
        P = LayerProgram(64, device="cuda")
        P.conv_dual(0, 0, FoldedConv.concat_k(fa, fb), 1, relu=True)
        P.split_only = False
        return P, 64
    P = LayerProgram(3, device="cuda")
    if op == "stem3":
        P.stem3(0, torch.randn(64, 3, 3, 3, generator=g) / 5, None)
        P.split_only = False
    else:
        P.stem7_fused(0, torch.randn(64, 3, 7, 7, generator=g) / 12, None)
        P.f16_only = False
    return P, 3


# RF_OP_STEM3 / RF_OP_CONV_DUAL: engine 4 only; RF_OP_STEM7: engines 2 / 4; engines 3 and 5 are conv output modes, not formats
ENGINE_REFUSALS = [("stem3", 0), ("stem3", 1), ("stem3", 2), ("conv_dual", 0), ("conv_dual", 1), ("conv_dual", 2),
                   ("stem7", 0), ("stem7", 1), ("maxpool", 3), ("maxpool", 5)]


@pytest.mark.parametrize("op,engine", ENGINE_REFUSALS)
def test_layer_op_engine_refusals_launch_nothing(rf, op, engine):
    P, c = engine_only_program(op)
    dtype = torch.float16 if engine == 2 and op != "stem7" else torch.float32
    x = rf.ops.Ragged(torch.zeros(16 * 16, c, device="cuda", dtype=dtype), [(16, 16)])
    torch.cuda.synchronize()
    n0 = rf._lib.launch_count()
    with pytest.raises(rf._lib.RFError):
        P.run(x, engine)
    assert rf._lib.launch_count() == n0


# ------------------------------------------------------------------ L2 normalisation (rf_l2norm_nhwc / _f16_nhwc / _split_nhwc)
def l2_rows(seed, P, C, eps_rows):
    """Rows over six decades of scale, a row of zeros and, for fp32 inputs, rows with norms in (1e-14, 1e-13) (the eps branch:
    x / 1e-12)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(P, C, generator=g) * torch.logspace(-3, 3, max(P, 1))[:P].view(-1, 1)
    if P > 1:
        x[P // 2] = 0
    if eps_rows and P > 2:
        r = torch.tensor([i for i in range(1, P, 3) if i != P // 2])
        x[r] = x[r] / x[r].norm(dim=1, keepdim=True) * (1e-14 + 9e-14 * torch.rand(len(r), 1, generator=g))
    return x


def l2_mask(P, masked):
    if not masked:
        return None
    m = torch.ones(P, dtype=torch.uint8)
    m[::3] = 0
    return m


def l2_call(rf, kind, xd, P, C, mask, y, planes):
    lib, ptr, st = rf._lib.lib, rf._lib.ptr, rf._lib.stream()
    md = mask.cuda() if mask is not None else None
    if kind == "split":
        rc = lib.rf_l2norm_split_nhwc(ptr(xd), P, C, ptr(md), ptr(y), ptr(planes[0]) if planes is not None else None,
                                      ptr(planes[1]) if planes is not None else None, st)
    elif kind == "f16":
        rc = lib.rf_l2norm_f16_nhwc(ptr(xd), P, C, ptr(md), ptr(y), st)
    else:
        rc = lib.rf_l2norm_nhwc(ptr(xd), P, C, ptr(md), ptr(y), st)
    rf._lib.check(rc)
    torch.cuda.synchronize()


L2_CASES = [(kind, P, C) for kind, cs in (("f32", (4, 132)), ("f16", (8, 264)), ("split", (8, 264))) for P in (0, 1, 7, 8, 9) for C in cs] + \
           [("f32", 13065, 1024), ("f16", 13065, 1024), ("split", 13065, 1024)]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("kind,P,C", L2_CASES)
def test_l2norm_vs_fp64(rf, kind, P, C, masked):
    """x / max(||x||, fp32(1e-12)) per row within (r_out + gamma_C / 2 + 2u) |ref| + atol: the C-term fp32 sum of squares
    (gamma_C, halved by the square root), the rounding of sqrtf and of the division.  P = 0 launches nothing; P = 7 / 9 leave
    a partial block of 8 warps; P = 13065 is NA at config 2; C = 132 / 264 wrap the lanes.  Masked rows are zero in y and in
    both planes; a row of zeros gives zeros.  Split input: the y-only, planes-only and both-outputs calls, planes bit-equal
    to each other and to to_split(y)."""
    x = l2_rows(P * 7 + C, P, C, kind == "f32")
    mask = l2_mask(P, masked)
    xd, xq = R.operand(x, kind)
    xd = xd.contiguous().cuda()
    ref = R.l2norm_ref(xq.cuda(), mask)
    bnd = R.gamma(C) / 2 + 2 * R.U
    n0 = rf._lib.launch_count()
    # buffers of at least one row, so that P = 0 still passes non-null pointers; the checks read the first P rows
    y32 = lambda: R.nan_output((max(P, 1), C), torch.float32)
    y16 = lambda: R.nan_output((2, max(P, 1), C), torch.float16)
    y = y32()
    if kind != "split":
        l2_call(rf, kind, xd, P, C, mask, y, None)
    else:
        both = y16()
        l2_call(rf, kind, xd, P, C, mask, y, both)
        y_only = y32()
        l2_call(rf, kind, xd, P, C, mask, y_only, None)
        planes = y16()
        l2_call(rf, kind, xd, P, C, mask, None, planes)
        y, y_only, both, planes = y[:P], y_only[:P], both[:, :P], planes[:, :P]
        assert torch.equal(_bits(y_only), _bits(y))
        assert torch.equal(_bits(planes), _bits(both)) and torch.equal(_bits(both), _bits(R.to_split(y)))
        R.check(R.from_split(planes), ref, ref, R.R_SPLIT + bnd, 0.0, R.ATOL["split"], "l2norm planes P %d C %d" % (P, C))
        if mask is not None:
            assert not bool(planes[:, ::3].any())
    if P == 0:
        assert rf._lib.launch_count() == n0
        return
    y = y[:P]
    worst = R.check(y, ref, ref, bnd, 0.0, 0.0, "l2norm %s P %d C %d" % (kind, P, C))
    if P > 1:
        assert not bool(y[P // 2].any())
    if mask is not None:
        assert not bool(y[::3].any())
    md = mask.cuda() if mask is not None else None
    assert torch.equal(_bits(rf.ops.l2norm(xd, md)), _bits(y))           # the ops wrapper picks the same kernel
    if kind == "split":
        assert torch.equal(_bits(rf.ops.l2norm_planes(xd, md)), _bits(planes))
    print("l2norm %s P %d C %d mask %s: worst error / allowance %.3g" % (kind, P, C, masked, worst))


def test_l2norm_refuses_unaligned_channels(rf):
    lib, ptr, st = rf._lib.lib, rf._lib.ptr, rf._lib.stream()
    n0 = rf._lib.launch_count()
    x32, y = torch.ones(4, 6, device="cuda"), torch.empty(4, 8, device="cuda")
    x16 = torch.ones(2, 4, 12, device="cuda", dtype=torch.float16)
    assert lib.rf_l2norm_nhwc(ptr(x32), 4, 6, None, ptr(y), st) != 0
    assert lib.rf_l2norm_f16_nhwc(ptr(x16), 4, 12, None, ptr(y), st) != 0
    assert lib.rf_l2norm_split_nhwc(ptr(x16), 4, 12, None, ptr(y), None, None, st) != 0
    assert lib.rf_l2norm_split_nhwc(ptr(x16), 4, 8, None, None, None, None, st) != 0          # no output
    assert rf._lib.launch_count() == n0


# ------------------------------------------------------------------ head epilogues
def softmax_flow_call(rf, logits, k):
    n, kk, h, w = logits.shape
    ld = logits.permute(0, 2, 3, 1).contiguous().cuda()
    flow = R.nan_output((n, 2, h, w), torch.float32)
    rf._lib.check(rf._lib.lib.rf_softmax_flow(rf._lib.ptr(ld), n, h, w, k, rf._lib.ptr(flow), rf._lib.stream()))
    torch.cuda.synchronize()
    return flow


SOFTMAX_SHAPES = [(1, 1, 1), (2, 5, 9), (3, 17, 3), (1, 60, 80)]


@pytest.mark.parametrize("spread", [3.0, 60.0])
@pytest.mark.parametrize("n,h,w", SOFTMAX_SHAPES)
@pytest.mark.parametrize("k", [3, 5, 7])
def test_softmax_flow_vs_fp64(rf, k, n, h, w, spread):
    """The flow head's epilogue (softmax over k*k channels, expected offset / size * 2) within
    (k^2 + 8) u (2 / size) sum p |g| + u |ref|: expf within 2 ulp (no fast-math), a k^2-term fp32 sum, three roundings.
    Logits lie on a 2^-12 grid below 2^11, so logit - max is exact, as the bound assumes; spread 60 puts logits beyond
    +-90, where expf without the max subtraction overflows.  Below 2^-126 fp32 rounds to an absolute 2^-150 rather than a
    relative u: e^(l - m) that underflow, the k^2 subnormal products e * g and sums, and the three roundings after them add
    at most (2 k^3 + 4) 2^-149 (the last factor 2 / size is up to 2) (the spread logits reach flows near 1e-50)."""
    g = torch.Generator().manual_seed(k * 100 + h)
    logits = torch.round(torch.randn(n, k * k, h, w, generator=g) * spread * 4096) / 4096
    if spread > 10:                                     # one logit of 100 per pixel at a random tap
        logits.scatter_(1, torch.randint(0, k * k, (n, 1, h, w), generator=g), 100.0)
    flow = softmax_flow_call(rf, logits, k)
    ref, absf = R.softmax_flow_ref(logits.cuda(), k)
    worst = R.check(flow, ref, absf, R.U, (k * k + 8) * R.U, (2 * k ** 3 + 4) * 2.0 ** -149, "softmax_flow k %d" % k)
    wrapped = rf.ops.softmax_flow(rf.ops.Ragged.from_nchw(logits.cuda()), k)
    assert torch.equal(wrapped, flow)
    print("softmax_flow k %d %dx%dx%d spread %g: worst error / allowance %.3g" % (k, n, h, w, spread, worst))


@pytest.mark.parametrize("n", [1, 255, 257, 100000])
def test_sigmoid_vs_fp64(rf, n):
    """The matchability head's sigmoid 1 / (1 + expf(-x)) within 2^-21 |ref| + 2^-126, from saturation at both ends (expf
    overflowing to inf gives 0) through 0."""
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g) * 8
    edges = torch.tensor([-200.0, -104.0, -88.5, -87.0, -20.0, -1e-6, 0.0, 1e-6, 20.0, 88.5, 200.0])
    x[:min(n, len(edges))] = edges[:n]
    xd = x.cuda()
    y = R.nan_output((n,), torch.float32)
    rf._lib.check(rf._lib.lib.rf_sigmoid(rf._lib.ptr(xd), n, rf._lib.ptr(y), rf._lib.stream()))
    torch.cuda.synchronize()
    ref = torch.sigmoid(xd.double())
    worst = R.check(y, ref, torch.zeros_like(ref), 2.0 ** -21, 0.0, 2.0 ** -126, "sigmoid n %d" % n)
    assert torch.equal(rf.ops.sigmoid(xd), y)
    print("sigmoid n %d: worst error / allowance %.3g" % (n, worst))
