"""The direct stems (RF_OP_STEM7 on engines 2 and 4) against fp64 at the edges of their own decomposition: the
FeatureExtractor stem (3x3 / stride 1 / pad 1) with the ResNet-50 stem (7x7 / stride 2 / pad 3) through the same helpers
(tests/stem_ref.py), unfused.  Output sizes on both sides of the 32-column strip and the 4-row step, single rows and columns,
batches in which a CTA runs many units and walks from one image into another of a different width, sixteen images, a NaN guard
band around a caller-owned output, two streams at once - and exact probes of the gather table: integer weights that name their
tap under impulse images, and all-integer images whose every partial sum is exact, both bit for bit against fp64 whatever the
order of accumulation.  tests/test_stem_ref.py holds, without a GPU, that the batches below run into the situations they are
chosen for on 132 and 114 SMs.  The pooled form of the 7x7 stem is held to the unfused one in tests/test_gpu_stem_pool.py."""
import pytest
import torch

import stem_ref as S
import wgmma_ref as R

pytestmark = pytest.mark.gpu

KS = {7: "7x7s2", 3: "3x3s1"}


def in_size(o, k):
    """An input extent whose stem output extent is o."""
    return S.STRIDE[k] * (o - 1) + 1


def in_sizes(out_sizes, k):
    return [(in_size(h, k), in_size(w, k)) for h, w in out_sizes]


# stem OUTPUT sizes (the input sizes follow with in_sizes): one pixel; one row below, at and past one and two strips; one
# column below, at and past one and two steps; a ragged batch of odd sizes; the pair size; one unit per CTA at the 3x3 stem;
# sixteen images
OUT_SIZES = {
    "1x1": [(1, 1)], "1x31": [(1, 31)], "1x32": [(1, 32)], "1x33": [(1, 33)], "1x65": [(1, 65)],
    "3x1": [(3, 1)], "4x1": [(4, 1)], "5x1": [(5, 1)], "9x1": [(9, 1)],
    "ragged": [(17, 35), (3, 5), (9, 33), (15, 61), (65, 15), (33, 64), (5, 31), (2, 97)],
    "480x640": [(480, 640)], "97x131": [(97, 131)],
    "sixteen": [(5 + 9 * i, 7 + 13 * i) for i in range(16)],
}
# the 7x7 stem already runs these in tests/test_gpu_wgmma_edges.py::test_stem7_layer_vs_fp64
HELD_ELSEWHERE = {7: ("1x1", "480x640", "sixteen"), 3: ()}
FP64_CASES = [(k, name) for k in KS for name in OUT_SIZES if name not in HELD_ELSEWHERE[k]]

# five images around 300 x 400 stem pixels of different widths: about 18 (3x3) / 37 (7x7) units per CTA on 132 SMs
MANY_UNITS = [(300, 400), (301, 391), (299, 417), (302, 385), (298, 409)]
# partial strips and steps in every image, and strips next to each other in the output rows
GUARD_SIZES = [(37, 53), (61, 29), (5, 131), (1, 1), (23, 70)]
# input sizes of the exact probes: strips and steps on both sides of their seams, and widths and heights whose remainders
# modulo 7 and 3 put the impulse lattices of stem_ref.impulse_images at every offset against those seams
PROBE_SIZES = [(19, 141), (9, 67), (18, 33), (19, 68), (1, 1), (8, 69), (20, 64), (21, 70), (70, 9), (5, 71), (22, 12), (23, 72), (4, 32),
               (3, 73), (24, 97), (12, 129)]


def images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]


@pytest.mark.parametrize("k,name", FP64_CASES, ids=["%s-%s" % (KS[k], n) for k, n in FP64_CASES])
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_vs_fp64(rf, engine, k, name):
    """Convolution + folded BN + ReLU against fp64 of the operands, element by element, in an output pre-filled with NaN."""
    P, fc = S.stem_program(*S.stem_args(7, k))
    xs = images(in_sizes(OUT_SIZES[name], k), 100 + list(OUT_SIZES).index(name))
    out, ohw = S.run_nan(rf, P, xs, engine)
    assert [tuple(v) for v in ohw] == OUT_SIZES[name]
    worst = S.check_stem(fc, k, xs, engine, out, ohw, "stem %s engine %d %s" % (KS[k], engine, name))
    print("stem %s engine %d %s: worst error / allowance %.3g" % (KS[k], engine, name, worst))


@pytest.mark.parametrize("k", list(KS), ids=list(KS.values()))
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_many_units_per_cta_across_images(rf, engine, k):
    """CTAs that run many units, start inside strips and walk from one image into the next of another width: fp64 element by
    element, two calls equal bit for bit, and every image's part equal to that image run alone."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = in_sizes(MANY_UNITS, k)
    d = S.describe(sizes, k, False, sms)
    need = ("three_units", "starts_mid_strip", "crosses_strip", "crosses_image_width")
    if not all(d[s] for s in need):
        assert sms not in (132, 114), d
        pytest.skip("on %d SMs this batch does not run into %s: choose another" % (sms, [s for s in need if not d[s]]))
    P, fc = S.stem_program(*S.stem_args(11, k))
    xs = images(sizes, 12)
    batch, ohw = S.run_nan(rf, P, xs, engine)
    batch = batch.clone()
    worst = S.check_stem(fc, k, xs, engine, batch, ohw, "stem %s engine %d" % (KS[k], engine))
    again, _ = S.run_nan(rf, P, xs, engine)
    assert torch.equal(S.bits(batch), S.bits(again))
    for i in range(len(xs)):
        alone, _ = S.run_nan(rf, P, [xs[i]], engine)
        assert torch.equal(S.bits(S.image_part(batch, ohw, i)), S.bits(alone)), i
    print("stem %s engine %d, %d units on %d SMs: worst error / allowance %.3g" %
          (KS[k], engine, S.stem_units(sizes, k, S.STRIDE[k], False)["total"], sms, worst))


@pytest.mark.parametrize("engine", [2, 4])
def test_stem3_sixteen_images_equal_images_alone(rf, engine):
    """The 3x3 stem on sixteen images: each image's part equals that image run alone bit for bit; a seventeenth is refused."""
    P, _ = S.stem_program(*S.stem_args(8, 3))
    sizes = OUT_SIZES["sixteen"]
    xs = images(sizes, 3)
    batch, ohw = S.run_nan(rf, P, xs, engine)
    batch = batch.clone()
    for i in range(16):
        alone, _ = S.run_nan(rf, P, [xs[i]], engine)
        assert torch.equal(S.bits(S.image_part(batch, ohw, i)), S.bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        P.run(rf.ops.Ragged(R.nhwc(xs + xs[:1]).cuda(), sizes + sizes[:1]), engine)


@pytest.mark.parametrize("engine", [2, 4])
def test_stem3_leaves_guard_band(rf, engine):
    """The 3x3 stem into a caller-owned buffer with a NaN guard of two tiles (128 pixels x 64 channels each) before its start
    and after its end, at sizes with partial strips and steps: the guards stay NaN and every output element is written and
    right.  The two planes of the split output are one allocation (the lo plane starts where the hi plane ends), so a store
    past the end of the hi plane or before the start of the lo plane lands in output rows, which the fp64 check covers."""
    guard = 2 * 128 * 64                                        # fp16 elements
    P, fc = S.stem_program(*S.stem_args(13, 3))
    xs = images(GUARD_SIZES, 14)
    x = rf.ops.Ragged(R.nhwc(xs).cuda(), GUARD_SIZES)
    # the program's compiled entry for this batch, with the guarded buffer in place of its own output buffer
    c = P._compile(x.hw, x.data.device, engine == 2, engine == 4)
    n = c["out_elems"] // 2
    flat = torch.full((n + 2 * guard,), float("nan"), dtype=torch.float16, device="cuda")
    c["bufs"][c["out_slot"]] = flat[guard:guard + n].view(torch.uint8)
    P._compiled[(tuple(x.hw), str(x.data.device), engine)] = c
    out, ohw = P.run(x, engine)
    assert len(P._compiled) == 1
    torch.cuda.synchronize()
    assert out.data_ptr() == flat.data_ptr() + 2 * guard
    assert bool(torch.isnan(flat[:guard]).all()), "the stem wrote before its output"
    assert bool(torch.isnan(flat[guard + n:]).all()), "the stem wrote past its output"
    worst = S.check_stem(fc, 3, xs, engine, out, ohw, "guarded stem engine %d" % engine)
    print("guarded stem 3x3s1 engine %d: worst error / allowance %.3g" % (engine, worst))


@pytest.mark.parametrize("engine", [2, 4])
def test_stem3_two_streams(rf, engine):
    """Two 3x3 stems on two streams at once (two of its CTAs share an SM's shared memory by design) give what each gives
    alone."""
    progs = [S.stem_program(*S.stem_args(s, 3))[0] for s in (21, 22)]
    inputs = [images(OUT_SIZES["ragged"], 121), images([(480, 640), (240, 320)], 122)]
    alone = [S.run_nan(rf, P, xs, engine)[0].clone() for P, xs in zip(progs, inputs)]
    xs = [rf.ops.Ragged(R.nhwc(x).cuda(), [(t.shape[2], t.shape[3]) for t in x]) for x in inputs]
    for P in progs:
        for c in P._compiled.values():
            c["bufs"][c["out_slot"]].view(torch.float16).fill_(float("nan"))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    outs = []
    for P, x, st in zip(progs, xs, streams):
        with torch.cuda.stream(st):
            outs.append(P.run(x, engine)[0])
    torch.cuda.synchronize()
    for i, out in enumerate(outs):
        assert torch.equal(S.bits(out), S.bits(alone[i])), i


# ------------------------------------------------------------------ exact probes of the gather table
def probe_program(weight, engine, k):
    """The stem with ``weight`` (integers) and no BatchNorm: the packed weights must be those integers, and there is no bias."""
    P, fc = S.stem_program(weight, None)
    assert fc.bias is None
    assert torch.equal(S.packed_weights(fc, engine, k), weight.double()), "the packed weights are not the probe's integers"
    if engine == 4:
        assert not bool(fc.w_split[1].any()), "integer weights with a lo plane"
    return P


@pytest.mark.parametrize("k", list(KS), ids=list(KS.values()))
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_tap_probes(rf, engine, k):
    """Impulse images under weights that name their tap: every output element is one exact product, so the output equals the
    fp64 convolution bit for bit on both engines, and a mismatch names the tap it should hold and the tap it holds."""
    weight = S.probe_weight(k)
    P = probe_program(weight, engine, k)
    xs = S.impulse_images(PROBE_SIZES, k)
    out, ohw = S.run_nan(rf, P, xs, engine)
    got = S.output_images(out, ohw, engine)
    for i, x in enumerate(xs):
        ref, _ = S.stem_ref(x.cuda(), weight.cuda(), None, k, S.STRIDE[k], (k - 1) // 2)
        bad = S.first_mismatch(got[i].cpu(), ref.cpu(), x, k)
        assert bad is None, "stem %s engine %d image %d %s: %s" % (KS[k], engine, i, PROBE_SIZES[i], bad)


@pytest.mark.parametrize("k", list(KS), ids=list(KS.values()))
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_integer_images_exact(rf, engine, k):
    """Integer images (|x| <= 8) under integer weights (|w| <= 8): every partial sum is an integer below 2^24, exact in the
    fp32 accumulators in any order, and every patch element next to the zero slots of the last k16 step (k = 27 .. 31,
    147 .. 159) is non-zero.  The output is the fp64 convolution rounded once to the output format: exact on engine 4
    (integers below 2^22 fit the split planes), fp16 rounding of the exact value on engine 2."""
    weight = (S.probe_weight(k) - 1) % 17 - 8
    P = probe_program(weight, engine, k)
    g = torch.Generator().manual_seed(31 + k)
    xs = [torch.randint(-8, 9, (1, 3, h, w), generator=g).float() for h, w in PROBE_SIZES]
    out, ohw = S.run_nan(rf, P, xs, engine)
    got = S.output_images(out, ohw, engine)
    for i, x in enumerate(xs):
        ref, _ = S.stem_ref(x.cuda(), weight.cuda(), None, k, S.STRIDE[k], (k - 1) // 2)
        assert float(ref.max()) < 2.0 ** 22
        if engine == 2:
            ref = ref.half().double()
        bad = (got[i] != ref).nonzero()
        assert not len(bad), ("stem %s engine %d image %d %s: %d elements differ, first (channel, y, x) = %s: got %r, exact %r" %
                              (KS[k], engine, i, PROBE_SIZES[i], len(bad), tuple(bad[0].tolist()[1:]), float(got[i][tuple(bad[0])]),
                               float(ref[tuple(bad[0])])))
