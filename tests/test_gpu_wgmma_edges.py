"""wgmma engine behaviour the per-engine convolution tests do not reach: the fused stem at layer level, the fp32-output
rounding contract, sixteen-image ragged batches, and the correlation kernels' arg-max keys (scores, exact ties, negative
maxima).  References are fp64 on the operands the kernels consume (tests/wgmma_ref.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import stem_ref as S
import wgmma_ref as R

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ stem (RF_OP_STEM7) on engines 2 and 4
STEM_SIZES = [[(1, 1)], [(1, 45)], [(38, 1)], [(17, 35), (3, 5), (9, 33)], [(480, 640)],
              [(5 + 9 * i, 7 + 13 * i) for i in range(16)]]


@pytest.mark.parametrize("sizes", STEM_SIZES, ids=["1x1", "1xW", "Hx1", "ragged_partial", "480x640", "sixteen"])
@pytest.mark.parametrize("engine", [2, 4])
def test_stem7_layer_vs_fp64(rf, engine, sizes):
    """7x7 / stride 2 / pad 3 + folded BN + ReLU of the fused stem against fp64 of its operands (fp16 / split input and
    weights): split-grade on engine 4, fp16 rounding on engine 2.  Sizes: single pixels and rows / columns, outputs that are
    not multiples of the 16 x 8 tile, the 480 x 640 pair size and a sixteen-image batch."""
    P, fc = S.stem_program(*S.stem_args(7, 7))
    g = torch.Generator().manual_seed(len(sizes) * 31 + sizes[0][1])
    xs = [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]
    out, ohw = S.run_nan(rf, P, xs, engine)
    worst = S.check_stem(fc, 7, xs, engine, out, ohw, "stem engine %d" % engine)
    print("stem engine %d %s: worst error / allowance %.3g" % (engine, sizes[:2], worst))


@pytest.mark.parametrize("engine", [2, 4])
def test_stem7_sixteen_images_equal_images_alone(rf, engine):
    P, _ = S.stem_program(*S.stem_args(8, 7))
    g = torch.Generator().manual_seed(3)
    sizes = STEM_SIZES[-1]
    xs = [torch.randn(1, 3, h, w, generator=g) for h, w in sizes]
    batch, ohw = S.run_nan(rf, P, xs, engine)
    batch = batch.clone()
    again, _ = S.run_nan(rf, P, xs, engine)
    assert torch.equal(batch.view(torch.int16), again.view(torch.int16))
    o = np.cumsum([0] + [h * w for h, w in ohw])
    for i in range(16):
        alone, _ = S.run_nan(rf, P, [xs[i]], engine)
        part = batch[:, o[i]:o[i + 1]] if engine == 4 else batch[o[i]:o[i + 1]]
        assert torch.equal(part.view(torch.int16), alone.view(torch.int16)), i
    with pytest.raises(rf._lib.RFError):
        P.run(rf.ops.Ragged(R.nhwc(xs + xs[:1]).cuda(), sizes + sizes[:1]), engine)


# ------------------------------------------------------------------ fp32 outputs: TF32 rounding after ReLU, none without
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("cout", [64, 128, 200])
@pytest.mark.parametrize("engine", [1, 3])
def test_fp32_output_rounding_contract(rf, engine, cout, relu):
    """Engines 1 and 3 (fp16 operands, fp32 output): with ReLU every output is TF32-representable (cvt.rna after the ReLU)
    and within TF32 rounding of fp64; without ReLU the output is plain fp32, within 2^-24 plus accumulation of fp64."""
    xs, w, bias, _ = R.conv_inputs(cout + engine, 64, cout, 3, [(13, 21), (4, 3), (1, 9)], False, 1)
    gots, refs, abss, r_out, c, atol, y = R.run_conv(rf, engine, xs, w, bias, None, 1, relu)
    assert r_out == (R.R_TF32 if relu else R.R_F32)
    worst = max(R.check(g, r, a, r_out, c, atol, "engine %d image %d" % (engine, i)) for i, (g, r, a) in enumerate(zip(gots, refs, abss)))
    tf = R.is_tf32(y.cpu())
    if relu:
        assert bool(tf.all()), "%d outputs are not TF32-rounded" % int((~tf).sum())
    else:
        assert float((~tf).float().mean()) > 0.9, "the output without ReLU is rounded"
    print("engine %d Cout %d relu %s: worst error / allowance %.3g" % (engine, cout, relu, worst))


# ------------------------------------------------------------------ sixteen-image ragged batches (RF_MAX_IMGS)
SIXTEEN = [(1, 128), (2, 64), (16, 8), (4, 32), (8, 16), (13, 21), (1, 1), (9, 7), (3, 40), (25, 2), (6, 6), (11, 17), (2, 3), (7, 30),
           (19, 5), (5, 12)]


def _slice(y, o, i):
    return y[:, o[i]:o[i + 1]] if y.dim() == 3 else y[o[i]:o[i + 1]]


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


@pytest.mark.parametrize("engine", [1, 2, 3, 4, 5])
def test_sixteen_image_batch_equals_images_alone(rf, engine):
    """A sixteen-image ragged batch (every tile width among the images): each image's output equals that image run alone,
    bit for bit; two identical calls give identical bits; a seventeenth image is refused."""
    cout = 136
    xs, w, bias, _ = R.conv_inputs(engine, 64, cout, 3, SIXTEEN, False, 1)
    gots, refs, abss, r_out, c, atol, y = R.run_conv(rf, engine, xs, w, bias, None, 1, True)
    for i, (g, r, a) in enumerate(zip(gots, refs, abss)):
        R.check(g, r, a, r_out, c, atol, "engine %d image %d of 16" % (engine, i))
    y2 = R.run_conv(rf, engine, xs, w, bias, None, 1, True)[-1]
    assert torch.equal(_bits(y), _bits(y2))
    o = np.cumsum([0] + [h * w for h, w in SIXTEEN])
    for i in range(16):
        alone = R.run_conv(rf, engine, [xs[i]], w, bias, None, 1, True)[-1]
        assert torch.equal(_bits(_slice(y, o, i)), _bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        R.run_conv(rf, engine, xs + xs[:1], w, bias, None, 1, True)


def test_dual_sixteen_image_batch_equals_images_alone(rf):
    from test_gpu_split import dual_check
    g = torch.Generator().manual_seed(16)
    x2s = [torch.randn(1, 128, 2 * h, 2 * w, generator=g) for h, w in SIXTEEN]
    x1s = [torch.randn(1, 64, h, w, generator=g) for h, w in SIXTEEN]
    w1, w2 = torch.randn(120, 64, generator=g) / 8, torch.randn(120, 128, generator=g) / 11
    bias = torch.randn(120, generator=g)
    worst, y = dual_check(rf, x1s, x2s, w1, w2, bias, 2, True)
    _, y2 = dual_check(rf, x1s, x2s, w1, w2, bias, 2, True)
    assert torch.equal(_bits(y), _bits(y2))
    o = np.cumsum([0] + [h * w for h, w in SIXTEEN])
    for i in range(16):
        _, alone = dual_check(rf, [x1s[i]], [x2s[i]], w1, w2, bias, 2, True)
        assert torch.equal(_bits(_slice(y, o, i)), _bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        dual_check(rf, x1s + x1s[:1], x2s + x2s[:1], w1, w2, bias, 2, True)


# ------------------------------------------------------------------ correlation: arg-max keys of every precision
def corr_call(rf, A, B, mode, planes=None):
    """Runs the mutual nearest-neighbour entry point (``mode`` = its precision, or "presplit") with a caller-owned workspace;
    returns (row keys, column keys, idx1, idx2) as numpy.  ``planes``: ((A_hi, A_lo), (B_hi, B_lo)) CUDA planes the pre-split
    form reads instead of the split of A and B."""
    lib, ptr = rf._lib.lib, rf._lib.ptr
    NA, Cc = A.shape
    NB = B.shape[0]
    cap = max(1, min(NA, NB))
    idx1 = torch.empty(cap, device="cuda", dtype=torch.int64)
    idx2 = torch.empty(cap, device="cuda", dtype=torch.int64)
    count = torch.zeros(1, device="cuda", dtype=torch.int32)
    if mode == "presplit":
        a, b = planes if planes is not None else (R.to_split(A).cuda(), R.to_split(B).cuda())
        wsz = lib.rf_corr_mutual_nn_presplit_workspace(NA, NB)
        ws = torch.empty(wsz, device="cuda", dtype=torch.uint8)
        rf._lib.check(lib.rf_corr_mutual_nn_presplit(ptr(a[0]), ptr(a[1]), NA, ptr(b[0]), ptr(b[1]), NB, Cc, ptr(idx1), ptr(idx2), ptr(count),
                                                     ptr(ws), wsz, rf._lib.stream()))
    else:
        wsz = lib.rf_corr_mutual_nn_workspace(NA, NB, Cc, mode)
        ws = torch.full((wsz,), 0xAB, device="cuda", dtype=torch.uint8)      # the call must zero the keys itself
        a, b = A.cuda(), B.cuda()
        rf._lib.check(lib.rf_corr_mutual_nn(ptr(a), NA, ptr(b), NB, Cc, ptr(idx1), ptr(idx2), ptr(count), ptr(ws), wsz,
                                            mode, rf._lib.stream()))
    torch.cuda.synchronize()
    keys = ws[:8 * (NA + NB)].view(torch.int64).cpu().numpy().view(np.uint64)
    n = int(count.item())
    return keys[:NA], keys[NA:], idx1[:n].cpu().numpy(), idx2[:n].cpu().numpy()


def check_keys(keys, S, absS, c, what):
    """Keys of one side (one per row of S): score within the allowance of the fp64 score at the decoded index, the index the
    fp64 arg-max wherever the top-2 gap exceeds twice the row's allowance.  Returns (scores, indices, worst ratio)."""
    score, idx = R.decode_key(keys)
    assert (idx >= 0).all() and (idx < S.shape[1]).all(), (what, "missing or out-of-range key")
    rows = np.arange(S.shape[0])
    s64, a64 = S[rows, idx], absS[rows, idx]
    tol = R.R_F32 * np.abs(s64) + c * a64
    err = np.abs(score.astype(np.float64) - s64)
    assert (err <= tol).all(), (what, "score", int(np.argmax(err - tol)), float(np.max(err / tol)))
    allow = 2 * (R.R_F32 * np.abs(S).max(1) + c * absS.max(1))
    top = np.sort(S, axis=1)
    best = S.argmax(1)
    clear = (top[:, -1] - top[:, -2] > allow) if S.shape[1] > 1 else np.ones(S.shape[0], bool)
    assert (idx[clear] == best[clear]).all(), (what, "arg-max", np.nonzero(idx[clear] != best[clear])[0][:5])
    assert (s64 >= top[:, -1] - allow).all(), (what, "picked score below the maximum")
    return score, idx, float((err / tol).max())


def corr_data(case):
    rs = np.random.RandomState(5)
    if case == "ties":
        NA, NB, Cc = 400, 300, 64
        A, B = rs.randn(NA, Cc), rs.randn(NB, Cc)
    elif case == "negative":
        NA, NB, Cc = 200, 150, 64
        A, B = rs.randn(NA, Cc), rs.randn(NB, Cc)
        A[:, 0] = -(np.abs(A[:, 0]) + 6)              # every score < 0: negative maxima on both sides
        B[:, 0] = np.abs(B[:, 0]) + 6
    elif case in ("row1", "col1"):                      # one feature vector on one side: a single-row / single-column tile
        NA, NB, Cc = (1, 333, 192) if case == "row1" else (333, 1, 192)
        A, B = np.abs(rs.randn(NA, Cc)), np.abs(rs.randn(NB, Cc))
    else:
        NA, NB, Cc = 333, 270, int(case[1:])
        A, B = np.abs(rs.randn(NA, Cc)), np.abs(rs.randn(NB, Cc))
        B[: NB // 2] = A[rs.permutation(NA)[: NB // 2]] + 0.1 * np.abs(rs.randn(NB // 2, Cc))
    A = (A / np.linalg.norm(A, axis=1, keepdims=True)).astype(np.float32)
    B = (B / np.linalg.norm(B, axis=1, keepdims=True)).astype(np.float32)
    if case == "ties":
        v, u = A[7].copy(), B[5].copy()
        A[135] = A[300] = v                             # equal rows in three row tiles
        B[200] = v                                      # column 200: best rows 7, 135, 300 (equal scores): 7 must win
        B[130] = B[260] = u                             # equal columns in three column tiles, in-tile positions 5, 2, 4
        A[50] = u                                       # row 50: best columns 5, 130, 260 (equal scores): 5 must win
    return torch.from_numpy(A), torch.from_numpy(B)


@pytest.mark.parametrize("case", ["ties", "negative", "c192", "c448", "c1024", "row1", "col1"])
@pytest.mark.parametrize("mode", [0, 1, 2, "presplit"])
def test_corr_argmax_keys_vs_fp64(rf, mode, case):
    """The correlation's per-row / per-column arg-max keys (f2ord(score) << 32 | ~index) read from the workspace: scores within
    the fp32 (precision 0: gamma_C = C u / (1 - C u), the bound of a C-term fp32 FMA chain), 3xTF32 (precision 1) or split
    (precision 2, pre-split planes) allowance of fp64 scores of the consumed operands, indices the fp64 arg-max wherever the
    gap allows, exact ties to the smallest index across row and column tiles, the two keys of a mutual pair with bit-identical
    scores, and the compacted pair list == the mutual pairs of the keys.  Sizes leave partial row and column tiles, down to a
    single row (row1) or a single column (col1); C = 64 / 192 / 448 give 1 to 14 K blocks, C = 1024 is the pipeline's
    feature depth (the 3xTF32 allowance scales with the number of truncating accumulations beyond C = 448: acc_tf32x3)."""
    A, B = corr_data(case)
    split = mode in (2, "presplit")
    Aq = R.from_split(R.to_split(A)) if split else A.double()
    Bq = R.from_split(R.to_split(B)) if split else B.double()
    S = (Aq.cuda() @ Bq.cuda().T).cpu().numpy()
    absS = (Aq.abs().cuda() @ Bq.abs().cuda().T).cpu().numpy()
    cu = A.shape[1] * 2.0 ** -24
    c = R.ACC["split"] if split else R.acc_tf32x3(A.shape[1]) if mode == 1 else cu / (1 - cu)
    rowk, colk, i1, i2 = corr_call(rf, A, B, mode)
    csc, cidx, cw = check_keys(colk, S.T, absS.T, c, "columns")
    rsc, ridx, rw = check_keys(rowk, S, absS, c, "rows")
    worst = max(cw, rw)
    mutual = cidx[ridx] == np.arange(len(ridx))
    assert np.array_equal(rsc[mutual].view(np.uint32), csc[ridx[mutual]].view(np.uint32)), "mutual pair scores differ"
    keep = mutual & (rsc.astype(np.float64) ** 2 > 0)
    assert np.array_equal(i1, np.nonzero(keep)[0]) and np.array_equal(i2, ridx[keep])
    if case == "ties":
        assert cidx[200] == 7, cidx[200]
        assert ridx[50] == 5, ridx[50]
        assert ridx[7] == ridx[135] == ridx[300] and rsc[7] == rsc[135] == rsc[300]
        assert csc[5] == csc[130] == csc[260] and cidx[5] == cidx[130] == cidx[260]
    if case == "negative":
        assert (csc < 0).all() and (rsc < 0).all()
    print("correlation %s %s: worst score error / allowance %.3g, %d pairs" % (mode, case, worst, len(i1)))
