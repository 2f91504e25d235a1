"""Exact-operand fp64 references for the wgmma engine (helper of the tensor-core tests, not a test module).

Every reference is computed on the operands the kernel actually consumes, in fp64, so that the only differences left are the
kernel's own: the output rounding and the tensor core's fp32 accumulation (plus, for the split kinds, the omitted lo * lo
term).  The check is element-wise,

    |got - ref| <= r_out * |ref| + c * absref + atol,

with absref = the same operation on |operands| (+ |bias| + |residual|).  r_out is the output format's rounding, c the
kind's accumulation allowance, atol the output format's subnormal floor.  c is at least 30x below 2^-11 for every kind, so a
kernel that lost the lo planes of a split operand (11-bit instead of 22-bit arithmetic) fails.

Operands as consumed:
  TF32 (engine 1): fp32 values that are TF32-representable (low 13 mantissa bits zero), so that the MMA products are exact;
  3xTF32 (correlation precision 1): the fp32 values (hi + lo, the omitted lo * lo and the TF32 reading of lo in the allowance);
  fp16 (engines 2, 3): the fp16 values;
  split (engines 4, 5, the stem on engine 4, correlation precision 2): hi + lo * 2^-11 of the fp16 planes.

The fp64 references of the SIMT layer kernels (max-pool, blur, pool + blur, im2col, L2 normalisation, the flow head's
softmax epilogue) live here too; tests/test_gpu_layer_ops.py holds their bounds.
"""
import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

# output rounding, relative
R_F16 = 2.0 ** -11          # fp16 round to nearest
R_TF32 = 2.0 ** -11         # fp32 rounded to nearest TF32 (cvt.rna) after ReLU
R_SPLIT = 2.0 ** -22        # hi = fp16(v), lo = fp16((v - hi) * 2^11)
R_F32 = 2.0 ** -24          # plain fp32
# absolute floors of the output formats (fp16 subnormal half-step; split: the lo plane's subnormal half-step * 2^-11)
ATOL = {"f16": 2.0 ** -25, "split": 2.0 ** -35, "f32": 0.0, "tf32": 0.0}
# accumulation allowance per operand kind, relative to absref: the tensor core's fp32 accumulation (which truncates, so on
# all-positive sums the error grows with K) and, for the split kinds, the omitted lo * lo term (<= 2^-22).  Set from the worst
# errors measured on an H100 80GB HBM3 (700 W power limit) over these tests: TF32 / fp16 convolutions ~1.8e-6, split
# convolutions ~0.6e-6, split correlation 2.7e-6 and 3xTF32 correlation 1.1e-5 of absref at C = 448 (one accumulator for all
# three products: 168 truncating accumulations).  Margins: 2x (TF32 / fp16), 2.8x (split), 1.4x (3xTF32).  Every value is
# >= 30x below 2^-11 so that 11-bit arithmetic cannot pass.
ACC = {"tf32": 2.0 ** -18, "f16": 2.0 ** -18, "split": 2.0 ** -17, "tf32x3": 2.0 ** -16}
ELEVEN_BIT = 2.0 ** -11
assert all(c * 30 <= ELEVEN_BIT for c in ACC.values())


def acc_tf32x3(C):
    """The 3xTF32 correlation's allowance at C channels.  Each truncating accumulation of a non-negative term loses less than
    one ulp of the partial sum, so the accumulation error of the all-positive scores grows with their number, 3 C / 8; the
    allowance measured at C = 448 is scaled by it beyond 448.  At the pipeline's C = 1024 the errors reach 1.004x the
    unscaled value (post-ReLU features on an H100 80GB HBM3, 700 W power limit)."""
    return ACC["tf32x3"] * max(1.0, C / 448.0)


# engine -> (operand kind, output format)
ENGINES = {1: ("tf32", "f32"), 2: ("f16", "f16"), 3: ("f16", "f32"), 4: ("split", "split"), 5: ("split", "f32")}
BK = {"tf32": 32, "f16": 64, "split": 64}


def stages(kind, bn):
    """Ring depth of wg_kernel<KIND, BN, MODE_CONV> (WgCfg in csrc/gemm_tc.cu): shared-memory budget / stage bytes, at most 6."""
    npl = 2 if kind in ("split", "tf32x3") else 1
    stage = npl * 128 * 128 + npl * bn * 128
    budget = 200 * 1024 if npl * bn >= 256 else 100 * 1024
    return min(6, budget // stage)


def bn_of(cout):
    return 128 if cout > 64 else 64


# ------------------------------------------------------------------ operand rounding
def tf32_trunc(t):
    """fp32 -> fp32 with the low 13 mantissa bits cleared (what a TF32 MMA reads)."""
    t = t.float().contiguous()
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def is_tf32(t):
    """True where an fp32 value is exactly representable in TF32."""
    return (t.float().contiguous().view(torch.int32) & 0x1FFF) == 0


def to_split(x):
    """fp32 -> [2, ...] fp16 planes (hi, lo * 2^11), saturating like the kernels."""
    x = x.float().clamp(-65504.0, 65504.0)
    hi = x.to(torch.float16)
    lo = ((x - hi.float()) * 2048.0).to(torch.float16)
    return torch.stack([hi, lo])


def from_split(s):
    """[2, ...] fp16 planes -> fp64 values they stand for (exact)."""
    return s[0].double() + s[1].double() / 2048.0


def tf32_round(t):
    """fp32 -> nearest TF32 value (ties to even), as FoldedConv packs the weights (model.py).  The kernels' round_out is
    tf32_rna."""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF).view(torch.float32)


def tf32_rna(t):
    """fp32 -> nearest TF32 value, ties away from zero: cvt.rna.tf32.f32, what round_tf32 (csrc/common.cuh) stores wherever a
    kernel's round_out is set (ReLU'd convolution outputs, engine 1's blur / pool + blur / im2col outputs)."""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def operand(x, kind):
    """(tensor the kernel reads, fp64 value it stands for) of an fp32 tensor.  TF32 operands are given to the kernel already
    TF32-representable, as the library's own producers store them (weights rounded once, activations rounded after ReLU):
    their products are exact whatever the MMA does with the low 13 bits.  "f32": the fp32 values as they are (SIMT kernels)."""
    if kind == "f32":
        x = x.float()
        return x, x.double()
    if kind == "tf32":
        t = tf32_round(x)
        return t, t.double()
    if kind == "f16":
        h = x.half()
        return h, h.double()
    s = to_split(x)
    return s, from_split(s)


# ------------------------------------------------------------------ references and the bound
def conv_ref(x, w, bias=None, residual=None, stride=1, pad=0, relu=False):
    """fp64 NCHW convolution + bias + residual (+ ReLU) and its absref (the same on absolute values)."""
    x, w = x.double(), w.double()
    ref = F.conv2d(x, w, None, stride=stride, padding=pad)
    absref = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=pad)
    if bias is not None:
        ref = ref + bias.double().view(1, -1, 1, 1)
        absref = absref + bias.double().abs().view(1, -1, 1, 1)
    if residual is not None:
        ref = ref + residual.double()
        absref = absref + residual.double().abs()
    if relu:
        ref = ref.clamp_min(0.0)
    return ref, absref


def bound(ref, absref, r_out, c, atol=0.0):
    return r_out * ref.abs() + c * absref + atol


def check(got, ref, absref, r_out, c, atol=0.0, what=""):
    """Element-wise |got - ref| <= r_out |ref| + c absref + atol.  NaN (an element the kernel never wrote) fails.  Returns the
    worst error / allowance ratio."""
    got = got.double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    b = bound(ref, absref, r_out, c, atol)
    ok = err <= b
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s: %d of %d elements outside |got - ref| <= %.3g |ref| + %.3g absref + %.3g; first at %s: got %r ref %r "
                             "absref %r" % (what, bad.shape[0], ok.numel(), r_out, c, atol, i, got[i].item(), ref[i].item(), absref[i].item()))
    return float((err / b.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ------------------------------------------------------------------ the layer kernels between the convolutions (elementwise.cu)
U = 2.0 ** -24                 # fp32 unit roundoff
EPS_L2 = float(np.float32(1e-12))


def gamma(n):
    """Bound on the relative error of an n-term fp32 sum or product chain: n u / (1 - n u)."""
    return n * U / (1 - n * U)


def _blur64(x, stride):
    c = x.shape[1]
    a = torch.tensor([1.0, 2.0, 1.0], dtype=torch.float64, device=x.device)
    f = (a[:, None] * a[None, :] / 16.0).expand(c, 1, 3, 3).contiguous()
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), f, stride=stride, groups=c)


def blur_ref(x, stride):
    """model/downsample.py: ReflectionPad2d(1) + depthwise [1 2 1]^2 / 16 at ``stride`` of (N, C, H, W), in fp64, and the same
    filter on |x|."""
    x = x.double()
    return _blur64(x, stride), _blur64(x.abs(), stride)


def poolblur_ref(x):
    """MaxPool2d(2, stride 1), then the stride-2 blur reflecting on the (H - 1) x (W - 1) pooled map; absref on |pooled|."""
    p = F.max_pool2d(x.double(), 2, 1)
    return _blur64(p, 2), _blur64(p.abs(), 2)


def maxpool_ref(x, k, stride, pad):
    """The maximum over the in-image part of each window (the padding never wins), fp64."""
    return F.max_pool2d(x.double(), k, stride, pad)


def im2col_ref(x, k, stride, pad, kpad):
    """[Ho * Wo, kpad] rows of a (1, C, H, W) image: the k x k patch of each output pixel in (r, s, c) order, zero outside the
    image and in columns k * k * C .. kpad - 1.  Same dtype as x: values are copied, never computed."""
    _, c, h, w = x.shape
    ho, wo = out_hw(h, w, k, stride, pad)
    xp = F.pad(x, (pad, pad, pad, pad))
    taps = [xp[0, :, r:r + stride * (ho - 1) + 1:stride, s:s + stride * (wo - 1) + 1:stride] for r in range(k) for s in range(k)]
    rows = torch.stack(taps, 0).permute(2, 3, 0, 1).reshape(ho * wo, k * k * c)      # (tap, C, Ho, Wo) -> (Ho, Wo, tap, C)
    return F.pad(rows, (0, kpad - k * k * c))


def l2norm_ref(x, mask=None):
    """x / max(||x||_2, fp32(1e-12)) per row of [P, C], in fp64 (F.normalize with the kernels' fp32 eps); rows whose mask
    is 0 are zero."""
    x = x.double()
    y = x / x.norm(dim=1, keepdim=True).clamp_min(EPS_L2)
    if mask is not None:
        y = torch.where(mask.view(-1, 1).to(y.device) != 0, y, torch.zeros_like(y))
    return y


def softmax_flow_ref(logits, k):
    """NetFlowCoarse's epilogue (model/model.py; MO.net_flow_coarse after its trunk) on (N, k*k, h, w) logits, in fp64:
    p = softmax over the k*k channels, flow = (sum p gx / w * 2, sum p gy / h * 2) with channel i*k + j at the offset
    (gx, gy) = (j - k//2, i - k//2).  Returns (flow (N, 2, h, w), the same sums of p |g|)."""
    lg = logits.double()
    _, kk, h, w = lg.shape
    p = torch.softmax(lg, 1)
    q = torch.arange(kk, device=lg.device)
    gx = (q % k - k // 2).double().view(1, -1, 1, 1)
    gy = (q // k - k // 2).double().view(1, -1, 1, 1)
    flow = torch.cat(((p * gx).sum(1, keepdim=True) / w * 2, (p * gy).sum(1, keepdim=True) / h * 2), 1)
    absf = torch.cat(((p * gx.abs()).sum(1, keepdim=True) / w * 2, (p * gy.abs()).sum(1, keepdim=True) / h * 2), 1)
    return flow, absf


# ------------------------------------------------------------------ tile widths (mirror of pick_tw in csrc/gemm_tc.cu)
TILE_WIDTHS = (8, 16, 32, 64, 128)


def pick_tw(Ho, Wo):
    best, best_area = 16, -1
    for tw in (16, 32, 8, 64, 128):
        th = 128 // tw
        area = ((Wo + tw - 1) // tw) * ((Ho + th - 1) // th)
        if best_area < 0 or area < best_area:
            best, best_area = tw, area
    return best


def out_hw(h, w, k, stride, pad):
    return (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1


# tile widths 8 .. 128 of a 3x3 / pad 1 convolution at stride 1 (first list) and at stride 2 (second list); the second list's
# last image is the 256-pixel TMA box (tw = 128 at stride 2: box[1] = tw * stride)
TW_SWEEP_S1 = [(8, 16), (16, 8), (4, 32), (2, 64), (1, 128)]
TW_SWEEP_S2 = [(16, 32), (32, 16), (8, 64), (4, 128), (2, 256)]


def ring_cases(kind, couts=(56, 120)):
    """1x1 layers (cin, cout, 1, sizes) whose K-block count KI = Cin / BK runs from 1 to 2 * STAGES + 1 of the instance, for
    each Cout (the defaults: BN 64 and BN 128, both with a partial N tile)."""
    return [(BK[kind] * n, cout, 1, [(5, 9)]) for cout in couts for n in range(1, 2 * stages(kind, bn_of(cout)) + 2)]


def conv_inputs(seed, cin, cout, k, sizes, res, stride):
    """Seeded fp32 CPU inputs (1, Cin, H, W) per size, weights / sqrt(fan-in), bias, and residuals (or None)."""
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(1, cin, h, w, generator=g) for h, w in sizes]
    w = torch.randn(cout, cin, k, k, generator=g) / float(np.sqrt(cin * k * k))
    bias = torch.randn(cout, generator=g)
    rs = [torch.randn(1, cout, *out_hw(h, ww, k, stride, k // 2), generator=g) for h, ww in sizes] if res else None
    return xs, w, bias, rs


def widths_covered(cases, strides):
    """{stride: set of tile widths} that the (k, sizes) cases run at the given strides (pad = k // 2)."""
    cov = {s: set() for s in strides}
    for k, sizes in cases:
        for s in strides:
            for h, w in sizes:
                cov[s].add(pick_tw(*out_hw(h, w, k, s, k // 2)))
    return cov


# ------------------------------------------------------------------ arg-max keys: (f2ord(score) << 32) | ~index
def f2ord(f):
    u = np.asarray(f, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000).astype(np.uint64)


def ord2f(o):
    o = np.asarray(o, dtype=np.uint64)
    u = np.where(o & 0x80000000, o & 0x7FFFFFFF, ~o & 0xFFFFFFFF).astype(np.uint32)
    return u.view(np.float32)


def encode_key(score, index):
    return (f2ord(score) << np.uint64(32)) | (~np.asarray(index, dtype=np.uint64) & np.uint64(0xFFFFFFFF))


def decode_key(key):
    """uint64 keys -> (fp32 scores, int64 indices); key 0 (never written) decodes to index -1."""
    key = np.asarray(key).view(np.uint64)
    score = ord2f(key >> np.uint64(32))
    index = (~key & np.uint64(0xFFFFFFFF)).astype(np.int64)
    return score, np.where(key == 0, -1, index)


# ------------------------------------------------------------------ direct library calls with caller-owned outputs
def nan_output(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def conv_call(rf, x, hw, cin, w_packed, w_tc, bias, residual, cout, k, stride, pad, relu, engine, y):
    """rf_conv2d_nhwc into ``y`` (pre-filled by the caller); ``x`` / ``residual`` / ``y`` device tensors in the engine's layout."""
    lib, ptr = rf._lib.lib, rf._lib.ptr
    chw = (C.c_int * (2 * len(hw)))(*[v for p in hw for v in p])
    rf._lib.check(lib.rf_conv2d_nhwc(ptr(x), len(hw), chw, cin, ptr(w_packed), ptr(w_tc), ptr(bias), ptr(residual), cout, k, k, stride, pad,
                                     int(relu), int(engine), ptr(y), rf._lib.stream()))
    return y


def nhwc(xs):
    """list of (1, C, H, W) CPU tensors -> [sum HW, C] (same dtype)."""
    return torch.cat([x[0].permute(1, 2, 0).reshape(-1, x.shape[1]) for x in xs], 0).contiguous()


def images(data, hw):
    """[sum HW, C] -> list of (1, C, H, W) CPU views."""
    out, o = [], 0
    for h, w in hw:
        out.append(data[o:o + h * w].reshape(1, h, w, -1).permute(0, 3, 1, 2))
        o += h * w
    return out


def run_conv(rf, engine, xs, w, bias, res, stride, relu):
    """One convolution on ``engine`` with caller-owned NaN-filled output.  xs / res: lists of fp32 (1, C, H, W) CPU tensors,
    w fp32 (Cout, Cin, k, k), bias fp32 or None.  Returns (fp64 outputs, fp64 refs, absrefs: lists of (1, C, H, W) device
    tensors, r_out, c, atol, the raw output tensor)."""
    kind, out = ENGINES[engine]
    cout, cin, k, _ = w.shape
    pad = k // 2
    hw = [(x.shape[2], x.shape[3]) for x in xs]
    ohw = [out_hw(h, ww, k, stride, pad) for h, ww in hw]
    P = sum(h * ww for h, ww in ohw)
    xd, xq = operand(nhwc(xs), kind)
    wt = w.permute(0, 2, 3, 1).reshape(cout, k * k * cin).contiguous()
    wd, wq = operand(wt, kind)
    wq = wq.view(cout, k, k, cin).permute(0, 3, 1, 2)
    rd, rq = (None, None)
    if res is not None:
        rd, rq = operand(nhwc(res), kind)
    xd = xd.contiguous().cuda()
    w_packed = w.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().cuda() if engine == 1 else None
    if out == "split":
        y = nan_output((2, P, cout), torch.float16)
    else:
        y = nan_output((P, cout), torch.float16 if out == "f16" else torch.float32)
    conv_call(rf, xd, hw, cin, w_packed, wd.contiguous().cuda(), bias.cuda() if bias is not None else None,
              rd.contiguous().cuda() if rd is not None else None, cout, k, stride, pad, relu, engine, y)
    torch.cuda.synchronize()
    # the fp64 references run on the device too (fp64 is exact enough; the CPU would take minutes on the larger cases)
    got = from_split(y) if out == "split" else y.double()
    gots = images(got, ohw)
    xqs = images(xq.cuda(), hw)
    rqs = images(rq.cuda(), ohw) if rq is not None else [None] * len(xs)
    wq, bq = wq.cuda(), bias.cuda() if bias is not None else None
    refs, abss = [], []
    for xi, ri in zip(xqs, rqs):
        r, a = conv_ref(xi, wq, bq, ri, stride, pad, relu)
        refs.append(r)
        abss.append(a)
    r_out = {"f16": R_F16, "split": R_SPLIT, "f32": (R_TF32 if relu and engine in (1, 3) else R_F32)}[out]
    return gots, refs, abss, r_out, ACC[kind], ATOL[out], y


def check_conv(rf, engine, xs, w, bias, res, stride, relu, what=""):
    """run_conv + the element-wise check of every image; prints and returns the worst ratio."""
    gots, refs, abss, r_out, c, atol, y = run_conv(rf, engine, xs, w, bias, res, stride, relu)
    worst = 0.0
    for i, (g, r, a) in enumerate(zip(gots, refs, abss)):
        worst = max(worst, check(g, r, a, r_out, c, atol, "%s image %d" % (what, i)))
    print("engine %d %s: worst error / allowance %.3g" % (engine, what, worst))
    return worst, y
