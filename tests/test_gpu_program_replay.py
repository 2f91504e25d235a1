"""Every layer program of the product replayed layer by layer on the image sets the pipeline itself runs, each layer against an
fp64 reference of the operands it read.

The image sets are recorded, not made up: a spy on ``LayerProgram.run`` records the ragged (H, W) list, the engine and the input
of every program call while one bench config-2 pair (480 x 640, variant A, 7 scales, scaleR 2, fine flow with match21), one
config-5 pair (376 x 1241, coarseSize 800, 3 scales, scaleR 1.2, two-level fine flow) and segNet (480 x 640 and 376 x 1241) run.

Each recorded call is then replayed on the program's own compiled entry (its layer list, activation buffers and sizes): prefix
n of the layer list runs through ``rf_run_layers`` for n = 1 .. len(ops), and the output of layer n - 1 is decoded from its slot
right away (``produced``).  Every layer's reference is computed from ``produced`` of the tensors it reads, never from the slots
at read time, so a slot the allocator hands out again too early fails at the layer that reads it.  The last prefix must equal
``LayerProgram.run`` bit for bit.  The stem with its fused max-pool (RF_LAYER_STEM_POOL) is one step.

Bounds (tests/wgmma_ref.py): convolutions |got - ref| <= r_out |ref| + ACC[kind] absref + ATOL[out] with the weights the kernel
reads (split planes, fp16, TF32 or fp32) and the exact-operand fp64 reference; max-pool exact; blur and pool + blur within
gamma_9; im2col bit for bit.  Under TF32, every operand a TF32 layer reads must be TF32-representable (the MMA truncates).
segNet's decoder (adaptive pooling at C = 2048, the PPM convolutions, the concat, conv_last) and the vote are checked at the
network's own sizes on the encoder's own conv5.
"""
import ctypes as C

import PIL.Image as Image
import pytest
import torch
import torch.nn.functional as F

import wgmma_ref as R
from oracle import synth
from stem_ref import packed_weights


ENGINE_NAMES = {4: "f16x3", 2: "f16", 1: "tf32"}
CORR_PRECISION = {4: 2, 2: 2, 1: 1}                 # bench.py: corr_precision per engine
ENGINES = (4, 2, 1)
FINE = ("features", "flow head", "matchability head")
PROGRAMS = [(e, p) for e in ENGINES for p in ("trunk",) + FINE] + [(4, "segnet encoder"), (4, "segnet conv_last")]


# ------------------------------------------------------------------ recording
def _models(rf, config):
    rsd = synth.resnet50_conv4_state(0)
    net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7),
           "netFlowCoarse": rf.model.NetFlowCoarse(7), "netMatch": rf.model.NetMatchability(7)}
    net["netFeatCoarse"].load_state_dict(synth.feature_extractor_state(0))
    net["netFlowCoarse"].load_state_dict(synth.net_flow_coarse_state(1))
    net["netMatch"].load_state_dict(synth.net_matchability_state(2))
    for m in net.values():
        m.cuda()
        m.eval()
    if config == 5:
        c = rf.CoarseAlignA(3, 1000, 0.05, "Homography", 800, 2, False, 1.2, True, False, resnet_state_dict=rsd, verbose=False)
    else:
        c = rf.CoarseAlignA(7, 1000, 0.05, "Homography", 480, 2, False, 2, True, False, resnet_state_dict=rsd, verbose=False)
    c.device_preproc = True
    return c, net


def _names(c, net):
    """program object id -> name, for the programs these models own."""
    names = {}
    for P in (c.net.program, c.net._program_f16, c.net._program_split):
        if P is not None:
            names[id(P)] = "trunk"
    for key, name in (("netFeatCoarse", "features"), ("netFlowCoarse", "flow head"), ("netMatch", "matchability head")):
        for P in getattr(net[key], "_fold", {}).values():
            names[id(P)] = name
    return names


@pytest.fixture(scope="module")
def recorded(rf):
    """{(engine, program name): [dict(P, hw, engine, x, what)]}: every distinct (program, image set, engine) the pipeline ran."""
    from ransac_flow_b200.program import LayerProgram
    from ransac_flow_b200.segnet import SegNet
    calls, real = [], LayerProgram.run

    def spy(self, x, engine):
        if not any(c["P"] is self and c["hw"] == list(x.hw) and c["engine"] == int(engine) for c in calls):
            calls.append(dict(P=self, hw=list(x.hw), engine=int(engine), x=x.data.clone()))
        return real(self, x, engine)

    names, keep = {}, []
    LayerProgram.run = spy
    try:
        for engine in ENGINES:
            rf.model.set_engine(ENGINE_NAMES[engine])
            rf.outil.corr_precision = CORR_PRECISION[engine]
            for config in (2, 5):
                c, net = _models(rf, config)
                h, w = (376, 1241) if config == 5 else (480, 640)
                s, t, _ = synth.make_pair(config, h, w)
                torch.manual_seed(1000)
                if config == 5:
                    out = rf.pipeline.align_pair_kitti(c, net, Image.fromarray(s), Image.fromarray(t), maxH=1)
                    assert len(out["H"]) == 1, "config 5: no hypothesis, the fine flow never ran"
                else:
                    out = rf.pipeline.align_pair_single(c, net, torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), with_match21=True)
                    assert len(out["H"]) == 1, "config 2: RANSAC found no homography, the fine flow never ran"
                torch.cuda.synchronize()
                names.update(_names(c, net))
                keep.append((c, net))
        sds = (synth.segnet_encoder_state(0), synth.segnet_decoder_state(0))
        seg = SegNet(None, None, 2, False, state_dicts=sds)
        for seed, (h, w) in enumerate(((480, 640), (376, 1241))):
            seg.run(Image.fromarray(synth.segnet_image(seed, h, w)))
        torch.cuda.synchronize()
        names[id(seg.encoder)], names[id(seg.head)] = "segnet encoder", "segnet conv_last"
        keep.append(seg)
    finally:
        LayerProgram.run = real
        rf.model.set_engine("fp32")
        rf.outil.corr_precision = 0
    out = {}
    for c in calls:
        c["what"] = names[id(c["P"])]
        out.setdefault((c["engine"], c["what"]), []).append(c)
    out["_keep"] = keep
    return out


# ------------------------------------------------------------------ fp64 references in NHWC ((H, W, C) per image)
def conv64(x, w, stride=1, pad=0, dil=1):
    """(H, W, Cin) * (Cout, k, k, Cin) -> (Ho, Wo, Cout) in the dtype of the operands, as k * k GEMMs over shifted views."""
    H, W, cin = x.shape
    cout, k = w.shape[0], w.shape[1]
    ho, wo = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1, (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    xp = F.pad(x, (0, 0, pad, pad, pad, pad))
    out = x.new_zeros(ho * wo, cout)
    for r in range(k):
        for s in range(k):
            tap = xp[r * dil:r * dil + stride * (ho - 1) + 1:stride, s * dil:s * dil + stride * (wo - 1) + 1:stride]
            out.addmm_(tap.reshape(-1, cin), w[:, r, s, :].t())
    return out.view(ho, wo, cout)


def absconv(x, w, stride=1, pad=0, dil=1):
    """An upper bound on conv(|x|, |w|) from one TF32 GEMM per tap: each operand is read with a relative error below 2^-10 and
    the positive fp32 sums of K terms are off by at most gamma_2K, so the fp32 result times (1 + 2^-8) / (1 - gamma_2K) is at
    least the exact sum.  absref only scales the allowance, so it need not be exact."""
    K = w.shape[1] * w.shape[2] * w.shape[3]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        a = conv64(x.abs().float(), w.abs().float(), stride, pad, dil).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return a * ((1 + 2.0 ** -8) / (1 - R.gamma(2 * K)))


def nchw(x):
    return x.permute(2, 0, 1)[None]


def nhwc(x):
    return x[0].permute(1, 2, 0)


def maxpool64(x, k, s, p):
    return nhwc(F.max_pool2d(nchw(x), k, s, p))


# ------------------------------------------------------------------ the program's layout
def layout(P, hw, engine):
    """(hws, formats) of every symbolic tensor: the sizes by _compile's rule and "split" / "f16" / "f32" by the engine and the
    layer flags."""
    from ransac_flow_b200 import program as pg
    hws = [list(hw)]
    for i, o in enumerate(P.ops):
        k, s, p, d = o[5], o[6], o[7], P.dil.get(i, 1)
        hws.append([((h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1) for h, w in hws[o[1]]])
    stem_in = P.ops[0][0] in (pg.RF_OP_IM2COL, pg.RF_OP_STEM7, pg.RF_OP_STEM3)
    fmts = []
    for t in range(len(P.chan)):
        fl = P.flags.get(t - 1, 0) if t else 0
        if engine == 1 or (t == 0 and stem_in):
            fmts.append("f32")
        elif engine == 4:
            fmts.append("f32" if fl & pg.RF_LAYER_OUT_F32 else "split")
        else:
            fmts.append("f32" if fl else "f16")
    return hws, fmts


def raw_view(buf, fmt, P_, C_):
    if fmt == "split":
        return buf[:P_ * C_ * 4].view(torch.float16).view(2, P_, C_)
    if fmt == "f16":
        return buf[:P_ * C_ * 2].view(torch.float16).view(P_, C_)
    return buf[:P_ * C_ * 4].view(torch.float32).view(P_, C_)


def decode(raw, fmt, hw):
    """Raw slot contents -> list of fp64 (H, W, C) images (exact)."""
    v = R.from_split(raw) if fmt == "split" else raw.double()
    out, o = [], 0
    for h, w in hw:
        out.append(v[o:o + h * w].view(h, w, -1))
        o += h * w
    return out


# ------------------------------------------------------------------ per-op checks
def conv_rule(engine, flags, relu, cin, k, stride):
    """(operand kind, r_out, atol) of a conv layer: what rf_run_layers runs it as (csrc/runner.cu)."""
    from ransac_flow_b200 import program as pg
    if engine == 4:
        return ("split", R.R_F32, 0.0) if flags & pg.RF_LAYER_OUT_F32 else ("split", R.R_SPLIT, R.ATOL["split"])
    r32 = R.R_TF32 if relu else R.R_F32           # fp32 outputs of ReLU layers are rounded to TF32 (round_out)
    if engine == 2:
        if flags:
            return ("tf32" if flags & pg.RF_LAYER_TF32 else "f16"), r32, 0.0
        return "f16", R.R_F16, R.ATOL["f16"]
    tc = stride in (1, 2) and cin % 32 == 0 and k in (1, 3)       # rf_conv2d_tc_supported; other layers run the exact FMA engine
    return ("tf32" if tc else "fma"), r32, 0.0


def weights(fc, kind, k, cin):
    """(Cout, k, k, Cin) fp64 values of the weights the kernel reads."""
    if kind == "split":
        w = R.from_split(fc.w_split)
    elif kind == "f16":
        w = fc.w_f16.double()
    elif kind == "tf32":
        w = fc.w_tc.double()
    else:
        w = fc.w.double().t()
    return w.reshape(w.shape[0], k, k, cin)


class Replay:
    def __init__(self, rf, rec):
        from ransac_flow_b200 import program as pg
        self.rf, self.pg, self.rec = rf, pg, rec
        self.P, self.hw, self.engine, self.x = rec["P"], rec["hw"], rec["engine"], rec["x"]
        self.worst = {}

    def note(self, kind, ratio):
        self.worst[kind] = max(self.worst.get(kind, 0.0), ratio)

    def run(self):
        rf, pg, P, engine = self.rf, self.pg, self.P, self.engine
        lib = rf._lib
        out, _ = P.run(rf.ops.Ragged(self.x, self.hw), engine)
        key = (tuple(self.hw), str(self.x.device), engine if engine in (2, 4) else 0)      # LayerProgram.run's cache key
        c = P._compiled[key]
        full = c["bufs"][c["out_slot"]][:c["out_elems"]].clone()
        slots = (C.c_void_p * c["nslots"])()
        slots[0] = self.x.data_ptr()
        for i in range(1, c["nslots"]):
            slots[i] = c["bufs"][i].data_ptr()
        hws, fmts = layout(P, self.hw, engine)
        n_t = len(P.chan)
        last_use = [0] * n_t
        for i, o in enumerate(P.ops):
            for t in (o[1], o[2], P.dual[i][0] if i in P.dual else -1):
                if t >= 0:
                    last_use[t] = i
        x0 = self.x.view(2, -1, P.chan[0]) if fmts[0] == "split" else self.x
        produced = {0: decode(x0, fmts[0], self.hw)}
        tf32ok = {0: fmts[0] == "f32" and bool(R.is_tf32(self.x).all())}
        i, steps = 0, 0
        while i < len(P.ops):
            o = P.ops[i]
            fused = o[0] == pg.RF_OP_STEM7 and bool(c["layers"][i].flags & pg.RF_LAYER_STEM_POOL)
            j = i + 1 if fused else i
            lib.check(lib.lib.rf_run_layers(c["layers"], j + 1, slots, len(self.hw), c["chw"], engine, lib.stream()))
            torch.cuda.synchronize()
            steps += 1
            t = j + 1
            n_pix = sum(h * w for h, w in hws[t])
            raw = raw_view(c["bufs"][c["layers"][j].dst], fmts[t], n_pix, P.chan[t])
            got = decode(raw, fmts[t], hws[t])
            assert all(not bool(g.isnan().any()) for g in got), "%s op %d: NaN in the output" % (self.rec["what"], j)
            self.check(i, fused, got, raw, produced, tf32ok)
            produced[t] = [g.clone() for g in got]
            tf32ok[t] = fmts[t] == "f32" and bool(R.is_tf32(raw).all())
            for s in list(produced):
                if s > 0 and s < t and last_use[s] <= j:
                    del produced[s]
            i = j + 1
        assert torch.equal(c["bufs"][c["out_slot"]][:c["out_elems"]], full), "the last prefix differs from LayerProgram.run"
        return steps

    def check(self, i, fused, got, raw, produced, tf32ok):
        pg, P, engine = self.pg, self.P, self.engine
        o = P.ops[i]
        op, src, res, cin, cout, k, s, pad, relu, fc = o
        name = "%s engine %d %s op %d" % (self.rec["what"], engine, self.hw, i)
        if op in (pg.RF_OP_CONV, pg.RF_OP_CONV_DUAL):
            fl, d = P.flags.get(i, 0), P.dil.get(i, 1)
            kind, r_out, atol = conv_rule(engine, fl, relu, cin, k, s)
            if op == pg.RF_OP_CONV_DUAL:
                src2, cin2, s2 = P.dual[i]
                w = R.from_split(fc.w_split)
                w1, w2 = w[:, :cin].reshape(cout, 1, 1, cin), w[:, cin:].reshape(cout, 1, 1, cin2)
                label, K = "conv_dual", cin + cin2
            else:
                w = weights(fc, kind, k, cin)
                label, K = "conv%dx%d%s%s%s" % (k, k, "/2" if s == 2 else "", " dil%d" % d if d > 1 else "", " +res" if res >= 0 else ""), k * k * cin
                if kind != {4: "split", 2: "f16", 1: "tf32"}[engine]:
                    label += " " + kind          # engine 2's TF32 head layer, engine 1's layers on the exact FMA engine
            if kind == "tf32":
                assert tf32ok[src], "%s: a TF32 layer reads operands that are not TF32-representable (the MMA truncates them)" % name
            c_acc = R.gamma(K) if kind == "fma" else R.ACC[kind]
            bias = fc.bias.double() if fc.bias is not None else None
            worst = 0.0
            for m, xi in enumerate(produced[src]):
                if op == pg.RF_OP_CONV_DUAL:
                    x2 = produced[src2][m][::s2, ::s2]
                    ref = conv64(xi, w1) + conv64(x2, w2)
                    absref = absconv(xi, w1) + absconv(x2, w2)
                else:
                    ref, absref = conv64(xi, w, s, pad, d), absconv(xi, w, s, pad, d)
                if bias is not None:
                    ref, absref = ref + bias, absref + bias.abs()
                if res >= 0:
                    ref, absref = ref + produced[res][m], absref + produced[res][m].abs()
                if relu:
                    ref = ref.clamp_min(0.0)
                worst = max(worst, R.check(got[m], ref, absref, r_out, c_acc, atol, "%s image %d" % (name, m)))
            self.note(label, worst)
        elif op in (pg.RF_OP_STEM7, pg.RF_OP_STEM3):
            if op == pg.RF_OP_STEM3:
                kind, w, c_acc, r_out, atol, label = "f32", fc.w.double().t().reshape(64, k, k, 3), 2.0 ** -18, R.R_SPLIT, R.ATOL["split"], "stem3x3/2 fp32"
            else:
                kind = "split" if engine == 4 else "f16"
                w = packed_weights(fc, engine, k).permute(0, 2, 3, 1).cuda()
                c_acc, r_out, atol = R.ACC[kind], (R.R_SPLIT if engine == 4 else R.R_F16), R.ATOL[kind]
                label = "stem%dx%d" % (k, k) + ("+pool" if fused else "")
            worst = 0.0
            for m, xi in enumerate(produced[0]):
                xq = R.operand(xi.float(), kind)[1]
                ref = (conv64(xq, w, s, pad) + fc.bias.double()).clamp_min(0.0)
                absref = absconv(xq, w, s, pad) + fc.bias.double().abs()
                if fused:       # max is monotone: the pooled error is at most the largest allowance in the window
                    b = R.bound(ref, absref, r_out, c_acc, atol)
                    worst = max(worst, R.check(got[m], maxpool64(ref, 3, 2, 1), maxpool64(b, 3, 2, 1), 0.0, 1.0, 0.0, "%s image %d" % (name, m)))
                else:
                    worst = max(worst, R.check(got[m], ref, absref, r_out, c_acc, atol, "%s image %d" % (name, m)))
            self.note(label, worst)
        elif op == pg.RF_OP_MAXPOOL:
            for m, xi in enumerate(produced[src]):
                ref = maxpool64(xi, k, s, pad)
                assert got[m].shape == ref.shape, name
                err = float((got[m] - ref).abs().max())
                assert err <= (R.ATOL["split"] if engine == 4 else 0.0), (name, m, err)
            self.note("maxpool", 0.0)
        elif op in (pg.RF_OP_BLUR, pg.RF_OP_POOLBLUR):
            r_out, atol = {1: (R.R_TF32, 0.0), 2: (R.R_F16, R.ATOL["f16"]), 4: (R.R_SPLIT, R.ATOL["split"])}[engine]
            worst = 0.0
            for m, xi in enumerate(produced[src]):
                ref, absref = R.blur_ref(nchw(xi), s) if op == pg.RF_OP_BLUR else R.poolblur_ref(nchw(xi))
                worst = max(worst, R.check(nchw(got[m]), ref, absref, r_out, R.gamma(9) * (1 + r_out), atol, "%s image %d" % (name, m)))
            if engine == 1:
                assert bool(R.is_tf32(raw).all()), "%s: engine-1 outputs are not TF32-rounded" % name
            self.note("blur/%d" % s if op == pg.RF_OP_BLUR else "poolblur", worst)
        elif op == pg.RF_OP_IM2COL:
            rows = torch.cat([R.im2col_ref(nchw(xi.float()), k, s, pad, cout) for xi in produced[0]], 0)
            exp = {1: R.tf32_rna(rows), 2: rows.half(), 4: R.to_split(rows)}[engine]
            assert torch.equal(raw.contiguous().view(torch.int16), exp.contiguous().view(torch.int16)), "%s: im2col rows differ" % name
            self.note("im2col", 0.0)
        else:
            raise AssertionError("%s: op %d has no reference" % (name, op))


def test_conv64_matches_conv2d():
    """The tap-GEMM reference equals F.conv2d (fp64, CPU) at strides, paddings and dilations the programs use."""
    g = torch.Generator().manual_seed(0)
    for k, s, p, d in ((3, 1, 1, 1), (3, 2, 1, 1), (1, 2, 0, 1), (7, 2, 3, 1), (3, 1, 4, 4), (3, 1, 2, 2)):
        x = torch.randn(1, 5, 11, 13, generator=g, dtype=torch.float64)
        w = torch.randn(4, 5, k, k, generator=g, dtype=torch.float64)
        ref = F.conv2d(x, w, stride=s, padding=p, dilation=d)
        got = conv64(nhwc(x), w.permute(0, 2, 3, 1), s, p, d)
        assert torch.allclose(nchw(got), ref, rtol=1e-12, atol=1e-12), (k, s, p, d)


# ------------------------------------------------------------------ the replays
@pytest.mark.gpu
@pytest.mark.parametrize("engine,what", PROGRAMS, ids=["e%d-%s" % (e, p.replace(" ", "_")) for e, p in PROGRAMS])
def test_program_replay_layer_by_layer(rf, recorded, engine, what):
    recs = recorded.get((engine, what), [])
    assert recs, "no %s call on engine %d was recorded" % (what, engine)
    for rec in recs:
        rp = Replay(rf, rec)
        steps = rp.run()
        print("replay %s engine %d images %s: %d ops in %d steps; worst error / allowance per op kind: %s" % (
            what, engine, rec["hw"], len(rec["P"].ops), steps, ", ".join("%s %.3g" % kv for kv in sorted(rp.worst.items()))))


@pytest.mark.gpu
def test_recorded_image_sets(recorded):
    """The configurations the pipeline really ran: the trunk on the 8-image config-2 pyramid and the 4-image config-5 one, the
    fine networks at two target sizes per configuration, segNet at its two distinct sizes of 480 x 640 and one of 376 x 1241."""
    for (engine, what), recs in sorted((k, v) for k, v in recorded.items() if k != "_keep"):
        print("engine %d %s: %s" % (engine, what, [r["hw"] for r in recs]))
    for engine in ENGINES:
        trunk = sorted([r["hw"] for r in recorded[(engine, "trunk")]], key=len)
        assert [len(h) for h in trunk] == [4, 8] and trunk[1][0] == (960, 1280) and trunk[1][-1] == (480, 640), trunk
        assert len(recorded[(engine, "features")]) >= 3
    enc = [r["hw"] for r in recorded[(4, "segnet encoder")]]
    assert [(304, 400), (376, 504)] in enc and [(152, 504)] in enc, enc


# ------------------------------------------------------------------ segNet's decoder and vote at the network's sizes
def _ints(v):
    return (C.c_int * len(v))(*[int(x) for x in v])


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(480, 640), (376, 1241)])
def test_segnet_decoder_and_vote_on_own_conv5(rf, recorded, H, W):
    from ransac_flow_b200.segnet import NUM_CLASS, POOL_SCALES, PPM_CHANNELS
    seg = recorded["_keep"][-1]
    lib, st = rf._lib.lib, rf._lib.stream()
    img = synth.segnet_image(7, H, W)
    distinct, order = seg.plan(H, W)
    with torch.no_grad():
        conv5 = seg.encode(seg.resize(torch.from_numpy(img).cuda(), distinct))
    c5 = conv5.data.clone()
    n, hw, C5 = conv5.n, conv5.hw, conv5.C
    assert C5 == 2048
    x = decode(c5, "split", hw)
    hwc = _ints([v for p in hw for v in p])
    # the four adaptive poolings: serial fp32 sums of the cell (area terms, each read as hi + lo 2^-11), one division, split store
    pooled = [torch.full((2, n * b * b, C5), float("nan"), device="cuda", dtype=torch.float16) for b in POOL_SCALES]
    rf._lib.check(lib.rf_adaptive_avgpool_split(c5.data_ptr(), n, hwc, C5, _ints(POOL_SCALES), len(POOL_SCALES),
                                                (C.c_void_p * 4)(*[t.data_ptr() for t in pooled]), st))
    torch.cuda.synchronize()
    worst = {}
    for b, y in zip(POOL_SCALES, pooled):
        got = decode(y, "split", [(b, b)] * n)
        for m, (h, w) in enumerate(hw):
            ref = nhwc(F.adaptive_avg_pool2d(nchw(x[m]), b))
            absref = nhwc(F.adaptive_avg_pool2d(nchw(x[m].abs()), b))
            ys = [(oy * h // b, -(-(oy + 1) * h // b)) for oy in range(b)]
            xs = [(ox * w // b, -(-(ox + 1) * w // b)) for ox in range(b)]
            area = torch.tensor([[(y1 - y0) * (x1 - x0) for x0, x1 in xs] for y0, y1 in ys], dtype=torch.float64, device="cuda")
            g = (area + 2) * R.U / (1 - (area + 2) * R.U)                 # gamma_(area + 2): area - 1 additions, the reads, the division
            worst["avgpool %d" % b] = max(worst.get("avgpool %d" % b, 0.0), R.check(
                got[m], ref, absref * g[..., None] * (1 + R.R_SPLIT), R.R_SPLIT, 1.0, R.ATOL["split"], "%dx%d bins %d image %d" % (H, W, b, m)))
    # the four PPM 1x1 convolutions (512 channels, BN, ReLU) on the pooled cells
    branches = []
    for j, (b, y, fc) in enumerate(zip(POOL_SCALES, pooled, seg.ppm_convs)):
        br = rf.ops.conv2d(rf.ops.Ragged(y, [(b, b)] * n), fc.w, fc.bias, PPM_CHANNELS, 1, 1, 0, True, None, rf.ops.ENGINE_SPLIT, fc.w_split).data
        branches.append(br)
        torch.cuda.synchronize()
        wq = R.from_split(fc.w_split).reshape(PPM_CHANNELS, 1, 1, C5)
        for m, (xi, gi) in enumerate(zip(decode(y, "split", [(b, b)] * n), decode(br, "split", [(b, b)] * n))):
            ref = (conv64(xi, wq) + fc.bias.double()).clamp_min(0.0)
            absref = absconv(xi, wq) + fc.bias.double().abs()
            worst["ppm conv %d" % b] = max(worst.get("ppm conv %d" % b, 0.0), R.check(gi, ref, absref, R.R_SPLIT, R.ACC["split"], R.ATOL["split"], "ppm conv bins %d image %d" % (b, m)))
    # the concat: conv5 bit for bit, the branches bilinearly upsampled with ATen's fp32 source coordinates
    cy = C5 + 4 * PPM_CHANNELS
    P_ = sum(h * w for h, w in hw)
    cat = torch.full((2, P_, cy), float("nan"), device="cuda", dtype=torch.float16)
    rf._lib.check(lib.rf_ppm_concat_split(c5.data_ptr(), n, hwc, C5, (C.c_void_p * 4)(*[t.data_ptr() for t in branches]), _ints(POOL_SCALES),
                                          4, PPM_CHANNELS, cat.data_ptr(), st))
    torch.cuda.synchronize()
    assert torch.equal(cat[:, :, :C5].contiguous().view(torch.int16), c5.view(torch.int16)), "conv5 is not copied bit for bit"
    gcat = decode(cat, "split", hw)
    for j, b in enumerate(POOL_SCALES):
        brq = decode(branches[j], "split", [(b, b)] * n)
        for m, (h, w) in enumerate(hw):
            ref = F.interpolate(nchw(brq[m]).float(), (h, w), mode="bilinear", align_corners=False).double()
            absref = F.interpolate(nchw(brq[m]).abs(), (h, w), mode="bilinear", align_corners=False)
            got = nchw(gcat[m][..., C5 + j * PPM_CHANNELS:C5 + (j + 1) * PPM_CHANNELS])
            worst["concat branch %d" % b] = max(worst.get("concat branch %d" % b, 0.0), R.check(
                got, ref, absref, R.R_SPLIT, 2.0 ** -20, R.ATOL["split"], "branch %d image %d" % (j, m)))
    # conv_last (3x3 4096 -> 512 + ReLU, 1x1 512 -> 150 fp32 logits), layer by layer on the concat
    rp = Replay(rf, dict(P=seg.head, hw=hw, engine=4, x=cat, what="segnet conv_last"))
    rp.run()
    worst.update(rp.worst)
    logits, ohw = seg.head.run(rf.ops.Ragged(cat, hw), 4)
    logits = logits.clone()
    assert ohw == hw and logits.dtype == torch.float32 and logits.shape[1] == NUM_CLASS
    # the vote: scores += softmax(bilinear(logits of pass k)) / 5, arg-max, mask; fp64 reference with ATen's fp32 coordinates
    mask = torch.full((H, W), float("nan"), device="cuda")
    cls = torch.full((H, W), -1, device="cuda", dtype=torch.int32)
    scores = torch.full((H, W, NUM_CLASS), float("nan"), device="cuda")
    rf._lib.check(lib.rf_seg_vote(logits.data_ptr(), n, hwc, NUM_CLASS, _ints(order), len(order), H, W, seg.segId, int(seg.segFg),
                                  mask.data_ptr(), cls.data_ptr(), scores.data_ptr(), st))
    torch.cuda.synchronize()
    imgs = decode(logits, "f32", hw)
    ref = torch.zeros(NUM_CLASS, H, W, dtype=torch.float64, device="cuda")
    for k in order:
        up = F.interpolate(nchw(imgs[k]).float(), (H, W), mode="bilinear", align_corners=False).double()
        ref += torch.softmax(up, 1)[0] / len(order)
    ref = ref.permute(1, 2, 0)
    dev = float((scores.double() - ref).abs().max())
    assert dev <= 1e-6, dev
    top2 = ref.topk(2, -1).values
    decided = (top2[..., 0] - top2[..., 1]) > 2e-6
    assert torch.equal(cls[decided].long(), ref.argmax(-1)[decided]), int((cls[decided].long() != ref.argmax(-1)[decided]).sum())
    # every other pixel is a proven tie: the kernel's class is within 2e-6 of the fp64 maximum
    picked = ref.gather(-1, cls.long().clamp_min(0)[..., None])[..., 0]
    assert bool(((top2[..., 0] - picked) <= 2e-6).all())
    hit = (cls == seg.segId).float()
    assert torch.equal(mask, 1 - hit if seg.segFg else hit)
    print("segNet %dx%d (distinct %s, passes %s): vote max |score - fp64| %.3g, undecided pixels %d; worst error / allowance: %s" % (
        H, W, distinct, order, dev, int((~decided).sum()), ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
