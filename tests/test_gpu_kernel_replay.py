"""Every kernel call outside the layer programs, checked on the operands the pipeline really gave it.

A spy wraps the kernel entries of the package (the callables ``test_kernel_replay_inventory.INVENTORY`` marks "replayed
here": those of ``ops``, ``validation.affine_sample_u8`` / ``val_keypoints``, ``corr_results.corr_keypoints`` and
``train_pairs.warp_sample_u8``, plus ``ops.imresize_keep``, which composes two of them) while real eager pairs run.  The
callers reach each entry through its module (``ops.<name>``, or the module's own globals), so patching the module attributes
catches every call.  For each call the spy clones every tensor argument before the call and every result, plus the
arguments the call writes in place, after it (on the current stream), and records the scalars, the strides and the data
pointer alignment, which decide the kernel variant.  At most two calls are kept per (op, shapes, dtypes, scalars).  The
graphed paths are compared bit for bit with these eager ones elsewhere, so a call under stream capture fails the spy.

Workloads (engine f16x3, correlation precision 2, unless noted): config 2 (``align_pair_single`` with match21 at 480 x 640,
also on engines fp32 / precision 0 and tf32 / precision 1), config 3 (``getFlow_all`` at 240 on that pair's outputs), config 4
(``align_pair_multi``, maxCoarse 3, with the segNet sky mask), config 5 (``align_pair_kitti_graph`` eagerly at 376 x 1241,
then ``getFlow_all_kitti`` with the hole filling), YFCC (``align_pair_yfcc`` at 480 x 640 with a CUDA background),
quick_start's ``align2images`` at 240 x 320 on engines tf32 and f16x3, the one path that runs the single CorrNeigh, the split
one without its second volume, and the fine flow without clamp (with align_corners = True on tf32), and:
  evalCorr        ``corr_results.score_pair`` on config 4's hypotheses (multiH, and onlyCoarse) and on a 480 x 480 pair
                  with matchability thresholds (0, 0.5, 0.5): the row count of the broadcast, two thresholds on one row
  training pair   ``align_train_pair`` (10 000 RANSAC iterations on the Philox stream) on a 480 x 720 source and a 512 x 640
                  target, on engines f16x3 / precision 2 (presplit matching) and fp32 / precision 0
  validation      ``validation.validate_pair`` on a 500 x 700 source and a 620 x 470 target with a non-identity theta and
                  keypoints on the target's last row and column, wrapping and out of range, on engines f16x3 and tf32

Each recorded output is then compared with a reference computed from that call's own recorded inputs, within the bound of
the op's own unit test (named at each check).  Only the correlation (``test_gpu_wgmma_edges.corr_call``, to read its arg-max
keys) and the two keypoint kernels (into fresh accumulators, to read their per-keypoint outputs) are run again; the fused
warp is also compared with the kernel composition it replaces, and the evalCorr keypoints with the dense device maps.  One
test per check of the last four entries edits a copy of a recorded call and requires the check to fail on it.
"""
import inspect

import numpy as np
import PIL.Image as Image
import pytest
import torch

import geometry_ref as G
import ransac_ref as RR
import wgmma_ref as R
from oracle import synth
from oracle import warp_oracle as WO
from geometry_ref import bilinear_zeros, coord_delta, gamma, unnormalize64
from test_gpu_corr_results import _binary, _dense
from test_gpu_kitti_graph import numpy_step
from test_gpu_ops import corr_neigh_ref
from test_gpu_program_replay import _models
from test_gpu_wgmma_edges import corr_call
from test_gpu_ransac_exact import check_certified, kernel_provider
from test_gpu_train_pairs import composition
from test_gpu_validation import _network, affine_image, tail_ref
from test_kernel_replay_inventory import INVENTORY, REPLAYED
from train_pair_ref import decided, warp_u8_ref

pytestmark = pytest.mark.gpu

SPIED = dict(tuple(k.split(".", 1)[::-1]) for k, w in INVENTORY.items() if w == REPLAYED)      # entry name -> its module
SPIED["imresize_keep"] = "ops"
IN_PLACE = {"remove_small_cc": ("match",), "kitti_region_step": ("Mask", "fgMask", "alive", "rec"), "val_keypoints": ("counts",),
            "corr_keypoints": ("counts", "err")}
KEEP = 2


# ------------------------------------------------------------------ recording
def _snap(v):
    """A recorded copy of one argument or result: tensors cloned with their layout, Ragged as (data, hw)."""
    from ransac_flow_b200.ops import Ragged
    if isinstance(v, torch.Tensor):
        return dict(t=v.detach().clone(), stride=tuple(v.stride()), align=v.data_ptr() % 16, contiguous=v.is_contiguous())
    if isinstance(v, Ragged):
        return dict(ragged=True, t=v.data.detach().clone(), hw=list(v.hw), align=v.data.data_ptr() % 16)
    if isinstance(v, (tuple, list)) and any(isinstance(x, (torch.Tensor, Ragged)) for x in v):
        return [_snap(x) for x in v]
    return v


def _key_part(v):
    if isinstance(v, dict) and "t" in v:
        return (tuple(v["t"].shape), str(v["t"].dtype), tuple(v.get("hw", ())))
    if isinstance(v, list):
        return tuple(_key_part(x) for x in v)
    if isinstance(v, (int, float, bool, str)) or v is None:
        return v
    return type(v).__name__


class Recorder:
    def __init__(self, rf):
        self.rf, self.real, self.calls, self.counts = rf, {}, {}, {}
        self.where = "?"

    def wrap(self, name):
        mod = getattr(self.rf, SPIED[name])
        fn = getattr(mod, name)
        sig = inspect.signature(fn)
        rec = self

        def spy(*args, **kw):
            assert not torch.cuda.is_current_stream_capturing(), "%s recorded under stream capture" % name
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            before = {k: _snap(v) for k, v in b.arguments.items()}
            out = fn(*args, **kw)
            after = {k: _snap(b.arguments[k]) for k in IN_PLACE.get(name, ()) if b.arguments[k] is not None}
            if name == "kitti_region_step" and b.arguments["rec"] is None:
                after["rec"] = _snap(out)
            key = (name,) + tuple((k, _key_part(v)) for k, v in sorted(before.items()))
            rec.counts[key] = rec.counts.get(key, 0) + 1
            if rec.counts[key] <= KEEP:
                rec.calls.setdefault(name, []).append(dict(args=before, after=after, out=_snap(out), where=rec.where))
            return out

        self.real[name] = (mod, fn)
        setattr(mod, name, spy)

    def __enter__(self):
        for n in SPIED:
            self.wrap(n)
        return self

    def __exit__(self, *exc):
        for n, (mod, fn) in self.real.items():
            setattr(mod, n, fn)


def _segnet_class(rf, sds, img):
    """A segNet class covering between 10 % and 90 % of ``img``: a sky mask with both values."""
    from ransac_flow_b200.segnet import SegNet
    _, cls, _ = SegNet(None, None, 2, False, state_dicts=sds).run(torch.from_numpy(img).cuda(), want_class=True)
    ids, counts = np.unique(cls.cpu().numpy(), return_counts=True)
    ok = [(f, int(i)) for f, i in zip(counts / counts.sum(), ids) if 0.1 <= f <= 0.9]
    return min(ok)[1] if ok else int(ids[0])


TH_CANDIDATES = (0.95, 0.9, 0.8, 0.6, 0.4, 0.2, 0.1)


def _score(rf, out, seed, mth, later=False, onlyCoarse=False):
    """``corr_results.score_pair`` on one aligned pair (the target's size is the flow's) with 400 synthetic keypoints: (xb, yb)
    in [-W, W) x [-H, H), the corners, -1 and -W / -H, one column out of range; (xa, ya) the merged flow's estimate plus
    noise, so that the distances fall on both sides of the thresholds.  ``later``: th is the first of TH_CANDIDATES at
    which a later hypothesis wins on 0.1 % of the map, a quarter of the keypoints lie where one does, and the kernel must
    report such a winner."""
    flow, Hs, match = out["flowDown8"], np.asarray(out["H"]).reshape(-1, 3, 3), out["matchDown8"]
    H, W = flow.shape[2] * 8, flow.shape[3] * 8
    rs = np.random.RandomState(seed)
    n = 400
    yb, xb = rs.randint(-H, H, n), rs.randint(-W, W, n)
    yb[:8] = [H - 1, H - 1, 0, -1, -H, 0, H - 1, 5]
    xb[:8] = [W - 1, 0, W - 1, -1, -W, -W, -1, W]
    f, m = rf.pipeline._compose_all(flow, Hs, match, H, W)
    th = 0.95
    if later:
        for th in TH_CANDIDATES:
            won = (m[0, 0] < th) & (m[1:, 0] >= th).any(0)
            if float(won.float().mean()) > 1e-3:
                break
        else:
            raise AssertionError("no threshold in %s lets a later hypothesis win" % (TH_CANDIDATES,))
        py, px = (v.cpu().numpy() for v in torch.nonzero(won, as_tuple=True))
        pick = rs.choice(len(py), n // 4)
        yb[8:8 + n // 4], xb[8:8 + n // 4] = py[pick], px[pick]
    fg = rf.pipeline.merge_first_wins(f, m.permute(0, 2, 3, 1), th)[0][0].cpu().numpy()
    e = np.nan_to_num(fg[yb % H, xb % W])
    xa = (e[:, 0] + 1) * 0.5 * (W - 1) + rs.normal(0, 6, n)
    ya = (e[:, 1] + 1) * 0.5 * (H - 1) + rs.normal(0, 6, n)
    kpts = tuple(np.asarray(v, dtype=np.float32) for v in (xa, ya, xb, yb))
    scores = rf.corr_results.CorrScores(mth, th, multiH=True, onlyCoarse=onlyCoarse)
    ho = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    rf.corr_results.score_pair(out, kpts, ((W, H), (W, H)), scores, pair=3, hyp_out=ho)
    if later:
        assert bool((ho > 0).any()), "th %.2f: no keypoint takes a later hypothesis" % th


def _validation_inputs(rf):
    """A 500 x 700 source and a 620 x 470 target (resized to 480 x 672 and 624 x 480: other sizes, other aspect ratios), a
    non-identity theta and int32 keypoints in the resized images: on the target's last column and last row, -1 and -W / -H
    (which wrap), one row out of range; (xa, ya) near the affine estimate, so that the distances spread over the thresholds."""
    V = rf.validation
    Is, It = synth.make_pair(31, 500, 700)[0], synth.make_pair(32, 620, 470)[1]
    theta = np.array([[1.02, 0.03, 0.02], [-0.02, 0.98, -0.03]], np.float32)
    ws, hs = V.resize_min_resolution_size(700, 500)
    wt, ht = V.resize_min_resolution_size(470, 620)
    rs = np.random.RandomState(9)
    n = 600
    xb, yb = rs.randint(-wt, wt, n), rs.randint(-ht, ht, n)
    xb[:40] = wt - 1
    yb[40:80] = ht - 1
    xb[80:90], yb[80:90] = -1, -1
    xb[90], yb[90] = -wt, -ht
    xb[91], yb[91] = 3, ht
    gx, gy = (2 * (xb % wt) + 1) / wt - 1.0, (2 * (yb % ht) + 1) / ht - 1.0
    xa = (theta[0, 0] * gx + theta[0, 1] * gy + theta[0, 2] + 1) * 0.5 * (ws - 1) + rs.normal(0, 8, n)
    ya = (theta[1, 0] * gx + theta[1, 1] * gy + theta[1, 2] + 1) * 0.5 * (hs - 1) + rs.normal(0, 8, n)
    return Is, It, theta, np.stack([np.trunc(xa), np.trunc(ya), xb, yb], 1).astype(np.int32)


@pytest.fixture(scope="module")
def recorded(rf):
    from ransac_flow_b200.segnet import SegNet
    rec = Recorder(rf)
    try:
        with rec:
            for engine, prec in (("f16x3", 2), ("fp32", 0), ("tf32", 1)):
                rf.model.set_engine(engine)
                rf.outil.corr_precision = prec
                rec.where = "config 2 %s" % engine
                c, net = _models(rf, 2)
                s, t, _ = synth.make_pair(2, 480, 640)
                torch.manual_seed(1000)
                out = rf.pipeline.align_pair_single(c, net, torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), with_match21=True)
                assert len(out["H"]) == 1, "config 2: no homography, the fine flow never ran"
                if engine == "f16x3":
                    rec.where = "config 3"
                    rf.pipeline.getFlow_all(out["flowDown8"], out["H"], out["matchDown8"], 240, 240, th=0.95, multiH=True)
                if engine != "fp32":
                    # quick_start/align2images: the single CorrNeigh (tf32) or the split one without its second volume (f16x3),
                    # the fine flow without clamp, sampled with align_corners = True on one engine
                    rec.where = "align2images %s" % engine
                    qs, qt, _ = synth.make_pair(21, 240, 320)
                    cq = rf.CoarseAlignC(7, 1000, 0.05, "Homography", 320, scaleR=1.2, resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False)
                    torch.manual_seed(1000)
                    q = rf.pipeline.align2images(cq, net, Image.fromarray(qs), Image.fromarray(qt), align_corners=engine == "tf32")
                    assert q is not None, "align2images: no homography"
                torch.cuda.synchronize()
            rf.model.set_engine("f16x3")
            rf.outil.corr_precision = 2
            sds = (synth.segnet_encoder_state(0), synth.segnet_decoder_state(0))
            rsd = synth.resnet50_conv4_state(0)
            _, net = _models(rf, 2)
            # config 4: the hypothesis loop with the sky of the target masked
            s, t, _ = synth.make_pair(4, 480, 640)
            rec.where = "config 4"
            c4 = rf.CoarseAlignA(7, 1000, 0.05, "Homography", 480, _segnet_class(rf, sds, t), False, 2, True, True, resnet_state_dict=rsd,
                                 verbose=False, segnet_state_dicts=sds)
            c4.device_preproc = True
            torch.manual_seed(1000)
            out4 = rf.pipeline.align_pair_multi(c4, net, torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), maxCoarse=3, segNet=True)
            torch.cuda.synchronize()
            # config 5: the KITTI pair, then its recomposition with the hole filling
            c5, net5 = _models(rf, 5)
            s, t, _ = synth.make_pair(5, 376, 1241)
            rec.where = "config 5"
            torch.manual_seed(1000)
            k = rf.pipeline.align_pair_kitti_graph(c5, net5, Image.fromarray(s), Image.fromarray(t), maxH=3)
            assert len(k["H"]) >= 1, "config 5: no hypothesis accepted"
            rec.where = "config 5 getFlow_all_kitti"
            rf.pipeline.getFlow_all_kitti(k["H"], k["flow_d2"], k["flow"], k["mask"], 376, 1241, interpolate=True)
            torch.cuda.synchronize()
            # YFCC: the four rotated targets with a device background
            s, t, _ = synth.make_rotated_pair(81, 480, 640, 1)
            rec.where = "YFCC"
            sky = SegNet(None, None, _segnet_class(rf, sds, t), False, state_dicts=sds).run(torch.from_numpy(t).cuda())[0]
            cy = rf.CoarseAlignB(7, 1000, 0.05, "Homography", 480, 1, True, True, True, False, 2, resnet_state_dict=rsd, verbose=False)
            cy.device_preproc = True
            torch.manual_seed(1000)
            rf.pipeline.align_pair_yfcc(cy, net, Image.fromarray(s), Image.fromarray(t), maxCoarse=3, It_bg=sky)
            torch.cuda.synchronize()
            # evalCorr: config 4's hypotheses, then a square pair with positive matchability thresholds
            assert len(out4["H"]) >= 2, "config 4: %d hypotheses, the merge has nothing to choose from" % len(out4["H"])
            rec.where = "evalCorr config 4"
            _score(rf, out4, 40, (0,), later=True)
            rec.where = "evalCorr config 4 onlyCoarse"
            _score(rf, out4, 41, (0,), onlyCoarse=True)
            s, t, _ = synth.make_pair(6, 480, 480)
            rec.where = "evalCorr 480x480"
            torch.manual_seed(1000)
            sq = rf.pipeline.align_pair_multi(c4, net, torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), maxCoarse=3)
            assert len(sq["H"]) >= 1, "480 x 480: no hypothesis accepted"
            _score(rf, sq, 42, (0, 0.5, 0.5))
            torch.cuda.synchronize()
            # the training-pair notebook on both matching branches, and MegaDepth validation on both CorrNeigh paths
            s, t, _ = synth.make_pair(2, 480, 720)
            t = np.asarray(Image.fromarray(t).resize((640, 512), Image.BILINEAR))
            vs, vt, theta, vk = _validation_inputs(rf)
            for engine, prec in (("f16x3", 2), ("fp32", 0)):
                rf.model.set_engine(engine)
                rf.outil.corr_precision = prec
                rec.where = "training pair %s" % engine
                model = rf.train_pairs.TrainPairModel(rsd, minSize=480)
                torch.manual_seed(1000)
                tp = rf.pipeline.align_train_pair(model, s, t)
                assert tp["kept"] and tp["status"] == rf.outil.RF_RANSAC_OK, ("training pair not kept", engine, tp["status"], tp["nbMatch"])
                torch.cuda.synchronize()
            for engine in ("f16x3", "tf32"):
                rf.model.set_engine(engine)
                rec.where = "validation %s" % engine
                rf.validation.validate_pair(_network(rf), vs, vt, theta, vk, rf.validation.new_counts(), pair=5)
                torch.cuda.synchronize()
    finally:
        rf.model.set_engine("fp32")
        rf.outil.corr_precision = 0
    return rec.calls


# ------------------------------------------------------------------ helpers
def T(v):
    return v["t"]


def cpu(v):
    return T(v).cpu().numpy()


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.view(np.uint8)


def shape_of(v):
    return "x".join(str(s) for s in T(v).shape) if isinstance(v, dict) and "t" in v else str(v)


def ragged_nchw(v):
    n = len(v["hw"])
    h, w = v["hw"][0]
    return T(v).view(n, h, w, -1).permute(0, 3, 1, 2)


# ------------------------------------------------------------------ per-op checks: each returns (worst ratio, variant, shapes)
def check_resize(rf, call):
    """Pillow on the host copy, bit for bit (test_gpu_ops.test_device_lanczos_bit_exact_vs_pil)."""
    a = call["args"]
    img, ow, oh, fn = cpu(a["img"]), a["out_w"], a["out_h"], a["fn"]
    H, W, ch = img.shape
    flt = Image.LANCZOS if "lanczos" in fn else Image.BILINEAR
    mode = "L" if ch == 1 else "RGB"
    ref = np.asarray(Image.fromarray(img[..., 0] if ch == 1 else img, mode).resize((ow, oh), resample=flt)).reshape(oh, ow, ch)
    got = cpu(call["out"])
    assert np.array_equal(got, ref), "%s %s -> %dx%d: %d bytes differ from Pillow" % (fn, img.shape, ow, oh, int((got != ref).sum()))
    v = ["h"] if ow != W else []
    if oh != H:
        src_aligned = ow != W or (a["img"]["contiguous"] and a["img"]["align"] % 4 == 0)
        v.append("resample_v_kernel" if (ow * ch) % 4 == 0 and src_aligned else "resample_u8_kernel")
    return 0.0, "%s %s" % ("lanczos" if "lanczos" in fn else "bilinear", "+".join(v) or "copy"), "%dx%dx%d->%dx%d" % (H, W, ch, oh, ow)


def check_bytescale(rf, call):
    """dropin.imresize at the map's own size (PIL copies): scipy's bytescale (test_gpu_sky.test_bytescale_is_scipy_bytescale)."""
    from ransac_flow_b200.dropin import imresize
    m, k = cpu(call["args"]["m"]), int(call["args"]["rot"]) % 4
    r = np.rot90(m, k)
    assert np.array_equal(cpu(call["out"]), imresize(r, r.shape)), "rot %d" % k
    return 0.0, "rot %d" % k, shape_of(call["args"]["m"])


def check_imresize_keep(rf, call):
    """imresize(np.rot90(m, rot), (h, w)) < 128 (test_gpu_sky.expected_keep)."""
    from ransac_flow_b200.dropin import imresize
    a = call["args"]
    m = a["m"]
    m = cpu(m) if isinstance(m, dict) else np.asarray(m, np.float32)
    k, h, w = int(a["rot"]) % 4, int(a["h"]), int(a["w"])
    ref = imresize(np.rot90(m, k), (h, w)) < 128
    assert np.array_equal(cpu(call["out"]), ref), int((cpu(call["out"]) != ref).sum())
    return 0.0, "rot %d, kept %.3f" % (k, ref.mean()), "%s->%dx%d" % (m.shape, h, w)


def check_preproc(rf, call):
    """ToTensor (+ Normalize) in torchvision's op order, bit for bit (test_gpu_ops.test_preproc_bit_exact)."""
    a = call["args"]
    t = T(a["img_u8"]).cpu().float().div(255)
    if a["normalize"]:
        t = (t - torch.tensor([0.485, 0.456, 0.406]).view(1, 3)) / torch.tensor([0.229, 0.224, 0.225]).view(1, 3)
    assert torch.equal(T(call["out"]).cpu(), t)
    n = T(a["img_u8"]).numel()
    vec = a["img_u8"]["align"] % 4 == 0 and call["out"]["align"] == 0 and n >= 12
    return 0.0, "preproc_vec_kernel" if vec else "preproc_kernel", shape_of(a["img_u8"])


def check_l2norm(rf, call):
    """x / max(||x||, 1e-12) within gamma_C / 2 + 2u (test_gpu_layer_ops.test_l2norm_vs_fp64); masked rows exactly zero."""
    a = call["args"]
    x = T(a["x2d"])
    if x.dim() == 3:
        xq, kind = R.from_split(x), "split"
    else:
        xq, kind = x.double(), "f16" if x.dtype == torch.float16 else "f32"
    mask = T(a["mask"]) if a["mask"] is not None else None
    ref = R.l2norm_ref(xq, mask)
    C_ = xq.shape[-1]
    y = T(call["out"])
    worst = R.check(y, ref, ref, R.gamma(C_) / 2 + 2 * R.U, 0.0, 0.0, "l2norm %s" % kind)
    if mask is not None:
        assert not bool(y[mask == 0].any()), "masked rows are not zero"
    zero_rows = int((xq.abs().sum(1) == 0).sum())
    return worst, "%s%s, %d zero rows" % (kind, " masked %d rows" % int((mask == 0).sum()) if mask is not None else "", zero_rows), shape_of(a["x2d"])


def check_l2norm_planes(rf, call):
    """The split planes of the normalised rows within R_SPLIT + gamma_C / 2 + 2u (test_l2norm_vs_fp64's planes check)."""
    a = call["args"]
    xq = R.from_split(T(a["x_split"]))
    mask = T(a["mask"]) if a["mask"] is not None else None
    ref = R.l2norm_ref(xq, mask)
    planes = T(call["out"])
    worst = R.check(R.from_split(planes), ref, ref, R.R_SPLIT + R.gamma(xq.shape[1]) / 2 + 2 * R.U, 0.0, R.ATOL["split"], "l2norm planes")
    if mask is not None:
        assert not bool(planes[:, mask == 0].any()), "masked rows are not zero"
    return worst, "split%s" % (" masked %d rows" % int((mask == 0).sum()) if mask is not None else ""), shape_of(a["x_split"])


# -- mutual nearest neighbours
def check_keys_device(keys, X, Y, c, what, chunk=2048):
    """test_gpu_wgmma_edges.check_keys with the fp64 scores S = X Y^T of one side computed on the device in row chunks and the
    top-2 selection by torch.topk: the key's score within R_F32 |s| + c |X||Y|^T of the fp64 score at its index; the fp64
    arg-max wherever the top-2 gap exceeds twice the row's allowance; never below the maximum by more than that.
    Returns (scores, indices, worst ratio)."""
    score, idx = (torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in R.decode_key(keys))
    assert bool((idx >= 0).all()) and bool((idx < Y.shape[0]).all()), (what, "missing or out-of-range key")
    Xa, Ya = X.abs(), Y.abs()
    worst = 0.0
    for r0 in range(0, X.shape[0], chunk):
        S = X[r0:r0 + chunk] @ Y.T
        A = Xa[r0:r0 + chunk] @ Ya.T
        rows = torch.arange(S.shape[0], device="cuda")
        ii = idx[r0:r0 + chunk]
        s64, a64 = S[rows, ii], A[rows, ii]
        tol = R.R_F32 * s64.abs() + c * a64
        err = (score[r0:r0 + chunk].double() - s64).abs()
        assert bool((err <= tol).all()), (what, "score", r0 + int((err - tol).argmax()), float((err / tol).max()))
        worst = max(worst, float((err / tol).max()))
        allow = 2 * (R.R_F32 * S.abs().amax(1) + c * A.amax(1))
        if S.shape[1] > 1:
            top = S.topk(2, dim=1).values
            clear = top[:, 0] - top[:, 1] > allow
        else:
            top = S
            clear = torch.ones(S.shape[0], dtype=torch.bool, device="cuda")
        best = S.argmax(1)
        assert bool((ii[clear] == best[clear]).all()), (what, "arg-max", r0 + torch.nonzero(ii[clear] != best[clear])[:5, 0])
        assert bool((s64 >= top[:, 0] - allow).all()), (what, "picked score below the maximum")
        del S, A
    return score, idx, worst


def _check_mutual(rf, call, mode, A, B, Aq, Bq, planes=None):
    c = R.ACC["split"] if mode in (2, "presplit") else R.acc_tf32x3(A.shape[1]) if mode == 1 else A.shape[1] * R.U / (1 - A.shape[1] * R.U)
    rowk, colk, i1, i2 = corr_call(rf, A, B, mode, planes)
    i1, i2 = torch.from_numpy(i1).cuda(), torch.from_numpy(i2).cuda()
    n = int(T(call["out"][2]).item())
    assert torch.equal(i1, T(call["out"][0])[:n]) and torch.equal(i2, T(call["out"][1])[:n]), "the re-run's pairs differ from the recorded call's"
    csc, cidx, cw = check_keys_device(colk, Bq, Aq, c, "columns")
    rsc, ridx, rw = check_keys_device(rowk, Aq, Bq, c, "rows")
    mutual = cidx[ridx] == torch.arange(len(ridx), device="cuda")
    assert torch.equal(rsc[mutual].view(torch.int32), csc[ridx[mutual]].view(torch.int32)), "mutual pair scores differ"
    keep = mutual & (rsc.double() ** 2 > 0)
    assert torch.equal(i1, torch.nonzero(keep)[:, 0]) and torch.equal(i2, ridx[keep]), "the pairs are not the mutual pairs of the keys"
    zero_rows = int((Bq.abs().sum(1) == 0).sum())
    return max(cw, rw), "precision %s, %d pairs, %d all-zero target rows" % (mode, n, zero_rows), "%dx%d C %d" % (A.shape[0], B.shape[0], A.shape[-1])


def check_corr_mutual_nn(rf, call):
    a = call["args"]
    A, B, mode = T(a["featA"]).contiguous(), T(a["featB"]).contiguous(), int(a["precision"])
    split = lambda X: R.from_split(R.to_split(X))
    Aq, Bq = (split(A), split(B)) if mode == 2 else (A.double(), B.double())
    return _check_mutual(rf, call, mode, A, B, Aq, Bq)


def check_corr_mutual_nn_presplit(rf, call):
    a = call["args"]
    p = [T(a[k]) for k in ("A_hi", "A_lo", "B_hi", "B_lo")]
    Aq = p[0].double() + p[1].double() / 2048.0
    Bq = p[2].double() + p[3].double() / 2048.0
    return _check_mutual(rf, call, "presplit", p[0], p[2], Aq, Bq, planes=((p[0], p[1]), (p[2], p[3])))


def check_build_matches(rf, call):
    """geometry_ref.build_matches_ref, bit for bit (test_gpu_geometry.test_build_matches_bit_exact)."""
    a = call["args"]
    cap = T(a["idx1"]).shape[0]
    v16 = cpu(a["valid16"]) if a["valid16"] is not None else None
    e1, e2, ek, n = G.build_matches_ref(cpu(a["idx1"]), cpu(a["idx2"]), int(cpu(a["count"])[0]), cpu(a["W1"]), cpu(a["H1"]), cpu(a["W2"]),
                                        cpu(a["H2"]), v16, cap)
    m1, m2, kept, cnt = (cpu(o) for o in call["out"])
    assert int(cnt[0]) == n and np.array_equal(bits(m1[:n]), bits(e1)) and np.array_equal(bits(m2[:n]), bits(e2)) and np.array_equal(kept[:n], ek)
    return 0.0, "%d of %d pairs kept%s" % (n, int(cpu(a["count"])[0]), " (valid16)" if v16 is not None else ""), "cap %d" % cap


def check_ransac(rf, call):
    """ransac_ref.ransac_given_H on the reduced sample table with the kernel's own DLT, bit for bit, then the certified bounds
    against LAPACK (test_gpu_ransac_exact.check_exact / check_certified), with the recorded raw table, M_dev and sample mode."""
    from ransac_flow_b200 import ops
    a = call["args"]
    m1, m2, raw = cpu(a["match1"]), cpu(a["match2"]), cpu(a["samples"])
    Md = int(cpu(a["M_dev"])[0]) if a["M_dev"] is not None else None
    mode = a["sample_mode"] if a["sample_mode"] is not None else (ops.SAMPLES_INDEX if Md is None else ops.SAMPLES_MOD)
    M = len(m1) if Md is None else min(Md, len(m1))
    H, nb, mask, st = (cpu(o) for o in call["out"])
    names = {ops.SAMPLES_INDEX: "index", ops.SAMPLES_MOD: "mod", ops.SAMPLES_PHILOX64: "philox64"}
    if M < 4:
        assert int(st[0]) == RR.TOO_FEW and int(nb[0]) == 0 and not mask.any()
        return 0.0, "%s, too few matches (%d)" % (names[mode], M), "M %d" % M
    if mode == ops.SAMPLES_PHILOX64:
        red = ((raw.view(np.uint64) >> np.uint64(32)) % np.uint64(M)).astype(np.int64)
    elif mode == ops.SAMPLES_MOD:
        red = raw % M
    else:
        red = raw
    a1, a2 = m1[:M], m2[:M]
    us = np.asarray(red).reshape(-1, 4)[RR.unique_rows(red)]
    tol = float(a["tolerance"])
    exp = RR.ransac_given_H(a1, a2, red, tol, kernel_provider(rf)(a1[us], a2[us]))
    assert int(st[0]) == exp["status"] and int(nb[0]) == exp["nbInlier"], (int(st[0]), exp["status"], int(nb[0]), exp["nbInlier"])
    assert np.array_equal(mask[:M].astype(bool), exp["mask"]) and not mask[M:].any()
    assert np.array_equal(H.reshape(3, 3).view(np.int32), exp["H"].view(np.int32))
    unc, amb, differ, _ = check_certified(a1, a2, red, tol, exp, "ransac")
    return 0.0, "%s, M %d, %d inliers, %d uncertified hypotheses" % (names[mode], M, exp["nbInlier"], unc), "M %d x %d iters" % (M, len(red))


def check_warp_grid(rf, call):
    """geometry_ref.warp_grid_f32, bit for bit (test_gpu_geometry.test_warp_grid_bit_exact)."""
    a = call["args"]
    Hm = cpu(a["H"]).reshape(-1, 9).astype(np.float32)
    ref = G.warp_grid_f32(Hm, a["h"], a["w"])
    assert np.array_equal(bits(cpu(call["out"])), bits(ref))
    return 0.0, "%d homographies" % len(Hm), "%dx%d" % (a["h"], a["w"])


def check_grid_sample(rf, call):
    """geometry_ref.grid_sample_ref's allowance (test_gpu_geometry.test_grid_sample_vs_fp64), output in the input's layout."""
    a = call["args"]
    inp, grid, ac = T(a["inp"]), T(a["grid"]), bool(a["align_corners"])
    ref, allow, outside = G.grid_sample_ref(inp.float().cpu().numpy(), grid.float().cpu().numpy(), ac)
    out = T(call["out"])
    worst = G.check(out.cpu().numpy(), ref, allow, "grid_sample")
    cl = a["inp"]["stride"][1] == 1 and inp.shape[1] > 1                  # the wrapper's rule, on the strides it was given
    assert call["out"]["stride"][1] == (1 if cl else out.shape[2] * out.shape[3]), "output layout"
    return worst, "ac %d, %s input, %d outside samples" % (ac, "channels-last" if cl else "strides %s" % (a["inp"]["stride"],), int(outside.sum())), \
        "%s grid %s" % (shape_of(a["inp"]), shape_of(a["grid"]))


def check_upsample(rf, call):
    """geometry_ref.upsample_ref's allowance (test_gpu_geometry.test_upsample_vs_fp64)."""
    a = call["args"]
    x = T(a["x"]).float()
    N, Cc, h, w = x.shape
    H, W = a["size"]
    ref, allow = G.upsample_ref(x.reshape(N * Cc, h, w).cpu().numpy(), H, W)
    worst = G.check(cpu(call["out"]).reshape(N * Cc, H, W), ref, allow, "upsample")
    return worst, "scale %.3g x %.3g" % (H / h, W / w), "%s->%dx%d" % (shape_of(a["x"]), H, W)


def check_compose_fine(rf, call):
    """geometry_ref.compose_fine_ref and compose_check (test_gpu_geometry.test_compose_fine_vs_fp64)."""
    a = call["args"]
    f8 = cpu(a["flowDown8"])[0]
    m12 = cpu(a["match12"])[0, 0] if a["match12"] is not None else None
    m21 = cpu(a["match21"])[0, 0] if a["match21"] is not None else None
    coarse = cpu(a["coarse"])[0]
    H, W = (coarse.shape[0], coarse.shape[1]) if a["size"] is None else (int(a["size"][0]), int(a["size"][1]))
    ref = G.compose_fine_ref(f8, m12, m21, coarse, H, W, bool(a["clamp"]), bool(a["align_corners"]))
    flow12, match, flowUp = call["out"]
    r, und = G.compose_check(ref, cpu(flow12)[0], cpu(match)[0, 0] if match is not None else None, cpu(flowUp)[0] if flowUp is not None else None)
    clamped = int((np.abs(ref["flowUp"]) == 1.0).any(-1).sum())
    return max(r.values()), "clamp %d ac %d m21 %d, %d undecided, %d at +-1" % (a["clamp"], a["align_corners"], m21 is not None, und, clamped), \
        "%s coarse %s -> %dx%d" % (f8.shape, coarse.shape, H, W)


# -- CorrNeigh
CORR_OUT = {0: (0.0, 0.0), 1: (R.R_TF32, 0.0), 2: (R.R_F16, R.ATOL["f16"])}


def _corr_refs(a):
    x, y = ragged_nchw(a["x"]).cpu(), ragged_nchw(a["y"]).cpu()
    return x, y, x.shape[1] * 2.0 ** -24 / (1 - x.shape[1] * 2.0 ** -24)


def _corr_half(got, ref, absref, k, mode, gamma, what):
    """test_gpu_ops.test_corr_neigh_kernels_match_fp64_reference's bound; the columns between k^2 and ldo are zero."""
    r_out, atol = CORR_OUT[mode]
    worst = R.check(got[:, :k * k].cpu(), ref, absref, r_out, gamma * (1 + r_out), atol, what)
    assert not bool(got[:, k * k:].any()), what + ": padding columns"
    if mode == 1:
        assert bool(R.is_tf32(got).all()), what + ": TF32-rounded output has low mantissa bits"
    return worst


def _variant(k, ldo, mode):
    return "%s ldo %d mode %s" % ("corr_neigh7_kernel" if k == 7 else "corr_neigh_kernel", ldo, mode)


def check_corr_neigh(rf, call):
    a = call["args"]
    k, mode = int(a["k"]), int(a["round_tf32"])
    x, y, gamma = _corr_refs(a)
    ref, absref = corr_neigh_ref(x, y, k)
    got = T(call["out"])
    return _corr_half(got, ref, absref, k, mode, gamma, "corr_neigh"), _variant(k, got.shape[1], mode), "%s C %d" % (a["x"]["hw"], x.shape[1])


def check_corr_neigh_pair(rf, call):
    a = call["args"]
    k, mode = int(a["k"]), int(a["round_tf32"])
    x, y, gamma = _corr_refs(a)
    both = T(call["out"][2])
    P = both.shape[0] // 2
    w1 = _corr_half(both[:P], *corr_neigh_ref(x, y, k), k, mode, gamma, "corr_neigh_pair xy")
    w2 = _corr_half(both[P:], *corr_neigh_ref(y, x, k), k, mode, gamma, "corr_neigh_pair yx")
    assert torch.equal(T(call["out"][0]), both[:P]) and torch.equal(T(call["out"][1]), both[P:])
    return max(w1, w2), "pair " + _variant(k, both.shape[1], mode), "%s C %d" % (a["x"]["hw"], x.shape[1])


def check_corr_neigh_pair_split(rf, call):
    """Split planes: fp32-grade sums (gamma_C) and the split's 2^-21 (test_corr_neigh_kernels_match_fp64_reference)."""
    a = call["args"]
    k, ldo = int(a["k"]), int(a["ldo"])
    x, y, gamma = _corr_refs(a)
    c12 = T(call["out"][0])
    P = c12.shape[1]
    halves = [("xy", R.from_split(c12), corr_neigh_ref(x, y, k))]
    if call["out"][1] is not None:
        both = T(call["out"][1])
        assert torch.equal(both[:, :P], c12)
        halves.append(("yx", R.from_split(both[:, P:]), corr_neigh_ref(y, x, k)))
    worst = 0.0
    for name, got, (ref, absref) in halves:
        worst = max(worst, R.check(got[:, :k * k].cpu(), ref, absref, 0.0, gamma, 2.0 ** -21, "corr_neigh_pair_split " + name))
        assert not bool(got[:, k * k:].any()), "padding columns"
    return worst, "split " + _variant(k, ldo, "split") + (" both" if len(halves) == 2 else ""), "%s C %d" % (a["x"]["hw"], x.shape[1])


def check_softmax_flow(rf, call):
    """wgmma_ref.softmax_flow_ref within (k^2 + 8) u sums + u |ref| (test_gpu_layer_ops.test_softmax_flow_vs_fp64)."""
    a = call["args"]
    k = int(a["k"])
    lg = ragged_nchw(a["logits"])
    ref, absf = R.softmax_flow_ref(lg, k)
    worst = R.check(T(call["out"]), ref, absf, R.U, (k * k + 8) * R.U, (2 * k ** 3 + 4) * 2.0 ** -149, "softmax_flow")
    return worst, "k %d" % k, "%s" % a["logits"]["hw"]


def check_sigmoid(rf, call):
    """fp64 sigmoid within 2^-21 |ref| + 2^-126 (test_gpu_layer_ops.test_sigmoid_vs_fp64)."""
    x = T(call["args"]["x"])
    ref = torch.sigmoid(x.double())
    worst = R.check(T(call["out"]), ref, torch.zeros_like(ref), 2.0 ** -21, 0.0, 2.0 ** -126, "sigmoid")
    near = int(((ref > 0.99) & (ref < 0.9999 + 1e-4)).sum())
    return worst, "%d values in [0.99, 0.9999]" % near, shape_of(call["args"]["x"])


def check_remove_small_cc(rf, call):
    """oracle.warp_oracle.remove_small_cc per map, bit for bit (test_gpu_kitti.test_remove_small_cc_fuzz_vs_oracle)."""
    a = call["args"]
    m = cpu(a["match"])
    H, W = m.shape[-2], m.shape[-1]
    maps = m.reshape(-1, H, W)
    ref = np.stack([WO.remove_small_cc(x, float(a["match_th"]), float(a["cc_th"])) for x in maps])
    got = cpu(call["after"]["match"]).reshape(-1, H, W)
    assert np.array_equal(got, ref), int((got != ref).sum())
    return 0.0, "%d maps, %d pixels removed" % (len(maps), int(((maps > a["match_th"]) & ~(ref > a["match_th"])).sum())), "%dx%d" % (H, W)


def check_kitti_region_step(rf, call):
    """The numpy statements of test_gpu_kitti_graph.numpy_step, bit for bit, at the threshold the pipeline's cmin encodes."""
    from ransac_flow_b200 import pipeline
    a, af = call["args"], call["after"]
    match, Mask, bg, fg = (cpu(a[k]).reshape(cpu(a["match"]).shape[-2:]) for k in ("match", "Mask", "bg", "fgMask"))
    status, alive, first, cmin = int(cpu(a["status"])[0]), int(cpu(a["alive"])[0]), bool(a["first"]), int(a["cmin"])
    th = [t for t in (0.005, 0.01) if pipeline.kitti_region_cmin(match.size, t) == cmin]
    assert th, "cmin %d is no known maskRegionTh's" % cmin
    want = numpy_step(match, Mask, bg, fg, status, alive, first, th[0])
    gM, gf = cpu(af["Mask"]).reshape(match.shape), cpu(af["fgMask"]).reshape(match.shape)
    ga, rec = int(cpu(af["alive"])[0]), cpu(af["rec"])
    assert np.array_equal(gM, want[0]) and np.array_equal(gf, want[1])
    assert ga == int(want[2]) and rec[0] == ga and rec[1] == want[3], (ga, rec, want[2:])
    return 0.0, "status %d first %d alive %d -> %d, count %d (cmin %d)" % (status, first, alive, ga, want[3], cmin), "%dx%d" % match.shape


def check_fill_nearest(rf, call):
    """Every unmatched pixel takes the flow of a matched pixel at exactly the EDT distance, matched pixels keep theirs (test_gpu_kitti.
    test_fill_nearest_matched_is_exact; between equidistant matched pixels any one is accepted)."""
    import scipy.ndimage as nd
    a = call["args"]
    f = T(a["flow"]).float()
    H, W = f.shape[1], f.shape[2]
    m = T(a["matched"]).reshape(H, W).bool()
    out = T(call["out"]) if not a["want_index"] else T(call["out"][0])
    mn = m.cpu().numpy()
    if not mn.any():
        assert torch.equal(out, f)
        return 0.0, "nothing matched", "%dx%d" % (H, W)
    d, (iy, ix) = nd.distance_transform_edt(~mn, return_indices=True)
    d2 = torch.from_numpy(np.round(d ** 2).astype(np.int64)).cuda()
    src = f[0][torch.from_numpy(iy).cuda(), torch.from_numpy(ix).cuda()]
    assert torch.equal(out[0][m], f[0][m]), "matched pixels changed"
    other = torch.nonzero(~(out[0] == src).all(-1))
    my, mx = torch.nonzero(m, as_tuple=True)
    fm = f[0][my, mx]
    for i0 in range(0, len(other), 256):             # pixels filled from another pixel than scipy's: an equidistant matched one
        p = other[i0:i0 + 256]
        dd = (my[None] - p[:, :1]) ** 2 + (mx[None] - p[:, 1:]) ** 2
        at = dd == d2[p[:, 0], p[:, 1]][:, None]
        same = (fm[None] == out[0][p[:, 0], p[:, 1]][:, None]).all(-1)
        assert bool((at & same).any(1).all()), "a pixel's flow is not that of a matched pixel at the EDT distance"
    return 0.0, "%.3f matched, %d ties resolved otherwise than scipy" % (mn.mean(), len(other)), "%dx%d" % (H, W)


# -- training pairs, validation, evalCorr
def check_warp_sample(rf, call):
    """Bit for bit against the composition it fuses (test_gpu_train_pairs.test_warp_sample_equals_its_composition), then
    floor(255 v) of train_pair_ref.warp_u8_ref (fp64 at the kernel's fp32 grid) on every byte outside the truncation band
    (test_warp_sample_vs_fp64)."""
    a = call["args"]
    H, src, h, w = T(a["H"]), T(a["src"]), int(a["h"]), int(a["w"])
    assert not a["align_corners"], "the composition samples with align_corners = False"
    got = T(call["out"])
    want = composition(rf, H, src, h, w)
    assert torch.equal(got, want), "%d bytes differ from the composition" % int((got != want).sum())
    src_np, got = src.cpu().numpy(), got.cpu().numpy().astype(np.int64)
    g32 = G.warp_grid_f32(H.cpu().numpy().reshape(1, 3, 3), h, w)[0]
    v, _ = warp_u8_ref(None, src_np, h, w, grid=(g32[..., 0], g32[..., 1]))
    _, allow, _ = G.grid_sample_ref((src_np.astype(np.float32) / np.float32(255)).transpose(2, 0, 1)[None], g32[None], False)
    band = 255.0 * allow[0].transpose(1, 2, 0) + 2 * 255.0 * G.U * v
    ok = decided(v, band)
    off = got != np.floor(v).astype(np.int64)
    assert not (off & ok).any(), "%d decided bytes differ from fp64's truncation" % int((off & ok).sum())
    assert np.abs(got - np.floor(v)).max() <= 1
    return 0.0, "%d of %d bytes in the truncation band, %d of them off by one" % (int((~ok).sum()), ok.size, int(off.sum())), \
        "%dx%d -> %dx%d" % (src_np.shape[0], src_np.shape[1], h, w)


def affine_ref(call):
    """The recorded affine_sample_u8 output as (3, h, w) fp64 with test_gpu_validation.affine_image's fp64 sample and the
    bound of test_affine_sample_fp64_and_torch."""
    a = call["args"]
    th, src, h, w = cpu(a["theta"]).reshape(2, 3), cpu(a["src"]), int(a["h"]), int(a["w"])
    Hin, Win = src.shape[:2]
    P, S = affine_image(th, h, w)
    ix, iy = unnormalize64(P[0], Win, False), unnormalize64(P[1], Hin, False)
    val, absval, Lx, Ly, _ = bilinear_zeros((src.astype(np.float32) / np.float32(255)).transpose(2, 0, 1), ix, iy)
    allow = gamma(7) * absval + Lx * (coord_delta(ix) + Win / 2.0 * gamma(2) * S[0]) + Ly * (coord_delta(iy) + Hin / 2.0 * gamma(2) * S[1])
    got = cpu(call["out"]).astype(np.float64).reshape(h, w, 3).transpose(2, 0, 1)
    return got, val, allow


def check_affine_sample(rf, call):
    got, val, allow = affine_ref(call)
    worst = G.check(got, val, allow, "affine_sample_u8")
    a = call["args"]
    return worst, "theta %s" % np.round(cpu(a["theta"]).astype(np.float64), 3).tolist(), "%s -> %dx%d" % (shape_of(a["src"]), a["h"], a["w"])


def _err_word(v):
    """The low 32 bits of the last int64 of an accumulator (or the int32 word itself), recorded or not."""
    t = T(v) if isinstance(v, dict) else v
    return int(np.ascontiguousarray(t.cpu().numpy().reshape(-1)[-1:]).view(np.int32)[0])


def check_val_keypoints(rf, call):
    """Run again into a fresh accumulator with dist_out / flow_out: the same count delta and error word as the recorded call;
    the fine flow and each distance within test_gpu_validation.tail_ref's fp64 bounds (test_keypoint_tail_fp64); the counts
    those of the fp64 distances except for keypoints within the bound of a threshold (set aside, at most 2 %, as
    test_dataset_matches_the_reference's MAX_ASIDE); the error word holds ``pair`` exactly when torch's index rule rejects a
    keypoint."""
    V = rf.validation
    a = call["args"]
    kp, H, W, hA, wA = T(a["kpts"]), int(a["size_t"][0]), int(a["size_t"][1]), int(a["size_s"][0]), int(a["size_s"][1])
    thr = np.asarray(a["thresholds"], dtype=np.float64).reshape(-1)
    cap = kp.shape[0]
    acc = torch.zeros_like(T(a["counts"]))
    acc[-1] = V.NO_ERROR
    d = torch.full((cap,), float("nan"), dtype=torch.float64, device="cuda")
    fo = torch.full((cap, 4), float("nan"), device="cuda")
    V.val_keypoints(T(a["flowDown8"]), T(a["theta"]), (H, W), (hA, wA), kp, T(a["count"]), acc, a["pair"], d, fo, a["thresholds"])
    counts, _ = V.read_counts(acc.cpu().numpy())
    delta = cpu(call["after"]["counts"])[:-1] - cpu(a["counts"])[:-1]
    assert np.array_equal(delta, counts), ("count delta", delta.tolist(), counts.tolist())
    n = min(int(cpu(a["count"])[0]), cap)
    k = kp[:n].cpu().numpy().astype(np.int64)
    ok = (k[:, 3] >= -H) & (k[:, 3] < H) & (k[:, 2] >= -W) & (k[:, 2] < W)
    want_err = a["pair"] if not ok.all() else V.NO_ERROR
    assert _err_word(acc) == want_err, ("re-run error word", _err_word(acc), want_err)
    assert _err_word(call["after"]["counts"]) == min(_err_word(a["counts"]), want_err), "recorded error word"
    dk, fk = d.cpu().numpy()[:n][ok], fo.cpu().numpy()[:n][ok]
    fl, ef, dref, adist = tail_ref(cpu(a["flowDown8"]), cpu(a["theta"]), H, W, hA, wA, k[ok])
    G.check(fk[:, :2], fl, ef, "val_keypoints fine flow")
    worst = G.check(dk, dref, adist, "val_keypoints distance")
    assert np.array_equal(counts[:-1], (dk[:, None] < thr).sum(0)) and counts[-1] == ok.sum(), "counts differ from dist_out's"
    near = (np.abs(dref[:, None] - thr) <= adist[:, None]).any(1)
    assert near.sum() <= 0.02 * len(dk), ("keypoints within the bound of a threshold", int(near.sum()), len(dk))
    exp = (dref[~near, None] < thr).sum(0) + (dk[near, None] < thr).sum(0)
    assert np.array_equal(counts[:-1], exp), ("counts differ from fp64's", counts.tolist(), exp.tolist())
    ys, xs = k[ok, 3] % H, k[ok, 2] % W
    return worst, "%d keypoints (%d on the last row / column, %d out of range, %d set aside), error word %s" % (
        n, int(((ys == H - 1) | (xs == W - 1)).sum()), int((~ok).sum()), int(near.sum()),
        "pair %d" % want_err if want_err != V.NO_ERROR else "untouched"), \
        "flow %s target %dx%d source %dx%d" % (shape_of(a["flowDown8"]), H, W, hA, wA)


def check_corr_keypoints(rf, call):
    """Run again into fresh accumulators with flow_out / match_out / hyp_out / dist_out: the same count delta and error word
    as the recorded call; the merged flow and matchability at each keypoint bit for bit against the dense device path
    (test_gpu_corr_results.test_kernel_against_dense), each winning hypothesis against geometry_ref.compose_fine_ref
    (test_composition_against_fp64), the counts equal to results.alignment_error on the dense maps, broadcast included."""
    C = rf.corr_results
    a = call["args"]
    f8, kp = T(a["flowDown8"]), T(a["kpts"])
    nH, _, h8, w8 = f8.shape
    Hd, Wd = 8 * h8, 8 * w8
    Ith, Itw, hA, wA = int(a["size_t"][0]), int(a["size_t"][1]), int(a["size_s"][0]), int(a["size_s"][1])
    mth, slots = [float(t) for t in np.reshape(a["mth"], -1)], [int(q) for q in np.reshape(a["slots"], -1)]
    th, multiH, onlyCoarse = a["th"], a["multiH"], a["onlyCoarse"]
    pg = np.asarray(a["thresholds"], dtype=np.float64)
    nT, J, cap = pg.size, len(mth), kp.shape[0]
    acc, err = torch.zeros_like(T(a["counts"])), torch.full((1,), C.NO_ERROR, dtype=torch.int32, device="cuda")
    fo, mo = torch.full((cap, 2), float("nan"), device="cuda"), torch.full((cap,), float("nan"), device="cuda")
    ho, do = torch.full((cap,), -1, dtype=torch.int32, device="cuda"), torch.full((cap, J), float("nan"), dtype=torch.float64, device="cuda")
    m8 = T(a["matchDown8"]) if a["matchDown8"] is not None else None
    C.corr_keypoints(f8, m8, T(a["H"]), (Ith, Itw), (hA, wA), kp, T(a["count"]), acc, err, a["thresholds"], mth, slots, th, multiH,
                     onlyCoarse, a["pair"], fo, mo, ho, do)
    rows = (max(slots) + 1) * (nT + 1)
    counts = acc.cpu().numpy()[:rows]
    delta = cpu(call["after"]["counts"]).reshape(-1)[:rows] - cpu(a["counts"]).reshape(-1)[:rows]
    assert np.array_equal(delta, counts), ("count delta", delta.tolist(), counts.tolist())
    n = min(int(cpu(a["count"])[0]), cap)
    k = kp[:n].cpu().numpy().astype(np.int64)
    inside = lambda h, w: (k[:, 3] >= -h) & (k[:, 3] < h) & (k[:, 2] >= -w) & (k[:, 2] < w)
    ok, okt = inside(Hd, Wd), inside(Ith, Itw)
    assert not (ok & ~okt).any(), "keypoints on the map but outside the target's view: a case this check does not cover"
    want_err = a["pair"] if not ok.all() else C.NO_ERROR
    assert _err_word(err) == want_err, ("re-run error word", _err_word(err), want_err)
    assert _err_word(call["after"]["err"]) == min(_err_word(a["err"]), want_err), "recorded error word"
    flow, Hs = f8.cpu().numpy(), T(a["H"]).cpu().numpy().reshape(-1, 3, 3)
    match = m8.cpu().numpy() if m8 is not None else None
    fg, mg = _dense(Hs, flow, match, multiH, th, onlyCoarse)
    ys, xs = k[ok, 3] % Hd, k[ok, 2] % Wd
    fk, mk, hk = fo.cpu().numpy()[:n][ok], mo.cpu().numpy()[:n][ok], ho.cpu().numpy()[:n][ok]
    assert np.array_equal(fk.view(np.int32), fg[0].cpu().numpy()[ys, xs].view(np.int32)), "merged flow differs from the dense path"
    assert np.array_equal(mk.view(np.int32), mg[0, ..., 0].cpu().numpy()[ys, xs].view(np.int32)), "matchability differs from the dense path"
    worst = 0.0
    if not onlyCoarse:
        for i in np.unique(hk):
            r = G.compose_fine_ref(flow[i], match[i, 0], match[i, 1], G.warp_grid_f32(Hs[i:i + 1], Hd, Wd)[0], Hd, Wd)
            sel = hk == i
            y, x = ys[sel], xs[sel]
            worst = max(worst, G.check(fk[sel], np.clip(r["flow12"][y, x], -1, 1), r["a_flow12"][y, x], "flow12 of hypothesis %d" % i))
            dd = r["decided"][y, x]
            worst = max(worst, G.check(mk[sel][dd], (r["match"] * r["inside"])[y, x][dd], (r["a_match"] * r["inside"])[y, x][dd],
                                       "match of hypothesis %d" % i))
    kf = [k[ok, c].astype(np.float32) for c in range(4)]
    cnt = counts.reshape(-1, nT + 1)
    for s in range(max(slots) + 1):
        exp_c, exp_n = np.zeros(nT), 0
        for q in [q for q in range(J) if slots[q] == s]:
            c, nb = rf.results.alignment_error(Itw, Ith, wA, hA, *kf, fg, _binary(fg, mg, mth[q]), pg)
            exp_c, exp_n = exp_c + c, exp_n + nb
        assert np.array_equal(cnt[s, :nT], exp_c) and cnt[s, nT] == exp_n, ("row %d" % s, cnt[s].tolist(), exp_c.tolist(), exp_n)
    wins = np.bincount(hk, minlength=nH)
    return worst, "nH %d%s th %.2f mth %s: winners %s, %d keypoints (%d out of range), scored %s, error word %s" % (
        nH, " onlyCoarse" if onlyCoarse else "", th, mth, wins.tolist(), n, int((~ok).sum()), cnt[:, nT].tolist(),
        "pair %d" % want_err if want_err != C.NO_ERROR else "untouched"), "map %dx%d target %dx%d" % (Hd, Wd, Ith, Itw)


CHECKS = {"_resize_u8": check_resize, "bytescale_mask_u8": check_bytescale, "imresize_keep": check_imresize_keep, "preproc_u8": check_preproc,
          "l2norm": check_l2norm, "l2norm_planes": check_l2norm_planes, "corr_mutual_nn": check_corr_mutual_nn,
          "corr_mutual_nn_presplit": check_corr_mutual_nn_presplit, "build_matches": check_build_matches, "ransac_homography": check_ransac,
          "warp_grid": check_warp_grid, "grid_sample": check_grid_sample, "upsample_bilinear": check_upsample, "compose_fine": check_compose_fine,
          "corr_neigh": check_corr_neigh, "corr_neigh_pair": check_corr_neigh_pair, "corr_neigh_pair_split": check_corr_neigh_pair_split,
          "softmax_flow": check_softmax_flow, "sigmoid": check_sigmoid, "remove_small_cc": check_remove_small_cc,
          "kitti_region_step": check_kitti_region_step, "fill_nearest_matched": check_fill_nearest, "warp_sample_u8": check_warp_sample,
          "affine_sample_u8": check_affine_sample, "val_keypoints": check_val_keypoints, "corr_keypoints": check_corr_keypoints}


def test_every_spied_op_has_a_check():
    assert set(CHECKS) == set(SPIED)


@pytest.mark.parametrize("name", sorted(SPIED))
def test_recorded_calls_vs_reference(rf, recorded, name):
    calls = recorded.get(name, [])
    assert calls, "%s: no call recorded; the workloads do not reach it" % name
    worst = 0.0
    for i, call in enumerate(calls):
        try:
            ratio, variant, shapes = CHECKS[name](rf, call)
        except AssertionError as e:
            raise AssertionError("%s call %d (%s): %s" % (name, i, call["where"], e)) from None
        worst = max(worst, ratio)
        print("%s [%s] %s: %s, error / allowance %.3g" % (name, call["where"], shapes, variant, ratio))
    print("%s: %d recorded calls, worst error / allowance %.3g" % (name, len(calls), worst))


# ------------------------------------------------------------------ each new check rejects a doctored record
def _copy(v):
    if isinstance(v, dict):
        return {k: _copy(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_copy(x) for x in v]
    return v.clone() if isinstance(v, torch.Tensor) else v


def _byte_up(rf, call):
    t = T(call["out"]).view(-1)
    t[int(torch.nonzero(t < 255)[0, 0])] += 1


def _affine_off(rf, call):
    _, _, allow = affine_ref(call)
    c, y, x = np.unravel_index(int(np.argmax(allow)), allow.shape)
    T(call["out"])[y * int(call["args"]["w"]) + x, c] += float(4 * allow[c, y, x])


def _count_up(rf, call):
    T(call["after"]["counts"]).view(-1)[0] += 1


def _val_err_cleared(rf, call):
    T(call["after"]["counts"])[-1] = rf.validation.NO_ERROR


def _corr_err_cleared(rf, call):
    T(call["after"]["err"])[0] = rf.corr_results.NO_ERROR


DOCTORED = {"warp_sample_u8 byte": ("warp_sample_u8", _byte_up), "affine_sample_u8 element": ("affine_sample_u8", _affine_off),
            "val_keypoints count": ("val_keypoints", _count_up), "val_keypoints error word": ("val_keypoints", _val_err_cleared),
            "corr_keypoints count": ("corr_keypoints", _count_up), "corr_keypoints error word": ("corr_keypoints", _corr_err_cleared)}


@pytest.mark.parametrize("case", sorted(DOCTORED))
def test_check_rejects_a_doctored_record(rf, recorded, case):
    """One recorded call, copied and edited on the host (an output byte + 1, an element moved by 4x its allowance, a count
    + 1, the error word cleared), must fail its check; nothing is launched with altered arguments."""
    name, doctor = DOCTORED[case]
    calls = recorded[name]
    if "error word" in case:
        what = "counts" if name == "val_keypoints" else "err"
        calls = [c for c in calls if _err_word(c["after"][what]) != getattr(rf, SPIED[name]).NO_ERROR]
        assert calls, "%s: no recorded call sets the error word" % name
    bad = _copy(calls[0])
    doctor(rf, bad)
    with pytest.raises(AssertionError):
        CHECKS[name](rf, bad)
