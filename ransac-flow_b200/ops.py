"""Functional wrappers over the C ABI: torch CUDA tensors in, torch CUDA tensors out.

PyTorch is plumbing here (device memory, streams); every operation below is one
or two launches of the library's own kernels.  Activations are NHWC fp32
"ragged batches" (`Ragged`): several images of different sizes packed back to
back so that one launch covers the whole 7-scale pyramid + target.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, need_cuda, ptr, stream

ENGINE_FP32 = 0      # exact fp32 FMA (SIMT)
ENGINE_TF32 = 1      # wgmma tensor cores, TF32 operands, fp32 accumulate
ENGINE_F16 = 2       # wgmma tensor cores, fp16 activations + weights in HBM, fp32 accumulate (ResNet-50 trunk)
ENGINE_SPLIT = 4     # wgmma tensor cores, fp16 hi / lo split activations + weights (22 significand bits, 3 MMAs per MAC): fp32-grade


def to_split(x):
    """fp32 [P, C] -> split tensor [2, P, C] fp16 (hi = fp16(x), lo = fp16((x - hi) * 2^11)): the engine-4 layout.  Torch
    elementwise ops: a conversion helper for tests and API edges, not on the pair path."""
    x = x.float().clamp(-65504.0, 65504.0)
    hi = x.to(torch.float16)
    lo = ((x - hi.float()) * 2048.0).to(torch.float16)
    return torch.stack([hi, lo]).contiguous()


def from_split(s):
    """split tensor [2, P, C] -> fp32 [P, C] (exact)."""
    return s[0].float() + s[1].float() * (1.0 / 2048.0)


class Ragged:
    """`data` [sum(H*W), C] fp32 CUDA + list of (H, W)."""

    def __init__(self, data, hw):
        self.data = data
        self.hw = [(int(h), int(w)) for h, w in hw]
        self._c = (C.c_int * (2 * len(self.hw)))(*[v for p in self.hw for v in p])

    @property
    def C(self):
        return self.data.shape[-1]

    @property
    def split(self):
        """True for an engine-4 split tensor ([2, P, C] fp16 planes)."""
        return self.data.dim() == 3

    @property
    def n(self):
        return len(self.hw)

    def offsets(self):
        o = [0]
        for h, w in self.hw:
            o.append(o[-1] + h * w)
        return o

    def image(self, i):
        """(1, C, H, W) view (channels_last memory) of image i - no copy."""
        o = self.offsets()
        h, w = self.hw[i]
        assert not self.split
        return self.data[o[i]:o[i + 1]].view(1, h, w, self.C).permute(0, 3, 1, 2)

    def to_nchw(self):
        """(N, C, H, W) view when all images share one size."""
        h, w = self.hw[0]
        assert all(p == (h, w) for p in self.hw)
        return self.data.view(self.n, h, w, self.C).permute(0, 3, 1, 2)

    @staticmethod
    def from_nchw(x):
        need_cuda(x)
        n, c, h, w = x.shape
        d = x.float().permute(0, 2, 3, 1).contiguous().view(n * h * w, c)
        return Ragged(d, [(h, w)] * n)


def _out_hw(hw, k, stride, pad):
    return [((h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1) for h, w in hw]


def conv2d(x, w_packed, bias, Cout, k, stride, pad, relu, residual=None, engine=ENGINE_FP32, w_tc=None):
    """conv + folded-BN bias (+ residual) (+ ReLU) on a ragged NHWC batch."""
    need_cuda(x.data, w_packed, bias, residual.data if residual is not None else None)
    ohw = _out_hw(x.hw, k, stride, pad)
    if residual is not None:           # the kernels read the residual at the output's pixel and channel offsets
        assert residual.hw == ohw and residual.C == Cout, (residual.hw, residual.C, ohw, Cout)
    if int(engine) == ENGINE_F16:      # x, residual, w_tc fp16 -> y fp16
        assert x.data.dtype == torch.float16 and w_tc is not None and w_tc.dtype == torch.float16
        assert residual is None or residual.data.dtype == torch.float16
    if int(engine) in (ENGINE_SPLIT, ENGINE_SPLIT + 1):      # split x / residual / weights -> split y (engine 5: fp32 y)
        assert x.split and x.data.is_contiguous() and w_tc is not None and w_tc.dim() == 3 and w_tc.dtype == torch.float16
        assert residual is None or (residual.split and residual.data.is_contiguous())
    P_out = sum(h * w for h, w in ohw)
    if int(engine) == ENGINE_SPLIT:
        y = torch.empty((2, P_out, Cout), device=x.data.device, dtype=torch.float16)
    else:
        y = torch.empty((P_out, Cout), device=x.data.device, dtype=torch.float16 if int(engine) == ENGINE_F16 else torch.float32)
    check(lib.rf_conv2d_nhwc(ptr(x.data), x.n, x._c, x.C, ptr(w_packed), ptr(w_tc), ptr(bias),
                             ptr(residual.data) if residual is not None else None,
                             Cout, k, k, stride, pad, int(relu), int(engine), ptr(y), stream()))
    return Ragged(y, ohw)


def conv1x1_dual_split(x1, x2, stride2, w_split, bias, relu):
    """Split engine: y = act(W[:, :C1] x1 + W[:, C1:] x2[::stride2, ::stride2] + bias) in one GEMM (x1, x2, y split ragged
    tensors; w_split [2][Cout][C1 + C2] fp16) - a bottleneck's conv3 fused with its down-sampling branch."""
    need_cuda(x1.data, x2.data, w_split, bias)
    assert x1.split and x2.split and x1.data.is_contiguous() and x2.data.is_contiguous() and x1.n == x2.n
    assert w_split.dim() == 3 and w_split.dtype == torch.float16 and w_split.shape[2] == x1.C + x2.C and w_split.is_contiguous()
    cout = w_split.shape[1]
    y = torch.empty((2, sum(h * w for h, w in x1.hw), cout), device=x1.data.device, dtype=torch.float16)
    check(lib.rf_conv1x1_dual_split(ptr(x1.data), ptr(x2.data), x1.n, x1._c, x2._c, x1.C, x2.C, int(stride2), ptr(w_split), ptr(bias),
                                    cout, int(relu), ptr(y), stream()))
    return Ragged(y, x1.hw)


def maxpool2d(x, k, stride, pad):
    need_cuda(x.data)
    ohw = _out_hw(x.hw, k, stride, pad)
    y = torch.empty((sum(h * w for h, w in ohw), x.C), device=x.data.device, dtype=torch.float32)
    check(lib.rf_maxpool2d_nhwc(ptr(x.data), x.n, x._c, x.C, k, stride, pad, ptr(y), stream()))
    return Ragged(y, ohw)


def blur_downsample(x, stride):
    need_cuda(x.data)
    ohw = _out_hw(x.hw, 3, stride, 1)
    y = torch.empty((sum(h * w for h, w in ohw), x.C), device=x.data.device, dtype=torch.float32)
    check(lib.rf_blur_downsample_nhwc(ptr(x.data), x.n, x._c, x.C, stride, ptr(y), stream()))
    return Ragged(y, ohw)


def l2norm(x2d, mask=None):
    """x2d [P, C] -> x / max(||x||, 1e-12) per row; rows with mask == 0 become zeros."""
    need_cuda(x2d, mask)
    if x2d.dim() == 3:                  # engine-4 output: split planes in, fp32 out
        assert x2d.dtype == torch.float16 and x2d.is_contiguous()
        y = torch.empty(x2d.shape[1:], device=x2d.device, dtype=torch.float32)
        check(lib.rf_l2norm_split_nhwc(ptr(x2d), x2d.shape[1], x2d.shape[2], ptr(mask), ptr(y), None, None, stream()))
        return y
    if x2d.dtype == torch.float16:      # engine-2 trunk output: fp16 in, fp32 out
        y = torch.empty(x2d.shape, device=x2d.device, dtype=torch.float32)
        check(lib.rf_l2norm_f16_nhwc(ptr(x2d), x2d.shape[0], x2d.shape[1], ptr(mask), ptr(y), stream()))
        return y
    y = torch.empty_like(x2d)
    check(lib.rf_l2norm_nhwc(ptr(x2d), x2d.shape[0], x2d.shape[1], ptr(mask), ptr(y), stream()))
    return y


def l2norm_planes(x_split, mask=None):
    """Engine-4 features [2, P, C] -> their L2-normalised rows as fp16 planes [2, P, C] (hi, lo * 2^11): exactly what the
    fp16-split correlation kernel reads, written by the normalisation itself (no fp32 copy, no split pass)."""
    need_cuda(x_split, mask)
    assert x_split.dim() == 3 and x_split.dtype == torch.float16 and x_split.is_contiguous()
    out = torch.empty_like(x_split)
    check(lib.rf_l2norm_split_nhwc(ptr(x_split), x_split.shape[1], x_split.shape[2], ptr(mask), None, ptr(out[0]), ptr(out[1]), stream()))
    return out


def corr_neigh(x, y, k, ldo=None, round_tf32=False):
    """x, y: Ragged with identical (h, w) per image -> Ragged with ``ldo`` (default k*k) channels; channels
    beyond k*k are zeros (ldo = 64 gives the heads a 128-byte aligned K-major operand).  ``round_tf32``: 0 / False =
    plain fp32, 1 / True = fp32 rounded to TF32, 2 = fp16 output (operand of the fp16-engine heads)."""
    need_cuda(x.data, y.data)
    assert x.data.dtype == torch.float32 and y.data.dtype == torch.float32
    h, w = x.hw[0]
    ldo = k * k if ldo is None else int(ldo)
    out = torch.empty((x.data.shape[0], ldo), device=x.data.device, dtype=torch.float16 if int(round_tf32) == 2 else torch.float32)
    check(lib.rf_corr_neigh_nhwc(ptr(x.data), ptr(y.data), x.n, h, w, x.C, k, ldo, int(round_tf32), ptr(out), stream()))
    return Ragged(out, x.hw)


def corr_neigh_pair(x, y, k, ldo=None, round_tf32=False):
    """``corr_neigh(x, y)`` and ``corr_neigh(y, x)`` from ONE launch (each dot product computed once, stored in both
    volumes).  Returns (corr_xy, corr_yx, both): ``both`` is the [2P, ldo] buffer the two halves live in, i.e. the
    two-image batch the matchability head runs on, without a concatenation copy."""
    need_cuda(x.data, y.data)
    assert x.data.dtype == torch.float32 and y.data.dtype == torch.float32 and x.hw == y.hw
    h, w = x.hw[0]
    ldo = k * k if ldo is None else int(ldo)
    P = x.data.shape[0]
    buf = torch.empty((2 * P, ldo), device=x.data.device, dtype=torch.float16 if int(round_tf32) == 2 else torch.float32)
    check(lib.rf_corr_neigh_pair_nhwc(ptr(x.data), ptr(y.data), x.n, h, w, x.C, k, ldo, int(round_tf32), ptr(buf[:P]), ptr(buf[P:]), stream()))
    return Ragged(buf[:P], x.hw), Ragged(buf[P:], x.hw), Ragged(buf, x.hw + x.hw)


def corr_neigh_pair_split(x, y, k, ldo, want_both=True):
    """Engine-4 form: CorrNeigh(x, y) as a split tensor [2, P, ldo] (the flow head's input) and, with ``want_both``, the
    two-image split tensor [2, 2P, ldo] = [CorrNeigh(x, y) ; CorrNeigh(y, x)] of the matchability head, from ONE launch."""
    need_cuda(x.data, y.data)
    assert x.data.dtype == torch.float32 and y.data.dtype == torch.float32 and x.hw == y.hw
    h, w = x.hw[0]
    P = x.data.shape[0]
    c12 = torch.empty((2, P, ldo), device=x.data.device, dtype=torch.float16)
    both = torch.empty((2, 2 * P, ldo), device=x.data.device, dtype=torch.float16) if want_both else None
    check(lib.rf_corr_neigh_pair_split(ptr(x.data), ptr(y.data), x.n, h, w, x.C, k, int(ldo), ptr(c12), ptr(both), stream()))
    return Ragged(c12, x.hw), (Ragged(both, x.hw + x.hw) if want_both else None)


def softmax_flow(logits, k):
    need_cuda(logits.data)
    h, w = logits.hw[0]
    out = torch.empty((logits.n, 2, h, w), device=logits.data.device, dtype=torch.float32)
    check(lib.rf_softmax_flow(ptr(logits.data), logits.n, h, w, k, ptr(out), stream()))
    return out


def sigmoid(x):
    need_cuda(x)
    y = torch.empty_like(x)
    check(lib.rf_sigmoid(ptr(x), x.numel(), ptr(y), stream()))
    return y


def preproc_u8(img_u8, normalize):
    """uint8 [P, 3] CUDA -> fp32 [P, 3] (ToTensor [+ Normalize])."""
    need_cuda(img_u8)
    out = torch.empty(img_u8.shape, device=img_u8.device, dtype=torch.float32)
    check(lib.rf_preproc_u8(ptr(img_u8), img_u8.shape[0], int(normalize), ptr(out), stream()))
    return out


# --------------------------------------------------------------------------- matching / RANSAC
def corr_mutual_nn(featA, featB, precision=0):
    """featA [NA, C], featB [NB, C] (rows = feature vectors) -> idx1, idx2 (int64 CUDA, capacity min(NA,NB)), count (int32 CUDA)."""
    need_cuda(featA, featB)
    NA, Cc = featA.shape
    NB = featB.shape[0]
    cap = max(1, min(NA, NB))
    dev = featA.device
    idx1 = torch.empty(cap, device=dev, dtype=torch.int64)
    idx2 = torch.empty(cap, device=dev, dtype=torch.int64)
    count = torch.zeros(1, device=dev, dtype=torch.int32)
    wsz = lib.rf_corr_mutual_nn_workspace(NA, NB, Cc, int(precision))
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_corr_mutual_nn(ptr(featA), NA, ptr(featB), NB, Cc, ptr(idx1), ptr(idx2), ptr(count),
                                ptr(ws), wsz, int(precision), stream()))
    return idx1, idx2, count


SAMPLES_INDEX, SAMPLES_MOD, SAMPLES_PHILOX64 = 0, 1, 2


def philox_words(nbIter, nbPoint, device, generator=None, out=None):
    """(nbIter, nbPoint) full-range 64-bit words from torch's CUDA generator: element i is (x << 32) | y of the curand4 call
    whose x torch.randint(M, (nbIter, nbPoint), device='cuda') reduces modulo M from the same generator state (and the
    generator advances by the same offset).  With ``SAMPLES_PHILOX64`` the RANSAC kernel therefore sees the reference's
    seeded sample stream (utils/outil.py:120) with M read on the device; the draw is graph-capturable.  ``generator``: a CUDA
    generator of its own instead of torch's default one.  ``out``: a contiguous (nbIter, nbPoint) int64 tensor to draw into
    (e.g. one table of a stack of tables)."""
    assert nbIter * nbPoint <= 256 * 1024, "beyond this size ATen maps several elements to one Philox subsequence"
    if out is None:
        out = torch.empty((nbIter, nbPoint), dtype=torch.int64, device=device)
    assert tuple(out.shape) == (nbIter, nbPoint) and out.dtype == torch.int64 and out.is_contiguous()
    return out.random_(-2 ** 63, None, generator=generator)


def corr_mutual_nn_presplit(A_hi, A_lo, B_hi, B_lo):
    """``corr_mutual_nn`` at precision 2 on operands that are already fp16 hi / lo planes ([N, C] each, contiguous)."""
    need_cuda(A_hi, A_lo, B_hi, B_lo)
    NA, Cc = A_hi.shape
    NB = B_hi.shape[0]
    for t in (A_hi, A_lo, B_hi, B_lo):
        assert t.dtype == torch.float16 and t.is_contiguous() and t.shape[1] == Cc
    cap = max(1, min(NA, NB))
    dev = A_hi.device
    idx1 = torch.empty(cap, device=dev, dtype=torch.int64)
    idx2 = torch.empty(cap, device=dev, dtype=torch.int64)
    count = torch.zeros(1, device=dev, dtype=torch.int32)
    wsz = lib.rf_corr_mutual_nn_presplit_workspace(NA, NB)
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_corr_mutual_nn_presplit(ptr(A_hi), ptr(A_lo), NA, ptr(B_hi), ptr(B_lo), NB, Cc, ptr(idx1), ptr(idx2), ptr(count), ptr(ws), wsz, stream()))
    return idx1, idx2, count


def ransac_homography(match1, match2, samples, tolerance, chunk=100, M_dev=None, sample_mode=None):
    """Returns device tensors (H [9] f32, nbInlier [1] i64, mask [M] u8, status [1] i32).  ``sample_mode``: SAMPLES_INDEX
    (default without ``M_dev``), SAMPLES_MOD (default with ``M_dev``: ``samples % M`` on the device) or SAMPLES_PHILOX64."""
    if sample_mode is None:
        sample_mode = SAMPLES_INDEX if M_dev is None else SAMPLES_MOD
    need_cuda(match1, match2, samples, M_dev)
    M = match1.shape[0]
    nbIter = samples.shape[0]
    dev = match1.device
    H = torch.empty(9, device=dev, dtype=torch.float32)
    nb = torch.empty(1, device=dev, dtype=torch.int64)
    mask = torch.empty(max(M, 1), device=dev, dtype=torch.uint8)
    status = torch.empty(1, device=dev, dtype=torch.int32)
    wsz = lib.rf_ransac_workspace(nbIter)
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_ransac_homography(ptr(match1), ptr(match2), M, ptr(M_dev), ptr(samples), int(sample_mode), nbIter, float(tolerance), int(chunk),
                                   ptr(H), ptr(nb), ptr(mask), ptr(status), ptr(ws), wsz, stream()))
    return H, nb, mask[:M], status


def homography_dlt(X, Y):
    need_cuda(X, Y)
    N = X.shape[0]
    H = torch.empty((N, 3, 3), device=X.device, dtype=torch.float32)
    check(lib.rf_homography_dlt(ptr(X), ptr(Y), N, ptr(H), stream()))
    return H


def prediction(match1, match2, H):
    need_cuda(match1, match2, H)
    N, M = H.shape[0], match1.shape[0]
    err = torch.empty((N, M), device=H.device, dtype=torch.float32)
    check(lib.rf_prediction(ptr(match1), ptr(match2), M, ptr(H), N, ptr(err), stream()))
    return err


def build_matches(idx1, idx2, count, W1, H1, W2, H2, valid16=None):
    need_cuda(idx1, idx2, count, W1, H1, W2, H2, valid16)
    cap = idx1.shape[0]
    dev = idx1.device
    m1 = torch.empty((cap, 3), device=dev, dtype=torch.float32)
    m2 = torch.empty((cap, 3), device=dev, dtype=torch.float32)
    kept = torch.empty(cap, device=dev, dtype=torch.int64)
    cnt = torch.zeros(1, device=dev, dtype=torch.int32)
    check(lib.rf_build_matches(ptr(idx1), ptr(idx2), ptr(count), ptr(W1), ptr(H1), ptr(W2), ptr(H2), ptr(valid16),
                               ptr(m1), ptr(m2), ptr(kept), ptr(cnt), cap, stream()))
    return m1, m2, kept, cnt


# --------------------------------------------------------------------------- YFCC pose
POSE_OK, POSE_TOO_FEW, POSE_NO_MODEL, POSE_NO_POSE = 0, 1, 2, 3


class PoseRecord(C.Structure):
    """Mirror of rf_pose_record_t (include/ransacflow_b200.h)."""
    _fields_ = [("status", C.c_int), ("n_points", C.c_int), ("niters", C.c_int), ("best_iter", C.c_int), ("best_cand", C.c_int),
                ("ransac_count", C.c_int), ("n_E", C.c_int), ("pose_count", C.c_int), ("pose_cand", C.c_int), ("pose_index", C.c_int),
                ("pose_counts", C.c_int * 40), ("E", C.c_double * 90), ("poses", C.c_double * 480), ("R", C.c_double * 9),
                ("t", C.c_double * 3)]


def pose_record(device):
    """A device buffer for one rf_pose_record_t."""
    return torch.zeros(C.sizeof(PoseRecord), device=device, dtype=torch.uint8)


def read_pose_record(rec):
    """The record as a dict of host values / numpy arrays (one device-to-host copy)."""
    r = PoseRecord.from_buffer_copy(rec.cpu().numpy().tobytes())
    nE = max(r.n_E, 0)
    return dict(status=r.status, n_points=r.n_points, niters=r.niters, best=(r.best_iter, r.best_cand), ransac_count=r.ransac_count,
                n_E=r.n_E, pose_count=r.pose_count, pose=(r.pose_cand, r.pose_index),
                pose_counts=np.array(r.pose_counts, dtype=np.int64).reshape(10, 4)[:nE],
                E=np.array(r.E).reshape(10, 3, 3)[:nE], poses=np.array(r.poses).reshape(10, 4, 3, 4)[:nE],
                R=np.array(r.R).reshape(3, 3), t=np.array(r.t).reshape(3, 1))


def record_E(rec):
    """The E field of a record buffer as a writable fp64 view [10][9] (tests supply their own E through it)."""
    off = PoseRecord.E.offset
    return rec[off:off + 90 * 8].view(torch.float64).view(10, 9)


def yfcc_matches(flow, mask, angle, sizeA, sizeB, norm1, norm2):
    """evaluation/evalYFCC/getResults.py:53-71 matches_from_flow + :29-50 norm_kp on the device: flow (H,W,2) fp32, mask (H,W)
    (non-zero = matched) -> (pts1, pts2 [H*W][2] fp64 capacity, N [1] int32 on the device).  ``norm1`` / ``norm2`` are norm_kp's
    (cx, cy, fx, fy) of each image.  A mask whose shape is not the rotated target grid's raises IndexError, as numpy does."""
    need_cuda(flow, mask)
    wA, hA = int(sizeA[0]), int(sizeA[1])
    wB, hB = int(sizeB[0]), int(sizeB[1])
    k = (int(angle) // 90) % 4
    H, W = int(mask.shape[0]), int(mask.shape[1])
    if mask.dim() != 2 or (H, W) != ((hB, wB) if k % 2 == 0 else (wB, hB)):
        raise IndexError("boolean index did not match indexed array: mask %s vs rotated grid %s"
                         % (tuple(mask.shape), (hB, wB) if k % 2 == 0 else (wB, hB)))
    assert tuple(flow.shape) == (H, W, 2), flow.shape
    flow = flow.float().contiguous()
    mask = (mask != 0).to(torch.uint8).contiguous() if mask.dtype != torch.uint8 else mask.contiguous()
    dev = flow.device
    cap = max(H * W, 1)
    pts1 = torch.empty((cap, 2), device=dev, dtype=torch.float64)
    pts2 = torch.empty((cap, 2), device=dev, dtype=torch.float64)
    N = torch.empty(1, device=dev, dtype=torch.int32)
    wsz = lib.rf_yfcc_matches_workspace(H, W)
    ws = torch.empty(max(wsz, 1), device=dev, dtype=torch.uint8)
    n1 = (C.c_double * 4)(*[float(v) for v in norm1])
    n2 = (C.c_double * 4)(*[float(v) for v in norm2])
    check(lib.rf_yfcc_matches(ptr(flow), ptr(mask), H, W, k, wB, hB, wA, hA, n1, n2, ptr(pts1), ptr(pts2), ptr(N), ptr(ws), wsz,
                              stream()))
    return pts1, pts2, N


def essential_ransac(pts1, pts2, N, threshold=0.0005, rec=None):
    """cv2.findEssentialMat(pts1[:N], pts2[:N], method=cv2.RANSAC, threshold) on the device (N: [1] int32 device count):
    -> (record buffer, mask [capacity] u8).  Read the record with ``read_pose_record``."""
    need_cuda(pts1, pts2, N)
    dev = pts1.device
    cap = int(pts1.shape[0])
    rec = pose_record(dev) if rec is None else rec
    mask = torch.zeros(max(cap, 1), device=dev, dtype=torch.uint8)
    wsz = lib.rf_essential_ransac_workspace(cap)
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_essential_ransac(ptr(pts1), ptr(pts2), cap, ptr(N), float(threshold), ptr(rec), ptr(mask), ptr(ws), wsz, stream()))
    return rec, mask


def recover_pose(pts1, pts2, mask, rec):
    """cv2.recoverPose(E, pts1, pts2, mask=mask) over the stacked E of ``rec`` with evalYFCC's loop (getResults.py:96-104):
    fills R, t and the count in the record; -> (mask_out [capacity] u8, cheirality bits [capacity] int64)."""
    need_cuda(pts1, pts2, mask, rec)
    dev = pts1.device
    cap = int(pts1.shape[0])
    out = torch.zeros(max(cap, 1), device=dev, dtype=torch.uint8)
    wsz = lib.rf_recover_pose_workspace(cap)
    ws = torch.zeros(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_recover_pose(ptr(pts1), ptr(pts2), cap, ptr(mask), ptr(rec), ptr(out), ptr(ws), wsz, stream()))
    return out, ws[:8 * cap].view(torch.int64)


def essential_samples(N):
    """The [1000][5] subset table of cv2.findEssentialMat's RANSAC for N = N[0] (device int32) points."""
    need_cuda(N)
    idx = torch.zeros((1000, 5), device=N.device, dtype=torch.int32)
    check(lib.rf_essential_samples(ptr(N), ptr(idx), stream()))
    return idx


def essential_five_point(pts1, pts2, idx):
    """Five-point solutions of the subsets idx [S][5]: (E [S][10][9] fp64, count [S] int32)."""
    need_cuda(pts1, pts2, idx)
    S = int(idx.shape[0])
    E = torch.full((max(S, 1), 10, 9), float("nan"), device=pts1.device, dtype=torch.float64)
    n = torch.full((max(S, 1),), -1, device=pts1.device, dtype=torch.int32)
    check(lib.rf_essential_five_point(ptr(pts1), ptr(pts2), ptr(idx.int().contiguous()), S, ptr(E), ptr(n), stream()))
    return E[:S], n[:S]


def essential_score(pts1, pts2, E, threshold=0.0005, want_err=False):
    """Sampson inlier counts of models E [M][9] (M <= 640) over all rows of pts1 / pts2 (and the fp32 errors [M][N])."""
    need_cuda(pts1, pts2, E)
    N, M = int(pts1.shape[0]), int(E.shape[0])
    counts = torch.zeros(max(M, 1), device=E.device, dtype=torch.int32)
    err = torch.full((M, N), float("nan"), device=E.device, dtype=torch.float32) if want_err else None
    check(lib.rf_essential_score(ptr(pts1.contiguous()), ptr(pts2.contiguous()), N, ptr(E.contiguous()), M, float(threshold),
                                 ptr(counts), ptr(err), stream()))
    return counts[:M], err


def fundamental_8point(pts1, pts2, N, rec=None):
    """cv2.findFundamentalMat(pts1[:N], pts2[:N], method=cv2.FM_8POINT) on the device (N: [1] int32 device count), the points
    cast to fp32 first as cv2 does: -> (record buffer, mask [capacity] u8, all ones over the first N rows when N >= 7).  The
    record's E holds F (1 candidate, or 1..3 when N == 7); ``recover_pose`` runs on it as on essential_ransac's record."""
    need_cuda(pts1, pts2, N)
    dev = pts1.device
    cap = int(pts1.shape[0])
    rec = pose_record(dev) if rec is None else rec
    mask = torch.zeros(max(cap, 1), device=dev, dtype=torch.uint8)
    wsz = lib.rf_fundamental_8point_workspace(cap)
    ws = torch.empty(wsz, device=dev, dtype=torch.uint8)
    check(lib.rf_fundamental_8point(ptr(pts1), ptr(pts2), cap, ptr(N), ptr(rec), ptr(mask), ptr(ws), wsz, stream()))
    return rec, mask


def fundamental_moments(pts1, pts2, N):
    """The reductions of fundamental_8point alone (N = N[0] >= 1): [51] fp64 = (m1c, m2c, scale1, scale2, A's upper triangle
    row by row) over the first N rows."""
    need_cuda(pts1, pts2, N)
    cap = int(pts1.shape[0])
    out = torch.full((51,), float("nan"), device=pts1.device, dtype=torch.float64)
    wsz = lib.rf_fundamental_8point_workspace(cap)
    ws = torch.empty(wsz, device=pts1.device, dtype=torch.uint8)
    check(lib.rf_fundamental_moments(ptr(pts1), ptr(pts2), cap, ptr(N), ptr(out), ptr(ws), wsz, stream()))
    return out


# --------------------------------------------------------------------------- warp
def warp_grid(H, h, w):
    need_cuda(H)
    H = H.reshape(-1, 9).contiguous().float()
    out = torch.empty((H.shape[0], h, w, 2), device=H.device, dtype=torch.float32)
    check(lib.rf_warp_grid(ptr(H), H.shape[0], h, w, ptr(out), stream()))
    return out


def grid_sample(inp, grid, align_corners=False):
    """F.grid_sample(inp, grid) bilinear / zeros.  Output has the memory format of the input."""
    need_cuda(inp, grid)
    inp = inp if inp.dtype == torch.float32 else inp.float()
    N, Cc, Hin, Win = inp.shape
    if grid.dim() != 4 or grid.shape[0] != N or grid.shape[3] != 2:
        raise ValueError("grid_sample: grid must be (N, Hout, Wout, 2) with the input's N = %d, got %s" % (N, tuple(grid.shape)))
    grid = grid.contiguous().float()
    Hout, Wout = grid.shape[1], grid.shape[2]
    if inp.stride(1) == 1 and Cc > 1:
        out = torch.empty((N, Hout, Wout, Cc), device=inp.device, dtype=torch.float32).permute(0, 3, 1, 2)
    else:
        out = torch.empty((N, Cc, Hout, Wout), device=inp.device, dtype=torch.float32)
    is_ = (C.c_longlong * 4)(*inp.stride())
    os_ = (C.c_longlong * 4)(*out.stride())
    check(lib.rf_grid_sample(ptr(inp), N, Cc, Hin, Win, is_, ptr(grid), Hout, Wout, int(align_corners), ptr(out), os_, stream()))
    return out


def upsample_bilinear(x, size):
    need_cuda(x)
    x = x.contiguous().float()
    N, Cc, h, w = x.shape
    out = torch.empty((N, Cc, size[0], size[1]), device=x.device, dtype=torch.float32)
    check(lib.rf_upsample_bilinear(ptr(x), N * Cc, h, w, size[0], size[1], ptr(out), stream()))
    return out


def compose_fine(flowDown8, match12, match21, coarse, clamp=True, align_corners=False, want_match=True, want_flowUp=False, size=None):
    """Fused tail of PredFlowMask.  flowDown8 (1,2,h8,w8); match12/match21 (1,1,h8,w8) or None; coarse (1,Hc,Wc,2).
    ``size`` = (H, W) of the outputs when it differs from the coarse grid's (the KITTI two-level flow)."""
    need_cuda(flowDown8, match12, match21, coarse)
    if flowDown8.dim() != 4 or flowDown8.shape[:2] != (1, 2):
        raise ValueError("compose_fine: flowDown8 must be (1, 2, h8, w8), got %s" % (tuple(flowDown8.shape),))
    _, _, h8, w8 = flowDown8.shape
    for name, m in (("match12", match12), ("match21", match21)):
        if m is not None and tuple(m.shape) != (1, 1, h8, w8):
            raise ValueError("compose_fine: %s must be (1, 1, %d, %d), got %s" % (name, h8, w8, tuple(m.shape)))
    if coarse.dim() != 4 or coarse.shape[0] != 1 or coarse.shape[3] != 2:
        raise ValueError("compose_fine: coarse must be (1, Hc, Wc, 2), got %s" % (tuple(coarse.shape),))
    _, Hc, Wc, _ = coarse.shape
    H, W = (Hc, Wc) if size is None else (int(size[0]), int(size[1]))
    dev = coarse.device
    flow12 = torch.empty((1, H, W, 2), device=dev, dtype=torch.float32)
    match = torch.empty((1, 1, H, W), device=dev, dtype=torch.float32) if (want_match and match12 is not None) else None
    flowUp = torch.empty((1, H, W, 2), device=dev, dtype=torch.float32) if want_flowUp else None
    check(lib.rf_compose_fine_ex(ptr(flowDown8.contiguous()), ptr(match12.contiguous()) if match12 is not None else None,
                                 ptr(match21.contiguous()) if match21 is not None else None, h8, w8, ptr(coarse.contiguous()),
                                 Hc, Wc, H, W, int(clamp), int(align_corners), ptr(flow12), ptr(match), ptr(flowUp), stream()))
    return flow12, match, flowUp


def remove_small_cc(match, match_th, cc_th):
    """evaluation/evalKITTI/evaluation.py:85-100 on the device, in place: match (N,1,H,W) / (N,H,W) / (H,W) fp32 CUDA.
    Returns ``match``."""
    need_cuda(match)
    assert match.dtype == torch.float32 and match.is_contiguous()
    H, W = int(match.shape[-2]), int(match.shape[-1])
    N = match.numel() // max(1, H * W)
    wsz = lib.rf_remove_small_cc_workspace(H, W)
    ws = torch.empty(wsz, device=match.device, dtype=torch.uint8)
    check(lib.rf_remove_small_cc(ptr(match), N, H, W, float(match_th), float(cc_th), ptr(ws), wsz, stream()))
    return match


def kitti_region_step(match, Mask, bg, fgMask, status, alive, first, cmin, rec=None):
    """One hypothesis of evaluation/evalKITTI/evaluation.py:316-326 on the device (``rf_kitti_region_step``): ``match``, ``bg``
    (H, W) fp32; ``Mask`` / ``fgMask`` (H, W) fp32 updated in place where the hypothesis is accepted; ``status`` the RANSAC
    status (int32 [1]); ``alive`` an int32 [1] flag, updated in place; ``cmin`` from ``pipeline.kitti_region_cmin``.  Returns
    ``rec`` (int32 [2] = {alive, count}; allocated when None).  Nothing is read back: graph-capturable."""
    need_cuda(match, Mask, bg, fgMask, status, alive, rec)
    H, W = int(match.shape[-2]), int(match.shape[-1])
    for name, t in (("match", match), ("Mask", Mask), ("bg", bg), ("fgMask", fgMask)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != H * W:
            raise ValueError("kitti_region_step: %s must be a contiguous fp32 (%d, %d) map" % (name, H, W))
    for name, t in (("status", status), ("alive", alive)):
        if t.dtype != torch.int32 or t.numel() != 1:
            raise ValueError("kitti_region_step: %s must be one int32" % name)
    if rec is None:
        rec = torch.empty(2, device=match.device, dtype=torch.int32)
    wsz = lib.rf_kitti_region_step_workspace(H, W)
    ws = torch.empty(wsz, device=match.device, dtype=torch.uint8)
    check(lib.rf_kitti_region_step(ptr(match), ptr(Mask), ptr(bg), ptr(fgMask), H, W, ptr(status), ptr(alive), int(bool(first)), int(cmin),
                                   ptr(rec), ptr(ws), wsz, stream()))
    return rec


def fill_nearest_matched(flow, matched, want_index=False):
    """evaluation/evalKITTI/getResults.py:87-93 on the device: flow (1,H,W,2) fp32, matched (H,W) / (1,H,W,1) bool ->
    flow with every unmatched pixel replaced by the flow of its nearest matched pixel (exact EDT) [, (H,W,2) int32 indices]."""
    need_cuda(flow, matched)
    flow = flow.contiguous().float()
    H, W = int(flow.shape[1]), int(flow.shape[2])
    m = matched.reshape(H, W).to(torch.uint8).contiguous()
    out = torch.empty_like(flow)
    idx = torch.empty((H, W, 2), device=flow.device, dtype=torch.int32) if want_index else None
    wsz = lib.rf_fill_nearest_matched_workspace(H, W)
    ws = torch.empty(wsz, device=flow.device, dtype=torch.uint8)
    check(lib.rf_fill_nearest_matched(ptr(flow), ptr(m), H, W, ptr(out), ptr(idx), ptr(ws), wsz, stream()))
    return (out, idx) if want_index else out


# --------------------------------------------------------------------------- PIL LANCZOS / BILINEAR on device
_coeff_cache = {}


def resample_coeffs(in_size, out_size, device, fn, non_blocking=False):
    """PIL's 8bpc resampling tables (``fn``: rf_lanczos_coeffs_host or rf_bilinear_coeffs_host) as device tensors, cached.
    ``non_blocking``: the tables go up from pinned memory on the current stream, without a host synchronisation.  Such
    tables are ordered on that stream only, so they are cached for that stream alone: blocking callers and other streams
    never see them."""
    key = (in_size, out_size, str(device), fn)
    if non_blocking:
        key += (torch.cuda.current_stream(device).cuda_stream,)
    if key not in _coeff_cache:
        ks = C.c_int(0)
        check(getattr(lib, fn)(in_size, out_size, None, None, 0, C.byref(ks)))
        bounds = np.zeros(2 * out_size, dtype=np.int32)
        kk = np.zeros(ks.value * out_size, dtype=np.int32)
        check(getattr(lib, fn)(in_size, out_size, bounds.ctypes.data_as(C.c_void_p), kk.ctypes.data_as(C.c_void_p), kk.size, C.byref(ks)))
        up = (lambda a: torch.from_numpy(a).pin_memory().to(device, non_blocking=True)) if non_blocking else (lambda a: torch.from_numpy(a).to(device))
        _coeff_cache[key] = (up(bounds), up(kk), ks.value)
    return _coeff_cache[key]


def resize_lanczos_u8(img, out_w, out_h, non_blocking=False):
    """PIL ``Image.resize((out_w, out_h), LANCZOS)`` on a uint8 [H, W, 3] CUDA tensor (bit-exact).  ``non_blocking``: see
    ``resample_coeffs``."""
    return _resize_u8(img, out_w, out_h, "rf_lanczos_coeffs_host", non_blocking)


def resize_bilinear_u8(img, out_w, out_h):
    """PIL ``Image.resize((out_w, out_h), BILINEAR)`` on a uint8 [H, W, 3] CUDA tensor (bit-exact)."""
    return _resize_u8(img, out_w, out_h, "rf_bilinear_coeffs_host")


def _resize_u8(img, out_w, out_h, fn, non_blocking=False):
    """PIL's two-pass 8bpc resampling (horizontal, then vertical) with the tables ``fn`` builds."""
    need_cuda(img)
    H, W, ch = img.shape
    cur = img.contiguous()
    if out_w != W:
        b, k, ks = resample_coeffs(W, out_w, img.device, fn, non_blocking)
        nxt = torch.empty((H, out_w, ch), device=img.device, dtype=torch.uint8)
        check(lib.rf_resample_u8(ptr(cur), H, W, ch, 1, ptr(b), ptr(k), ks, out_w, ptr(nxt), stream()))
        cur, W = nxt, out_w
    if out_h != H:
        b, k, ks = resample_coeffs(H, out_h, img.device, fn, non_blocking)
        nxt = torch.empty((out_h, W, ch), device=img.device, dtype=torch.uint8)
        check(lib.rf_resample_u8(ptr(cur), H, W, ch, 0, ptr(b), ptr(k), ks, out_h, ptr(nxt), stream()))
        cur = nxt
    return cur


# --------------------------------------------------------------------------- the drivers' background-mask resize
def bytescale_mask_u8(m, rot=0):
    """``scipy.misc.bytescale(np.rot90(m, rot))`` of a float32 (H, W) CUDA map, as SciPy 1.2's ``imresize`` (``dropin.imresize``)
    byte-scales it: uint8 (H, W), or (W, H) for an odd ``rot``.  Min and max are reduced on the device (graph-capturable)."""
    need_cuda(m)
    assert m.dim() == 2 and m.dtype == torch.float32, (m.dim(), m.dtype)
    m = m.contiguous()
    H, W = int(m.shape[0]), int(m.shape[1])
    k = int(rot) % 4
    out = torch.empty((W, H) if k % 2 else (H, W), device=m.device, dtype=torch.uint8)
    wsz = lib.rf_bytescale_mask_u8_workspace(H, W)
    ws = torch.empty(wsz, device=m.device, dtype=torch.uint8)
    check(lib.rf_bytescale_mask_u8(ptr(m), H, W, k, ptr(out), ptr(ws), wsz, stream()))
    return out


def imresize_keep(m, h, w, rot=0):
    """``imresize(np.rot90(m, rot), (h, w)) < 128`` as a bool (h, w) CUDA tensor (True = kept, not background).  ``m``: a float32
    (H, W) map, CUDA or host (copied to the current device)."""
    if not torch.is_tensor(m):
        m = torch.from_numpy(np.ascontiguousarray(m, dtype=np.float32))
    if not m.is_cuda:
        m = m.to(device=torch.device("cuda", torch.cuda.current_device()), dtype=torch.float32)
    u8 = bytescale_mask_u8(m, rot)
    r = _resize_u8(u8.view(u8.shape[0], u8.shape[1], 1), int(w), int(h), "rf_bilinear_coeffs_host")     # PIL BILINEAR, mode L
    return (r < 128).view(int(h), int(w))


def imresize_mask(m, h, w, rot=0):
    """``(dropin.imresize(np.rot90(m, rot), (h, w)) < 128).astype(np.float32)`` on the device: a float32 (h, w) CUDA tensor,
    1 = kept.  The background map of evaluation/evalHpatch/evaluation.py:180, evalCorr:187, evalYFCC:200/212, evalKITTI:248:
    byte-scaling (``rf_bytescale_mask_u8``), then PIL's BILINEAR passes (``rf_resample_u8``, skipped where a side keeps its
    size), then the comparison.  No host read: it can be captured in a CUDA graph once its resampling tables exist."""
    return imresize_keep(m, h, w, rot).float()
