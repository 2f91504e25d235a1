"""Coarse-aligned training pairs (README §4.1, and the pair step of §4.3 "Fine-tuning on your own dataset"):
train/generate_coarse_aligned_pair.ipynb on the device, for every pair of a dataset.

  cell 7  : ``outil.resizeImg`` of the ORIGINAL source to min side minSize // 2, minSize, minSize * 2 and of the target to
            minSize (PIL LANCZOS, ``round(w / ratio / 16) * 16`` with Python's half-to-even ``round``: ``pipeline.fine_sizes``,
            not CoarseAlign's ``ResizeMinSize``); ImageNet ``ToTensor + Normalize``, ResNet-50 conv1..layer3, ``F.normalize``
  cell 9  : the source rows concatenated Down2, 1, Up2 (ascending size: arg-max ties go to the smallest index, so the order
            is part of the result), ``mutualMatching(featpMultiScale, feat2T)``, ``match1`` = the TARGET's (H2, W2, 1),
            ``match2`` = the SOURCE's (H1, W1, 1)
  cell 11 : ``outil.RANSAC(nbIter, match1, match2, tolerance, 4, Homography)``
  cell 13 : ``len(match1Inlier) > 50`` keeps the pair; the grid of ``HomographyWarper(h1, w1).warp_grid(bestParam)`` (on the
            SOURCE's size) samples the TARGET (``ToTensor`` only), and ``ToPILImage`` truncates ``x * 255`` to uint8

The keep rule is the notebook's: RANSAC's third return value is the bool ``isInlier`` array of length M, not the inliers, so
a pair is kept when RANSAC returned a model and M > 50, whatever its inlier count (``nbInlier`` is reported beside it).

The one deliberate departure: the notebook raises on some pairs (M = 0: ``torch.randint``'s RuntimeError; 1 <= M <= 3, or a
RANSAC whose remainder chunk finds no model: the TypeError of utils/outil.py:162).  A dataset generator must not stop on one
bad pair, so such pairs are not kept and their record carries the RANSAC status and M (``notebook_exception``).

Steps 6 and 7 (grid, sampling, truncation) are one kernel, ``rf_warp_sample_u8``, which reads H from device memory.
"""
import numpy as np
import torch

from . import ops, outil, pipeline
from ._lib import check, lib, need_cuda, ptr, stream
from .coarseAlignFeatMatch import ResNet50Conv4, _CoarseAlignBase, conv4_features, ransac_device, resnet50_state

KEEP_MIN_MATCHES = 50           # cell 13: len(match1Inlier) > 50


# --------------------------------------------------------------------------- kernel entry
def warp_sample_u8(H, src, h, w, align_corners=False, out=None):
    """``(255 * F.grid_sample(ToTensor(src), warp_grid(H, h, w))).byte()`` in one kernel: H a 9-float CUDA tensor (read on the
    device), ``src`` a uint8 (Hin, Win, 3) CUDA image.  Returns the uint8 (h, w, 3) CUDA image (into ``out`` when given)."""
    need_cuda(H, src, out)
    if H.dtype != torch.float32 or H.numel() != 9 or not H.is_contiguous():
        raise ValueError("warp_sample_u8: H must be 9 contiguous float32 values")
    if src.dtype != torch.uint8 or src.dim() != 3 or src.shape[2] != 3 or not src.is_contiguous():
        raise ValueError("warp_sample_u8: src must be a contiguous uint8 (H, W, 3) image")
    if out is None:
        out = torch.empty((h, w, 3), device=src.device, dtype=torch.uint8)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (h, w, 3) or not out.is_contiguous():
        raise ValueError("warp_sample_u8: out must be a contiguous uint8 (h, w, 3) image")
    check(lib.rf_warp_sample_u8(ptr(H), ptr(src), int(src.shape[0]), int(src.shape[1]), int(h), int(w), int(bool(align_corners)),
                                ptr(out), stream()))
    return out


# --------------------------------------------------------------------------- host rules
def train_pair_sizes(w, h, minSize):
    """cell 7: the (w, h) of I1Down2, I1, I1Up2 for a w x h source (or of I2 at index 1 for a w x h target)."""
    return [pipeline.fine_sizes(w, h, 16, m) for m in (minSize // 2, minSize, minSize * 2)]


def keep_pair(status, nbMatch):
    """cell 13's ``len(match1Inlier) > 50``: RANSAC returned a model (``isInlier`` has M entries; ``[]`` otherwise) and M > 50."""
    return int(status) == outil.RF_RANSAC_OK and int(nbMatch) > KEEP_MIN_MATCHES


def notebook_exception(status, nbMatch):
    """What the notebook raises on this pair: "RuntimeError" (M = 0, ``torch.randint``), "TypeError" (1 <= M <= 3, or no model
    in RANSAC's remainder chunk: utils/outil.py:162), or None."""
    if int(nbMatch) == 0:
        return "RuntimeError"
    if int(status) in (outil.RF_RANSAC_NO_MODEL, outil.RF_RANSAC_TOO_FEW):
        return "TypeError"
    return None


# --------------------------------------------------------------------------- the pair model
class TrainPairModel:
    """The notebook's settings and its ResNet-50 conv4 trunk.  ``resnet_state_dict``: torchvision ImageNet weights or the
    MoCo checkpoint the notebook loads by default (``{'model': {'module.<key>': ...}}``, cell 2); nothing is downloaded.
    ``sample_generator``: the CUDA generator RANSAC draws from (None: torch's default one, the notebook's stream)."""

    nbPoint = 4

    def __init__(self, resnet_state_dict, minSize=480, nbIter=10000, tolerance=0.05):
        self.net = ResNet50Conv4(resnet50_state(resnet_state_dict))
        self.minSize, self.nbIter, self.tolerance = int(minSize), int(nbIter), float(tolerance)
        self.sample_generator = None


def _device_u8(I):
    """A PIL image, numpy array or uint8 (H, W, 3) tensor as a uint8 CUDA image."""
    if torch.is_tensor(I):
        return I if I.is_cuda else I.cuda()
    return _CoarseAlignBase._to_device_u8(I)


def _matches(feats):
    """Cell 9 on the conv4 features of (Down2, 1, Up2, target): the mutual nearest neighbours of the three source scales' rows
    (in that order) and the target's, and their cell-centre coordinates.  Returns (source matches (H1, W1, 1), target matches
    (H2, W2, 1), the count [1], the mutual pairs' source and target row indices), all on the device."""
    o, dev = feats.offsets(), feats.data.device
    if feats.split:
        sp, tp = feats.data[:, :o[3]], feats.data[:, o[3]:o[4]]
        idx1, idx2, count = ops.corr_mutual_nn_presplit(sp[0], sp[1], tp[0], tp[1])
    else:
        idx1, idx2, count = ops.corr_mutual_nn(feats.data[:o[3]], feats.data[o[3]:o[4]], outil.corr_precision)
    WH = [outil._wh(feats.hw[i][0], feats.hw[i][1], dev) for i in range(4)]           # getWHTensor of each feature map
    W1 = torch.cat([WH[i][2] for i in range(3)])
    H1 = torch.cat([WH[i][3] for i in range(3)])
    m_src, m_tgt, _, cnt = ops.build_matches(idx1, idx2, count, W1, H1, WH[3][2], WH[3][3], None)
    return m_src, m_tgt, cnt, idx1, idx2


def _train_device(model, I1, I2, samples=None):
    """Cells 7-13 for uint8 (H, W, 3) CUDA images, everything queued on the current stream and nothing read back.  Returns a
    ``pipeline.DevicePair``: ``packed`` = [status, M, nbInlier, H(9), isInlier(capacity)] as float32, ``maps`` = (I1 resized,
    I2 warped into I1's frame), both uint8 (h1, w1, 3), as the one entry of a list."""
    with torch.no_grad():
        w1, h1 = int(I1.shape[1]), int(I1.shape[0])
        sizes = train_pair_sizes(w1, h1, model.minSize)
        src = [ops.resize_lanczos_u8(I1, w, h) for (w, h) in sizes]                  # Down2, 1, Up2 (ascending)
        w2, h2 = pipeline.fine_sizes(int(I2.shape[1]), int(I2.shape[0]), 16, model.minSize)
        tgt = ops.resize_lanczos_u8(I2, w2, h2)
        feats, _ = conv4_features(model.net, src + [tgt])                             # one ragged batch of four images
        m_src, m_tgt, cnt, _, _ = _matches(feats)
        H, nb, mask, status = ransac_device(m_tgt, m_src, cnt, model.nbIter, model.nbPoint, model.tolerance, model.sample_generator,
                                            samples)
        I1r = src[1]
        I2w = warp_sample_u8(H, tgt, int(I1r.shape[0]), int(I1r.shape[1]))
        packed = torch.cat([status.float(), cnt.float(), nb.float(), H, mask.float()])
        return pipeline.DevicePair(packed, [(I1r, I2w)], (int(I1r.shape[0]), int(I1r.shape[1])), ())


def _unpack_train(host, maps):
    """The host side of ``_train_device``: ``align_train_pair``'s dict."""
    status, M, nb = int(host[0]), int(host[1]), int(host[2])
    ok = status == outil.RF_RANSAC_OK
    return dict(kept=keep_pair(status, M), status=status, nbMatch=M, nbInlier=nb if ok else 0,
                H=host[3:12].reshape(3, 3).astype(np.float32), isInlier=host[12:12 + M] > 0.5 if ok else np.zeros(0, dtype=bool),
                I1=maps[0][0], I2=maps[0][1])


def align_train_pair(model, I1, I2, samples=None):
    """One pair of the notebook on the device with one pinned read at the end.  ``I1`` (source) / ``I2`` (target): uint8 HWC
    images (PIL, numpy or CUDA).  Returns dict(kept, status (RF_RANSAC_*), nbMatch (M), nbInlier, H (3, 3) float32, isInlier
    (M,) bool (empty without a model), I1 the resized source and I2 the target warped into its frame, both uint8 (h1, w1, 3)
    CUDA tensors).  Under ``torch.manual_seed(s)`` RANSAC draws the notebook's own CUDA ``torch.randint`` stream; ``samples``:
    an injected (nbIter, 4) index table instead."""
    pair = _train_device(model, _device_u8(I1), _device_u8(I2), samples)
    return _unpack_train(pipeline._read_back(pair)[0], pair.maps)


class GraphedTrainPairAligner(pipeline.GraphedAligner):
    """``align_train_pair`` as one CUDA graph per (I1 shape, I2 shape), LRU-bounded by ``max_graphs``, replayed per pair; RANSAC
    draws inside the graph, so successive replays use fresh samples.  A capture costs a few warm-up runs and its own memory:
    graphs pay off when sizes repeat (a dataset of one camera, or images resized to a few sizes beforehand); a MegaDepth-style
    dataset with a new size for most pairs is better served by ``align_train_pair``.  It can be a ``ConcurrentAligner`` lane
    (``make_models`` returning ``(TrainPairModel, None)``, ``make_aligner=GraphedTrainPairAligner``).  ``fetch`` clones the two
    images out of the graph's static buffers (``copy=False``: the live buffers, overwritten by the next replay with these
    sizes)."""

    def __init__(self, model, network=None, warmup=2, max_graphs=8):
        super().__init__(model, network, warmup=warmup, max_graphs=max_graphs)

    def _device(self, s_in, t_in):
        return _train_device(self.coarse, s_in, t_in)

    def _unpack(self, host, bg, maps, size, shapes):
        return _unpack_train(host, maps)
