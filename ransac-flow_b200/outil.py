"""Drop-in for the reference's ``outil`` module (utils/outil.py) on the H100 library.

Same function names, argument meaning, return types and error behaviour for the
hot-path functions; the arithmetic runs in the library's CUDA kernels.
``Affine`` / ``Hough`` / ``Translation`` / ``SaliencyCoef`` are dead or unbatched
host code in the reference (its RANSAC is hard-coded for homographies,
utils/outil.py:122-130) and are out of scope: they exist only as names.
"""
import numpy as np
import PIL.Image as Image
import torch

from . import ops
from ._lib import RFError

RF_RANSAC_OK, RF_RANSAC_NONE, RF_RANSAC_NO_MODEL, RF_RANSAC_TOO_FEW = 0, 1, 2, 3

# precision of the dense correlation: 0 = exact fp32 FMA, 1 = 3xTF32 on wgmma, 2 = fp16 split on wgmma
corr_precision = 0


def resizeImg(I, strideNet, minSize=400, mode=Image.LANCZOS):
    """utils/outil.py:6-19 (host, PIL)."""
    w, h = I.size
    wratio, hratio = w / minSize, h / minSize
    resizeRatio = min(wratio, hratio)
    w, h = w / resizeRatio, h / resizeRatio
    resizeW = round(w / strideNet) * strideNet
    resizeH = round(h / strideNet) * strideNet
    return I.resize((resizeW, resizeH), resample=mode)


_wh_cache = {}


def _wh(h, w, device):
    """Row / column index of every cell of an (h, w) grid, flattened row-major, plus the cell-centre
    coordinates.  Evaluated once per grid size with IEEE fp32 division on the host (torch's CUDA kernels
    turn ``x / scalar`` into ``x * (1 / scalar)``, which is off by an ulp from utils/outil.py:22-23 as the
    CPU evaluates it) and cached on the device."""
    key = (int(h), int(w), str(device))
    if key not in _wh_cache:
        r = torch.arange(0, h).view(-1, 1).expand(h, w).contiguous().view(-1)
        c = torch.arange(0, w).view(1, -1).expand(h, w).contiguous().view(-1)
        W = ((r.float() + 0.5) / h - 0.5) * 2
        H = ((c.float() + 0.5) / w - 0.5) * 2
        _wh_cache[key] = tuple(t.to(device) for t in (r, c, W, H))
    return _wh_cache[key]


def getWHTensor(feat):
    """utils/outil.py:21-24: cell-centre coordinates in [-1, 1] ("W" = rows/y, "H" = cols/x)."""
    _, _, W, H = _wh(feat.size(2), feat.size(3), feat.device)
    return W, H


def getWHTensor_Int(feat):
    """utils/outil.py:26-29."""
    r, c, _, _ = _wh(feat.size(2), feat.size(3), feat.device)
    return r, c


def _rows(feat):
    """(C, N) tensor -> [N, C] contiguous rows, without a copy when it is a transposed view."""
    t = feat.t()
    return t if t.is_contiguous() else t.contiguous()


def mutualMatching(featA, featB):
    """utils/outil.py:32-45.  featA (C, NA), featB (C, NB) -> (index1, index2) int64, sorted by index1.
    One fused kernel (+ a compaction kernel); the NA x NB score matrix is never materialised."""
    idx1, idx2, count = ops.corr_mutual_nn(_rows(featA.float()), _rows(featB.float()), corr_precision)
    n = int(count.item())              # same host sync as the reference's nonzero() (utils/outil.py:43)
    return idx1[:n], idx2[:n]


def Homography(X, Y):
    """utils/outil.py:68-87: X, Y (N,4,3) -> (N,3,3) fp32 CUDA (unit norm, LAPACK's sign), no host round trip."""
    return ops.homography_dlt(X.contiguous().float(), Y.contiguous().float())


def Affine(X, Y):
    raise NotImplementedError("outil.Affine is out of scope: the reference's RANSAC only works for homographies "
                              "(utils/outil.py:122-130, SURVEY.md A.3 #2)")


Hough = Translation = SaliencyCoef = Affine


def Prediction(X, Y, H21):
    """utils/outil.py:97-100: X, Y (1,M,3) or (M,3); H21 (N,3,3) -> (N,M)."""
    X2 = X.reshape(-1, 3).contiguous().float()
    Y2 = Y.reshape(-1, 3).contiguous().float()
    return ops.prediction(X2, Y2, H21.reshape(-1, 9).contiguous().float())


def ScoreRANSAC(match1, match2, tolerance, samples, Transform):
    """utils/outil.py:102-113."""
    X = match1[samples]
    Y = match2[samples]
    H21 = Transform(X, Y)
    dets = torch.det(H21)
    error = Prediction(match1.unsqueeze(0), match2.unsqueeze(0), H21)
    isInlier = error < tolerance
    return H21, torch.sum(isInlier, dim=1) * (dets > 1e-6).long()


def RANSAC_device(match1, match2, samples, tolerance, M_dev=None):
    """Device-resident form used by the fused pair pipeline: no host sync."""
    return ops.ransac_homography(match1.contiguous().float(), match2.contiguous().float(), samples.contiguous(), tolerance, 100, M_dev)


def RANSAC(nbIter, match1, match2, tolerance, nbPoint, Transform):
    """utils/outil.py:117-164.  Returns (H np (3,3) f32, nbInlier np int64, isInlier np bool (M,), match2[isInlier] np)
    or (None, 0, [], []); raises like the reference in its corner cases."""
    if Transform is not Homography:
        raise NotImplementedError("RANSAC is hard-coded for homographies (utils/outil.py:122-130)")
    nbMatch = len(match1)
    samples = torch.randint(nbMatch, (nbIter, nbPoint), device=match1.device)      # utils/outil.py:120
    if nbPoint != 4:
        raise IndexError("index 3 is out of bounds for dimension 1 with size %d" % nbPoint)   # utils/outil.py:125
    if nbMatch < 4:
        raise RFError("RANSAC needs at least 4 matches (callers return None before calling, coarseAlignFeatMatch.py:171)")
    H, nb, mask, status = RANSAC_device(match1, match2, samples, tolerance)
    packed = torch.cat([H, nb.float(), status.float()]).cpu().numpy()               # one D2H for the scalars
    st = int(packed[10])
    if st == RF_RANSAC_NONE:
        return None, 0, [], []
    if st == RF_RANSAC_NO_MODEL:
        raise TypeError("'NoneType' object is not subscriptable")                   # utils/outil.py:162
    isInlier = mask.bool()
    return (packed[:9].reshape(3, 3).astype(np.float32), nb.cpu().numpy()[0], isInlier.cpu().numpy(),
            match2[isInlier].cpu().numpy())
