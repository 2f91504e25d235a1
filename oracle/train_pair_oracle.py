"""Oracle (test infrastructure): train/generate_coarse_aligned_pair.ipynb (cells 7-13) restated on the CPU in fp32 on the
other oracle modules, with the RANSAC draw hoisted out (``samples``: the (nbIter, 4) table its ``torch.randint`` returns).

  cell 7  : ``outil.resizeImg`` (``pair_oracle.resize_img``) of the original source to minSize // 2, minSize, minSize * 2 and
            of the target to minSize; ImageNet preprocessing, ResNet-50 conv4, ``F.normalize``
  cell 9  : source rows Down2, 1, Up2; ``mutualMatching``; match1 = target (H2, W2, 1), match2 = source (H1, W1, 1)
  cell 11 : ``outil.RANSAC`` (``RANSAC_from_samples``)
  cell 13 : kept when ``len(isInlier) > 50``; the target sampled on the homography grid of the source's size, ``ToPILImage``
            (``x * 255`` truncated to uint8)
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import model_oracle as MO
from . import outil_oracle as OO
from . import pair_oracle as PO
from . import warp_oracle as WO


def _feat(I, sd):
    return F.normalize(MO.resnet50_conv4(PO.preproc(I).unsqueeze(0), sd))


def features(sd, I1_org, I2_org, minSize=480):
    """Cell 7 and the feature half of cell 9: (the resized source scales, the resized target, featpMultiScale (1024, NA) with the
    rows Down2, 1, Up2, feat2T (1024, NB), WMultiScale, HMultiScale, W2, H2)."""
    I1s = [PO.resize_img(I1_org, 16, m) for m in (minSize // 2, minSize, minSize * 2)]
    I2 = PO.resize_img(I2_org, 16, minSize)
    feats, Ws, Hs = [], [], []
    for I in I1s:
        f = _feat(I, sd)
        W, H = OO.getWHTensor(f.shape[2], f.shape[3])
        feats.append(f.contiguous().view(f.shape[1], -1))
        Ws.append(W)
        Hs.append(H)
    f2 = _feat(I2, sd)
    W2, H2 = OO.getWHTensor(f2.shape[2], f2.shape[3])
    return (I1s, I2, torch.cat(feats, dim=1).numpy(), f2.contiguous().view(f2.shape[1], -1).numpy(), np.concatenate(Ws),
            np.concatenate(Hs), W2, H2)


def train_pair(sd, I1_org, I2_org, samples, minSize=480, tolerance=0.05):
    """``I1_org`` (source) / ``I2_org`` (target): PIL images.  Returns dict(sizes [(w, h)] of I1Down2, I1, I1Up2, I2; I1 the
    resized source (uint8 HWC); nbMatch; match1, match2; H (3, 3) or None; isInlier (M,) bool or []; kept; I2Sample the warped
    target (uint8 (h1, w1, 3)) or None when not kept).  Raises where the notebook raises (M = 0: RuntimeError, as
    ``torch.randint(0, ...)``; no model in the remainder chunk: TypeError)."""
    I1s, I2, featp, feat2T, WMulti, HMulti, W2, H2 = features(sd, I1_org, I2_org, minSize)
    i1, i2 = OO.mutualMatching(featp, feat2T)
    one = np.ones(len(i1), dtype=np.float32)
    match2 = np.stack([HMulti[i1], WMulti[i1], one], axis=1)
    match1 = np.stack([H2[i2], W2[i2], one], axis=1)
    out = dict(sizes=[I.size for I in I1s] + [I2.size], I1=np.asarray(I1s[1]), nbMatch=len(match1), match1=match1, match2=match2)
    if len(match1) == 0:
        raise RuntimeError("random_ expects 'from' to be less than 'to'")           # torch.randint(0, ...)
    best, _, isInlier, _ = OO.RANSAC_from_samples(match1, match2, samples, tolerance)
    out.update(H=best, isInlier=isInlier, kept=len(isInlier) > 50, I2Sample=None)
    if out["kept"]:
        w1, h1 = I1s[1].size
        grid = WO.warp_grid(torch.from_numpy(best.astype(np.float32))[None], h1, w1)
        s = WO.grid_sample(PO.to_tensor(I2).unsqueeze(0), grid)[0]
        out["I2Sample"] = s.mul(255).byte().permute(1, 2, 0).numpy()
    return out
