"""Oracle (test infrastructure) for train/validation.py: a torch-CPU fp32 restatement of the MegaDepth validation on
``model_oracle``'s networks, pinned to tests/golden/validation_megadepth.npz by tests/test_validation_host.py.

  sizes     : validation.py:22-24 (``round(w / ratio) // 16 * 16``, Python's half-to-even ``round``)
  keypoints : validation.py:18-19,26-29 (float32 arrays times a Python float), truncated by ``int()`` (:42)
  pair      : validation.py:80-107 (ToTensor, ``F.affine_grid`` / ``F.grid_sample``, the fine flow with ``up8X``, the CPU
              linspace grid, the clamp, the composition)
  distances : validation.py:33-53 (fp32 estimate, fp64 distance; the strict compare with the pixel grid)
"""
import numpy as np
import PIL.Image as Image
import torch
import torch.nn.functional as F

from . import model_oracle as MO

PIXEL_GRID = np.around(np.logspace(0, np.log10(36), 8).reshape(-1, 8))


def resize_size(w, h, minSize=480, strideNet=16):
    ratio = min(w / float(minSize), h / float(minSize))
    return round(w / ratio) // strideNet * strideNet, round(h / ratio) // strideNet * strideNet


def scaled_keypoints(x, y, w, h, minSize=480, strideNet=16):
    new_w, new_h = resize_size(w, h, minSize, strideNet)
    x = np.array(list(map(float, x.split(";")))).astype(np.float32)
    y = np.array(list(map(float, y.split(";")))).astype(np.float32)
    return x * (new_w / float(w)), y * (new_h / float(h))


def _to_tensor(img):
    return torch.from_numpy(np.array(img)).permute(2, 0, 1)[None].float().div(255)


def pair_distances(Is, It, theta, XA, YA, XB, YB, states, k=7, with_flow=False):
    """One pair: ``Is`` / ``It`` the original uint8 (H, W, 3) images, ``theta`` (2, 3) float32, the four coordinate strings.
    Returns the float64 distance of every keypoint (IndexError as torch indexing raises it); ``with_flow``: and the fine
    network's (1, 2, h8, w8) flow."""
    (hs0, ws0), (ht0, wt0) = Is.shape[:2], It.shape[:2]
    ws, hs = resize_size(ws0, hs0)
    wt, ht = resize_size(wt0, ht0)
    Xs, Ys = scaled_keypoints(XA, YA, ws0, hs0)
    Xt, Yt = scaled_keypoints(XB, YB, wt0, ht0)
    IsT = _to_tensor(Image.fromarray(Is).resize((ws, hs), resample=Image.LANCZOS))
    ItT = _to_tensor(Image.fromarray(It).resize((wt, ht), resample=Image.LANCZOS))
    with torch.no_grad():
        flowGlobalT = F.affine_grid(torch.from_numpy(np.asarray(theta, dtype=np.float32))[None], ItT.size(), align_corners=False)
        IsSample = F.grid_sample(IsT, flowGlobalT, align_corners=False)
        fs = F.normalize(MO.feature_extractor(IsSample, states["netFeatCoarse"]))
        ft = F.normalize(MO.feature_extractor(ItT, states["netFeatCoarse"]))
        flow8 = MO.net_flow_coarse(MO.corr_neigh(ft, fs, k), states["netFlowCoarse"], k)
        flowUp = F.interpolate(flow8, scale_factor=8, mode="bilinear", align_corners=True)
        gy = torch.linspace(-1, 1, steps=ht).view(1, -1, 1, 1).expand(1, ht, wt, 1)
        gx = torch.linspace(-1, 1, steps=wt).view(1, 1, -1, 1).expand(1, ht, wt, 1)
        flowCoarse = torch.clamp(flowUp.permute(0, 2, 3, 1) + torch.cat((gx, gy), dim=3), min=-1, max=1)
        flowFinal = F.grid_sample(flowGlobalT.permute(0, 3, 1, 2), flowCoarse, align_corners=False).permute(0, 2, 3, 1)
    f = flowFinal[0].numpy()
    d = []
    for j in range(len(Xt)):
        xa, ya, xb, yb = int(Xs[j]), int(Ys[j]), int(Xt[j]), int(Yt[j])
        if not (-ht <= yb < ht and -wt <= xb < wt):
            raise IndexError("keypoint %d: index out of bounds" % j)
        ex = (f[yb, xb, 0] + np.float32(1)) * np.float32(0.5) * np.float32(ws - 1)
        ey = (f[yb, xb, 1] + np.float32(1)) * np.float32(0.5) * np.float32(hs - 1)
        d.append(((float(ex) - xa) ** 2 + (float(ey) - ya) ** 2) ** 0.5)
    d = np.array(d, dtype=np.float64)
    return (d, flow8.numpy()) if with_flow else d


def precision(dists):
    """validation.py:49-51,110 over a list of per-pair distance arrays."""
    prec, total = np.zeros(8), 0
    for d in dists:
        prec += np.sum(np.asarray(d).reshape(-1, 1) < PIXEL_GRID, axis=0)
        total += len(d)
    with np.errstate(invalid="ignore"):
        return prec / total
