"""CPU oracle of evalYFCC's pair loop (evaluation/evalYFCC/evaluation.py:179-274) and the generator of its golden vectors.

  align_pair_yfcc : the four-rotation target search (:191-212) and the re-matching hypothesis loop (:214-274) on
                    ``oracle.pair_oracle.CoarseAlignOracle(variant="B")``, recording the sample table of every RANSAC call;
  gen_yfcc        : tests/golden/yfcc_rotation_search.npz from the UNMODIFIED reference - evalYFCC's own ``CoarseAlign``
                    class and the driver's ``PredFlowMask`` (compiled from the script's AST), the loop statements restated:

    python tests/yfcc_oracle.py            # needs the reference checkout ($RF_REFERENCE), writes tests/golden/
"""
import os
import sys

import numpy as np
import PIL.Image as Image
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import model_oracle as MO  # noqa: E402
from oracle import pair_oracle as PO  # noqa: E402
from oracle import synth  # noqa: E402
from oracle import warp_oracle as WO  # noqa: E402

ANGLES = (0, 90, 180, 270)


def imresize(arr, size):
    """``scipy.misc.imresize(arr, (h, w))`` of SciPy <= 1.2 (removed since): byte-scale a non-uint8 array to 0..255
    (``bytescale``: (x - min) * 255 / (max - min), span 1 when constant, + 0.5, truncated), then PIL's bilinear resize."""
    a = np.asarray(arr)
    if a.dtype != np.uint8:
        cmin, cmax = a.min(), a.max()
        cscale = cmax - cmin if cmax != cmin else 1
        a = (((a - cmin) * (255.0 / cscale)).clip(0, 255) + 0.5).astype(np.uint8)
    return np.asarray(Image.fromarray(a).resize((int(size[1]), int(size[0])), Image.BILINEAR))


def background(It_bg, k, size):
    """:193 / :200 / :212: the unrotated map (all ones without segNet) rotated by np.rot90, imresize, < 128.  size = (w, h)."""
    return (imresize(np.rot90(It_bg, k), (size[1], size[0])) < 128).astype(np.float32)


class CoarseAlignYFCC(PO.CoarseAlignOracle):
    """Variant B; ``inject`` (optional list of (nbIter, 4) tables) feeds the RANSAC calls in order instead of the seeded draw."""

    def __init__(self, resnet_sd, inject=None, **kw):
        super().__init__(resnet_sd, variant="B", **kw)
        self.inject = None if inject is None else list(inject)

    def _ransac(self, match1, match2):
        if self.inject is not None:
            self.raw_samples = self.inject.pop(0)
        return super()._ransac(match1, match2)


def align_pair_yfcc(coarse, net, Is, It, maxCoarse=10, maskRegionTh=0.01, It_bg=None):
    """One pair through evaluation/evalYFCC/evaluation.py:179-274 (PIL ``Is`` / ``It``; ``It_bg``: the segNet map of the
    unrotated target or None).  Returns dict(H, flowDown8, matchDown8, flow12, match, angle, nbInlierRot, Hrot, It_bg);
    ``coarse.all_samples`` holds the table of every RANSAC call."""
    coarse.setSource(Is)
    segNet = It_bg is not None
    if not segNet:
        It_bg = np.ones((It.size[1], It.size[0]), dtype=np.float32)
    ItList = [It] + [It.rotate(a, expand=True) for a in ANGLES[1:]]
    nbInlier, Hrot = [], []
    for j in range(4):
        coarse.setTarget(ItList[j])
        bg = background(It_bg, j, coarse.It.size)
        bestPara, InlierMask = coarse.getCoarse(((1 - bg) > 0.5).astype(np.float32))
        nbInlier.append(0 if bestPara is None else int(np.sum(InlierMask)))
        Hrot.append(np.zeros((3, 3), np.float32) if bestPara is None else bestPara)
    best = int(np.argmax(nbInlier))
    coarse.setTarget(ItList[best])
    Itw, Ith = coarse.It.size
    bg = background(It_bg, best, (Itw, Ith)) if segNet else np.ones((Ith, Itw), dtype=np.float32)
    featt = F.normalize(MO.feature_extractor(coarse.ItTensor, net["netFeatCoarse"]))
    grid = WO.base_grid(Ith, Itw)
    Mask = np.zeros((Ith, Itw), dtype=np.float32)
    Hs, flows8, matches8, flows, matches = [], [], [], [], []
    nbCoarse = 0
    while nbCoarse <= maxCoarse:
        fgMask = ((Mask + (1 - bg)) > 0.5).astype(np.float32)
        bestPara, _ = coarse.getCoarse(fgMask)
        if bestPara is None:
            break
        flowCoarse = WO.warp_grid(bestPara[None], Ith, Itw)
        flowFine, matchFine, f8, m8 = PO.pred_flow_mask(coarse.IsTensor, featt, flowCoarse, grid, net, with_match21=True)
        if (matchFine * (1 - fgMask)).mean() > maskRegionTh or nbCoarse == 0:
            Hs.append(bestPara[None])
            flows8.append(f8)
            matches8.append(m8)
            flows.append(flowFine)
            matches.append(matchFine)
            nbCoarse += 1
            Mask = ((Mask + matchFine * (1 - fgMask)) >= 1.0).astype(np.float32)     # :235-236 (len(...) is never 0 there)
        else:
            break
    cat = lambda l: np.concatenate(l, axis=0) if l else np.zeros((0,))
    return dict(H=cat(Hs), flowDown8=cat(flows8), matchDown8=cat(matches8), flow12=flows, match=matches, angle=ANGLES[best],
                nbInlierRot=nbInlier, Hrot=np.stack(Hrot), It_bg=bg.astype(bool))


# --------------------------------------------------------------------------------------------------------------------------
GOLDEN_ARGS = dict(seed=6, h=96, w=128, k=1, nbScale=3, nbIter=500, minSize=96, scaleR=1.5, maxCoarse=3, torch_seed=1000)


def gen_yfcc():
    """The reference's evalYFCC ``CoarseAlign`` (variant B, CPU) and ``PredFlowMask`` on a 96x128 pair whose target is
    rotated by 90 degrees, through the loop statements of evaluation.py:191-274 (no segNet), every ``torch.randint`` of
    ``outil.RANSAC`` recorded."""
    import types
    import torchvision
    from oracle import gen_golden as GG
    a = GOLDEN_ARGS
    src, tgt, _ = synth.make_rotated_pair(a["seed"], a["h"], a["w"], a["k"])
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    real_resnet50 = torchvision.models.resnet50

    def seeded_resnet50(*args, **kw):
        net = real_resnet50(weights=None)
        net.load_state_dict(synth.resnet50_conv4_state(0), strict=False)
        return net
    torchvision.models.resnet50 = seeded_resnet50
    res = types.ModuleType("resnet50")
    res.resnet50 = seeded_resnet50
    misc = types.ModuleType("scipy.misc")
    misc.imresize = imresize
    import scipy
    scipy.misc = misc
    try:
        mod = GG._coarse_align_common(os.path.join(GG.REF, "evaluation/evalYFCC/coarseAlignFeatMatch.py"), "ref_coarse_B_yfcc",
                                      {"segEval": types.ModuleType("segEval"), "resnet50": res, "scipy.misc": misc})
        model = GG.ref_model()
        network = GG._ref_networks(model)
        PredFlowMask = GG.extract_function(os.path.join(GG.REF, "evaluation/evalYFCC/evaluation.py"), "PredFlowMask",
                                           {"torch": torch, "F": F})
        rec = []
        with GG.cpu_as_cuda(), torch.no_grad(), GG.replay_randint(None, rec):
            coarseModel = mod.CoarseAlign(a["nbScale"], a["nbIter"], 0.05, "Homography", a["minSize"], 1, True, False, True, False,
                                          a["scaleR"])
            torch.manual_seed(a["torch_seed"])
            # evaluation.py:187-212 (segNet off)
            coarseModel.setSource(Is)
            It_bg = np.ones((It.size[1], It.size[0]), dtype=np.float32)
            ItList = [It, It.rotate(90, expand=True), It.rotate(180, expand=True), It.rotate(270, expand=True)]
            It_bg_List = [It_bg, np.rot90(It_bg), np.rot90(It_bg, 2), np.rot90(It_bg, 3)]
            nbInlier, Hrot, calls_rot = [], [], []
            for j in range(4):
                coarseModel.setTarget(ItList[j])
                Itw, Ith = coarseModel.It.size
                It_bg = It_bg_List[j]
                It_bg = (imresize(It_bg, (Ith, Itw)) < 128).astype(np.float32)
                fgMask = ((1 - It_bg) > 0.5).astype(np.float32)
                n0 = len(rec)
                bestPara, InlierMask = coarseModel.getCoarse(fgMask)
                calls_rot.append(len(rec) - n0)
                if bestPara is None:
                    nbInlier.append(0)
                    Hrot.append(np.zeros((3, 3), np.float32))
                else:
                    nbInlier.append(np.sum(InlierMask))
                    Hrot.append(bestPara)
            coarseModel.setTarget(ItList[np.argmax(nbInlier)])
            angle = [0, 90, 180, 270][np.argmax(nbInlier)]
            Itw, Ith = coarseModel.It.size
            It_bg = np.ones((Ith, Itw), dtype=np.float32)
            featt = F.normalize(network["netFeatCoarse"](coarseModel.ItTensor))
            gridY = torch.linspace(-1, 1, steps=Ith).view(1, -1, 1, 1).expand(1, Ith, Itw, 1)
            gridX = torch.linspace(-1, 1, steps=Itw).view(1, 1, -1, 1).expand(1, Ith, Itw, 1)
            grid = torch.cat((gridX, gridY), dim=3)
            # evaluation.py:225-274 (kornia is absent: the oracle's warp_grid stands in for HomographyWarper.warp_grid)
            Mask = np.zeros((Ith, Itw), dtype=np.float32)
            Coarse_Flow_Tensor, Fine_Flow_Tensor, Fine_Mask_Tensor = [], [], []
            nbCoarse = 0
            while nbCoarse <= a["maxCoarse"]:
                fgMask = ((Mask + (1 - It_bg)) > 0.5).astype(np.float32)
                bestPara, InlierMask = coarseModel.getCoarse(fgMask)
                if bestPara is None:
                    break
                bestPara = torch.from_numpy(bestPara).unsqueeze(0)
                flowCoarse = WO.warp_grid(bestPara, Ith, Itw)
                flowFine, matchFine, flowFineDown8, matchFineDown8 = PredFlowMask(coarseModel.IsTensor, featt, flowCoarse, grid, network)
                if (matchFine * (1 - fgMask)).mean() > 0.01 or nbCoarse == 0:
                    Coarse_Flow_Tensor.append(bestPara.numpy())
                    Fine_Flow_Tensor.append(flowFineDown8)
                    Fine_Mask_Tensor.append(matchFineDown8)
                    nbCoarse += 1
                    matchFine = matchFine if len(Fine_Mask_Tensor) == 0 else matchFine * (1 - fgMask)
                    Mask = ((Mask + matchFine) >= 1.0).astype(np.float32)
                else:
                    break
    finally:
        torchvision.models.resnet50 = real_resnet50
        for name in ("segEval", "resnet50"):
            sys.modules.pop(name, None)
    assert len(Coarse_Flow_Tensor) > 0
    GG.save("yfcc_rotation_search", src=src, tgt=tgt, k=np.int64(a["k"]), angle=np.int64(angle), nbInlierRot=np.asarray(nbInlier, np.int64),
            Hrot=np.stack(Hrot).astype(np.float32), calls_rot=np.asarray(calls_rot, np.int64),
            samples=np.stack([s for _, s in rec]), nbMatch=np.asarray([m for m, _ in rec], np.int64),
            H=np.concatenate(Coarse_Flow_Tensor, 0), flowDown8=np.concatenate(Fine_Flow_Tensor, 0),
            matchDown8=np.concatenate(Fine_Mask_Tensor, 0), It=np.asarray(coarseModel.It))


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_yfcc()
