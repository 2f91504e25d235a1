"""CPU restatement of evaluation/evalCorr/getResults.py's loop (:178-257), built on ``warp_oracle.get_flow_corr`` (getFlow) and
``warp_oracle.warp_grid`` (getFlow_Coarse), pinned to tests/golden/corr_results.npz.  Sizes come from the images' headers,
as ``ResizeMinResolution*`` computes them; alignmentError is restated with its binary-map broadcast, its int64 truncation and
numpy's index rule.  ``calls`` receives (pair, th, selected indices, distances) per alignmentError call, as the golden
records them."""
import hashlib
import os

import numpy as np
import PIL.Image as Image
import torch

from . import warp_oracle as WO

PIXEL_GRID = np.around(np.logspace(0, np.log10(36), 8).reshape(-1, 8))
COLUMNS = ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB")


def image(seed, w, h):
    """The synthetic RGB image of a seed: smooth gradients plus noise, uint8 (h, w, 3)."""
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * 255.0 / max(w - 1, 1), y * 255.0 / max(h - 1, 1), (x + y) * 127.0 / max(w + h - 2, 1)], axis=2)
    return np.clip(base + rs.normal(0, 20, (h, w, 3)), 0, 255).astype(np.uint8)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case_setup(g, name, root):
    """Write golden case ``name`` of corr_results.npz ``g`` under ``root`` as the generator did (images checked against their
    SHA-256): returns (DataFrame, testDir, finePth, coarsePth, argv without the directories, subcommand, reference error)."""
    import pandas as pd
    shape, kind, sub, missing, extra, err = [str(v) for v in g["%s_meta" % name]]
    missing = [int(v) for v in missing.split(",") if v]
    imgs, fine, coarse = os.path.join(root, "imgs"), os.path.join(root, "fine"), os.path.join(root, "coarse")
    for d in (fine, coarse, os.path.join(imgs, "scene0"), os.path.join(imgs, "scene1")):
        os.makedirs(d, exist_ok=True)
    cols = {c: [str(v) for v in g["csv_%s_%s_%s" % (shape, kind, c)]] for c in COLUMNS}
    for p in range(int(g["n_pairs"])):
        ws, hs, sseed, wt, ht, tseed = [int(v) for v in g["img_%s_%d" % (shape, p)]]
        s, t = image(sseed, ws, hs), image(tseed, wt, ht)
        if [digest(s), digest(t)] != [str(v) for v in g["sha_%s_%d" % (shape, p)]]:
            raise RuntimeError("corr_results golden: the synthetic images of pair %d differ from the generator's" % p)
        d = imgs if cols["scene"][p] == "/" else os.path.join(imgs, cols["scene"][p])
        Image.fromarray(s).save(os.path.join(d, "s%d.png" % p))
        Image.fromarray(t).save(os.path.join(d, "t%d.png" % p))
        if p in missing:
            continue
        Hs, flow, match = (g["%s_%s_%d" % (k, shape, p)] for k in ("H", "flow", "match"))
        tag = "%d_%dH.npy" % (p, len(Hs))
        np.save(os.path.join(fine, "flow_" + tag), flow)
        np.save(os.path.join(fine, "mask_" + tag), match)
        np.save(os.path.join(fine, "maskBG_" + tag), np.ones((8 * flow.shape[2], 8 * flow.shape[3]), bool))
        np.save(os.path.join(coarse, "flow_" + tag), Hs)
    df = pd.DataFrame(cols, dtype=str)
    return df, imgs, fine, coarse, extra.split(), sub, err


def case_args(extra):
    """(multiH, th, matchabilityTH, dataset, onlyCoarse) of a case's extra argv, with getResults.py's defaults."""
    a = dict(multiH=False, th=0.95, mth=[0], dataset="MegaDepth", onlyCoarse=False)
    k = 0
    while k < len(extra):
        if extra[k] == "--multiH":
            a["multiH"] = True
        elif extra[k] == "--onlyCoarse":
            a["onlyCoarse"] = True
        elif extra[k] == "--th":
            a["th"] = float(extra[k + 1])
            k += 1
        elif extra[k] == "--dataset":
            a["dataset"] = extra[k + 1]
            k += 1
        elif extra[k] == "--matchabilityTH":
            a["mth"] = []
            while k + 1 < len(extra) and not extra[k + 1].startswith("--"):
                a["mth"].append(float(extra[k + 1]))
                k += 1
        k += 1
    return a["multiH"], a["th"], a["mth"], a["dataset"], a["onlyCoarse"]


def resize_keypoints(minSize, size, x, y, strideNet=16):
    """ResizeMinResolution (getResults.py:41-57) minus the image: (new size, float32 keypoints)."""
    x = np.array(list(map(float, x.split(";")))).astype(np.float32)
    y = np.array(list(map(float, y.split(";")))).astype(np.float32)
    w, h = size
    ratio = min(w / float(minSize), h / float(minSize))
    new_w, new_h = round(w / ratio), round(h / ratio)
    new_w, new_h = new_w // strideNet * strideNet, new_h // strideNet * strideNet
    return (new_w, new_h), x * (new_w / float(w)), y * (new_h / float(h))


def alignment_error(wB, hB, wA, hA, XA, YA, XB, YB, flow, match2, pixelGrid, record=None):
    """getResults.py:15-38 on CPU tensors."""
    estimX = flow.narrow(3, 1, 1).view(1, 1, hB, wB)
    estimY = flow.narrow(3, 0, 1).view(1, 1, hB, wB)
    estimY = ((estimY + 1) * 0.5 * (wA - 1)).squeeze().numpy()
    estimX = ((estimX + 1) * 0.5 * (hA - 1)).squeeze().numpy()
    match = match2.squeeze().numpy()
    xa, ya, xb, yb = XA.astype(np.int64), YA.astype(np.int64), XB.astype(np.int64), YB.astype(np.int64)
    index = np.where(match[yb, xb] > 0.5)[0]
    xa, ya, xb, yb = xa[index], ya[index], xb[index], yb[index]
    d = ((estimY[yb, xb] - xa) ** 2 + (estimX[yb, xb] - ya) ** 2) ** 0.5
    if record is not None:
        record(index, np.asarray(d, dtype=np.float64))
    if len(index) == 0:
        return np.zeros(pixelGrid.shape[1]), 0
    return np.sum(d.reshape((-1, 1)) <= pixelGrid, axis=0), len(index)


def get_results(df, testDir, finePth, coarsePth, multiH, th, matchabilityTH, dataset, onlyCoarse=False, minSize=480, calls=None):
    """The loop of getResults.py over ``df``: {threshold: (precision, validAlign)}; raises what the script raises."""
    precAllAlign, validAlign = {}, {}
    for t in matchabilityTH:
        precAllAlign[t] = np.zeros(8)
        validAlign[t] = 0
    flowList = os.listdir(finePth)
    t = matchabilityTH[-1]
    for i in range(len(df)):
        scene = df["scene"][i]
        path = lambda n: os.path.join(os.path.join(testDir, scene), n) if scene != "/" else os.path.join(testDir, n)
        with Image.open(path(df["source_image"][i])) as im:
            (Isw, Ish), Xs, Ys = resize_keypoints(minSize, im.size, df["XA"][i], df["YA"][i])
        with Image.open(path(df["target_image"][i])) as im:
            (Itw, Ith), Xt, Yt = resize_keypoints(minSize, im.size, df["XB"][i], df["YB"][i])
        if dataset != "RobotCar":
            valid = (Xs > 0) * (Xs < Isw) * (Ys > 0) * (Ys < Ish) * ((Xt > 0) * (Xt < Itw) * (Yt > 0) * (Yt < Ith))
            Xs, Ys, Xt, Yt = Xs[valid], Ys[valid], Xt[valid], Yt[valid]
        nbH = next((f.split("_")[2].split("H")[0] for f in flowList if f.split("_")[1] == str(i)), None)
        if nbH is None:
            precAllAlign[0] = precAllAlign[t] + np.zeros(8)
            validAlign[0] += len(Xs)
            continue
        tag = "{}_{}H.npy".format(i, nbH)
        flow = np.load(os.path.join(finePth, "flow_" + tag)).astype(np.float32)
        param = np.load(os.path.join(coarsePth, "flow_" + tag)).astype(np.float32)
        h, w = flow.shape[2] * 8, flow.shape[3] * 8
        if onlyCoarse:
            fg, mg = WO.warp_grid(param[:1], h, w), torch.ones(1, h, w, 1)
        else:
            match = np.load(os.path.join(finePth, "mask_" + tag)).astype(np.float32)
            fg, mg = WO.get_flow_corr(flow, param, match, th=th, multiH=multiH)
        for t in matchabilityTH:
            inside = ((fg.narrow(3, 0, 1) >= -1) * (fg.narrow(3, 0, 1) <= 1)).float() * \
                     ((fg.narrow(3, 1, 1) >= -1) * (fg.narrow(3, 1, 1) <= 1)).float()
            mb = (mg >= t).float() * inside.permute(0, 3, 1, 2) if t > 0 else torch.ones(mg.size())
            rec = None if calls is None else (lambda idx, d, i=i, t=t: calls.append((i, t, idx, d)))
            pd_, nb = alignment_error(Itw, Ith, Isw, Ish, Xs, Ys, Xt, Yt, fg, mb, PIXEL_GRID, rec)
            precAllAlign[t] = precAllAlign[t] + pd_
            validAlign[t] += nb
    with np.errstate(invalid="ignore", divide="ignore"):
        return {t: (precAllAlign[t] / validAlign[t], validAlign[t]) for t in matchabilityTH}
