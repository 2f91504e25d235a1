"""The on-disk formats of the evaluation drivers and the metrics of the getResults scripts (SURVEY.md section 8f-3), so
that results written here are read by the reference's ``getResults.py`` and vice versa.

  save_pair / load_pair            : evaluation/evalHpatch/evaluation.py:244-260 (identical in evalCorr :244-260)
  save_rotation                    : evaluation/evalYFCC/evaluation.py:270-271 (rotation.json, read by evalYFCC/getResults.py)
  getFlow_all_from_files           : evaluation/evalHpatch/getResults.py:16-63 (file lookup + np.load + composition)
  getFlow_from_files               : evaluation/evalCorr/getResults.py:78-134 / evalYFCC/getResults.py:132-190 (flow AND matchability)
  save_pair_kitti / kitti_pairs    : evaluation/evalKITTI/evaluation.py:43-47,338-344; evalKITTI/getResults.py:190-193
  getFlow_all_kitti_from_files     : evaluation/evalKITTI/getResults.py:95-141
  epe_hpatches                     : evaluation/evalHpatch/getResults.py:147-157,224-250
  alignment_error                  : evaluation/evalCorr/getResults.py:15-38
  epe_kitti                        : evaluation/evalKITTI/getResults.py:221-230
  save_train_pair / write_train_pairs : train/generate_coarse_aligned_pair.ipynb's pairs in the layout data/dataloader.py:40-60 reads

File IO and the sparse-keypoint lookups are host code as in the reference; the dense compositions run on the library's
kernels (``pipeline.getFlow_all`` / ``getFlow_all_kitti``), the dense metrics are elementwise torch on the tensors' device.
"""
import os

import numpy as np
import torch

from . import ops, pipeline


# --------------------------------------------------------------------------- evalHpatch / evalCorr / evalYFCC
def save_pair(outCoarse, outFine, idx, out, It_bg=None):
    """Write what evaluation.py:244-260 writes for pair ``idx``: ``outFine/maskBG_{idx}_{nH}H.npy`` (bool (H,W)),
    ``outFine/mask_{idx}_{nH}H.npy`` (nH,2,h8,w8) fp32, ``outCoarse/flow_{idx}_{nH}H.npy`` (nH,3,3) fp32 homographies and
    ``outFine/flow_{idx}_{nH}H.npy`` (nH,2,h8,w8) fp32.  ``out`` is the dict ``pipeline.align_pair*`` returns.  Nothing is
    written when no hypothesis was accepted (evaluation.py:244).  Returns nH."""
    nH = len(out["H"])
    if nH == 0:
        return 0
    f8 = np.asarray(out["flowDown8"], dtype=np.float32)
    if It_bg is None:
        It_bg = np.ones((f8.shape[2] * 8, f8.shape[3] * 8), dtype=np.float32)
    tag = "%s_%dH.npy" % (str(idx), nH)
    np.save(os.path.join(outFine, "maskBG_" + tag), np.asarray(It_bg).astype(bool))
    np.save(os.path.join(outFine, "mask_" + tag), np.asarray(out["matchDown8"], dtype=np.float32))
    np.save(os.path.join(outCoarse, "flow_" + tag), np.asarray(out["H"], dtype=np.float32))
    np.save(os.path.join(outFine, "flow_" + tag), f8)
    return nH


def save_rotation(outSceneFine, angle_rotation):
    """evaluation/evalYFCC/evaluation.py:270-271: ``outSceneFine/rotation.json``, the json dump of {pair index: angle} (the
    keys become strings: evalYFCC/getResults.py reads ``rotation[str(i)]``).  ``angle_rotation``: the ``angle`` of
    ``pipeline.align_pair_yfcc`` per pair.  Returns the path."""
    import json
    path = os.path.join(outSceneFine, "rotation.json")
    with open(path, "w") as f:
        json.dump({k: int(v) for k, v in angle_rotation.items()}, f)
    return path


def find_nbH(pairID, flowList):
    """getResults.py:17-25: the hypothesis count encoded in the file name of pair ``pairID`` (None when absent)."""
    for flowName in flowList:
        parts = flowName.split("_")
        if len(parts) >= 3 and parts[1] == str(pairID):
            return parts[2].split("H")[0]
    return None


def load_pair(pairID, finePath, coarsePath, flowList=None):
    """np.load of the three tensors getFlow_all reads (getResults.py:27-36): (flow, param, match) or None."""
    nbH = find_nbH(pairID, os.listdir(finePath) if flowList is None else flowList)
    if nbH is None:
        return None
    tag = "{}_{}H.npy".format(pairID, nbH)
    return (np.load(os.path.join(finePath, "flow_" + tag)).astype(np.float32),
            np.load(os.path.join(coarsePath, "flow_" + tag)).astype(np.float32),
            np.load(os.path.join(finePath, "mask_" + tag)).astype(np.float32))


def getFlow_all_from_files(pairID, finePath, coarsePath, flowList, multiH, th, outW, outH, with_match21=False):
    """evaluation/evalHpatch/getResults.py:16-63 with its argument order minus ``warper`` / ``grid`` (regenerated on the
    device): returns flowGlobal (1,outH,outW,2) CUDA, or [] when the pair has no files (``with_match21``: the evalCorr /
    evalYFCC composition, evalCorr/getResults.py:78-136)."""
    t = load_pair(pairID, finePath, coarsePath, flowList)
    if t is None:
        return []
    flow, param, match = t
    return pipeline.getFlow_all(flow, param, match, outH, outW, th=th, multiH=multiH, with_match21=with_match21)


def getFlow_from_files(pairID, finePath, flowList, coarsePath, maskPath, multiH, th):
    """evaluation/evalCorr/getResults.py:78-134 ``getFlow`` with its own argument order (``maskPath`` only serves the
    reference's unused ``maskBG`` load): (flowGlobal, matchGlobal) CUDA at 8x the saved resolution, or ([], [])."""
    t = load_pair(pairID, finePath, coarsePath, flowList)
    if t is None:
        return [], []
    flow, param, match = t
    return pipeline.getFlow_corr(flow, param, match, th=th, multiH=multiH)


# --------------------------------------------------------------------------- evalYFCC pose
def getFlow_yfcc_from_files(pairID, finePath, flowList, coarsePath, maskPath, multiH, th):
    """evaluation/evalYFCC/getResults.py:132-190 ``getFlow``: (flowGlobal (H,W,2) fp32, match_binary (H,W) bool) CUDA, the
    first-hypothesis-wins binary map multiplied by ``maskPath/maskBG_{pairID}_{nH}H.npy``; ([], []) when the pair has no files."""
    if flowList is None:
        flowList = os.listdir(finePath)
    t = load_pair(pairID, finePath, coarsePath, flowList)
    if t is None:
        return [], []
    flow, param, match = t
    bg = np.load(os.path.join(maskPath, "maskBG_{}_{}H.npy".format(pairID, find_nbH(pairID, flowList))))
    flowGlobal, _, mb = pipeline.getFlow_corr_binary(flow, param, match, th=th, multiH=multiH)
    mb = mb.squeeze() * torch.as_tensor(np.asarray(bg), device=mb.device).bool()
    return flowGlobal.squeeze(), mb


def yfcc_pose(flowGlobal, match_binary, size_A, size_B, angle, K_A, K_B, org_A, org_B, ransac=True, threshold=0.0005):
    """getResults.py:318-325 on the device: matches_from_flow + norm_kp + opencv_decompose (cv2.findEssentialMat(RANSAC) and
    cv2.recoverPose over the stacked candidates), every stage on the current stream; the host reads one record at the end.
    ``size_*`` = resized_shapes[id] (w, h), ``org_*`` = org_imsizes[id] (w, h).  Returns ((R, t) or None, match count)."""
    if not ransac:
        raise NotImplementedError("yfcc_pose: the non-RANSAC branch (cv2.findFundamentalMat(FM_8POINT) fed to recoverPose) "
                                  "is not implemented")
    flowGlobal = torch.as_tensor(flowGlobal).cuda()
    match_binary = torch.as_tensor(match_binary).cuda()
    n1 = _norm_params(org_A, size_A, np.asarray(K_A, dtype=np.float64))
    n2 = _norm_params(org_B, size_B, np.asarray(K_B, dtype=np.float64))
    pts1, pts2, N = ops.yfcc_matches(flowGlobal, match_binary, angle, size_A, size_B, n1, n2)
    rec, mask = ops.essential_ransac(pts1, pts2, N, threshold)
    ops.recover_pose(pts1, pts2, mask, rec)
    r = ops.read_pose_record(rec)
    if r["status"] != ops.POSE_OK or r["pose_count"] <= 0:
        return None, r["n_points"]
    return (r["R"], r["t"]), r["n_points"]


def yfcc_pose_8point(flowGlobal, match_binary, size_A, size_B, angle, K_A, K_B, org_A, org_B):
    """``yfcc_pose`` on the driver's non-RANSAC branch (getResults.py without --ransac): cv2.findFundamentalMat(FM_8POINT) and
    cv2.recoverPose over its stacked candidates, every stage on the current stream; the host reads one record at the end.
    Returns ((R, t) or None, match count)."""
    flowGlobal = torch.as_tensor(flowGlobal).cuda()
    match_binary = torch.as_tensor(match_binary).cuda()
    n1 = _norm_params(org_A, size_A, np.asarray(K_A, dtype=np.float64))
    n2 = _norm_params(org_B, size_B, np.asarray(K_B, dtype=np.float64))
    pts1, pts2, N = ops.yfcc_matches(flowGlobal, match_binary, angle, size_A, size_B, n1, n2)
    rec, mask = ops.fundamental_8point(pts1, pts2, N)
    ops.recover_pose(pts1, pts2, mask, rec)
    r = ops.read_pose_record(rec)
    if r["status"] != ops.POSE_OK or r["pose_count"] <= 0:
        return None, r["n_points"]
    return (r["R"], r["t"]), r["n_points"]


def opencv_decompose(pts1, pts2, ransac, threshold=0.0005):
    """getResults.py:75-111 on the device, both branches: ransac=True cv2.findEssentialMat(RANSAC, threshold), ransac=False
    cv2.findFundamentalMat(FM_8POINT), then cv2.recoverPose over the stacked candidates.  pts1 / pts2: (N, 2) normalised points
    (numpy or torch).  Returns ((R, t) or None, mask_final) as the driver does; mask_final is the winning candidate's recoverPose
    mask, (N, 1) uint8 on the device, or None.  (The driver's own mask_final aliases the array cv2 writes in place, so with
    stacked candidates it ends as the last candidate's mask; the driver never reads it.)  The host reads one record."""
    dev = torch.device("cuda", torch.cuda.current_device())
    P1 = torch.as_tensor(np.asarray(pts1) if not torch.is_tensor(pts1) else pts1).to(dev, torch.float64).reshape(-1, 2).contiguous()
    P2 = torch.as_tensor(np.asarray(pts2) if not torch.is_tensor(pts2) else pts2).to(dev, torch.float64).reshape(-1, 2).contiguous()
    N = int(P1.shape[0])
    Nd = torch.tensor([N], dtype=torch.int32, device=dev)
    if ransac:
        rec, mask = ops.essential_ransac(P1, P2, Nd, threshold)
    else:
        rec, mask = ops.fundamental_8point(P1, P2, Nd)
    out, _ = ops.recover_pose(P1, P2, mask, rec)
    r = ops.read_pose_record(rec)
    if r["status"] != ops.POSE_OK or r["pose_count"] <= 0:
        return None, None
    return (r["R"], r["t"]), out[:N].view(N, 1)


def _norm_params(org_size, new_size, K):
    """norm_kp's (cx, cy, fx, fy) (getResults.py:29-50), in its statement order."""
    w, h = org_size
    w_n, h_n = new_size
    cx = (w - 1.0) * 0.5
    cy = (h - 1.0) * 0.5
    cx += K[0, 2]
    cy += K[1, 2]
    fx = K[0, 0]
    fy = K[1, 1]
    cx *= (w_n / w)
    cy *= (h_n / h)
    fx *= (w_n / w)
    fy *= (h_n / h)
    return float(cx), float(cy), float(fx), float(fy)


def evaluate_R_t(R_gt, t_gt, R_pred, t_pred):
    """getResults.py:114-129: (rotation error, translation-direction error) in degrees (host numpy on 3 x 3s)."""
    t_gt = np.asarray(t_gt).flatten()
    t_pred = np.asarray(t_pred).flatten()
    R = np.asarray(R_gt) @ np.asarray(R_pred).T
    err_q = np.arccos((np.trace(R) - 1) / 2) * 180 / np.pi
    t_pred = t_pred / (np.linalg.norm(t_pred))
    t_gt = t_gt / (np.linalg.norm(t_gt))
    err_t = np.arccos(t_gt[None, :] @ t_pred[:, None]).item() * 180 / np.pi
    return err_q, err_t


def pose_accuracy(errors):
    """getResults.py:335-347: {'Acc@5', 'Acc@10', 'Acc@15', 'Acc@20'}, the fraction of pose errors below each threshold."""
    e = np.array(errors)
    return {"Acc@%d" % th: np.sum(e < th) / float(len(e)) for th in (5, 10, 15, 20)}


def yfcc_pose_errors(pairs_ids, finePath, coarsePath, maskPath, rotation, R_list, T_list, K_list, org_imsizes, resized_shapes,
                     multiH=True, th=0.95, ransac=True, threshold=0.0005, flowList=None):
    """The per-pair loop of getResults.py:298-331 for one scene: the max of the rotation and translation errors per pair, 180 for
    a pair with no files, no matches or no model.  ``R_list`` / ``T_list`` / ``K_list`` / ``org_imsizes`` are what the driver
    reads from its calibration files (``T_list[i]`` as the driver's ``np.array(calib['T']).T``), ``resized_shapes`` its
    getResizedSize per image, ``rotation`` the loaded rotation.json."""
    def pose(*args):
        return yfcc_pose(*args, ransac=ransac, threshold=threshold)
    return _pose_errors(pose, pairs_ids, finePath, coarsePath, maskPath, rotation, R_list, T_list, K_list, org_imsizes,
                        resized_shapes, multiH, th, flowList)


def yfcc_pose_errors_8point(pairs_ids, finePath, coarsePath, maskPath, rotation, R_list, T_list, K_list, org_imsizes,
                            resized_shapes, multiH=True, th=0.95, flowList=None):
    """``yfcc_pose_errors`` on the driver's non-RANSAC branch (getResults.py run without --ransac), through
    ``yfcc_pose_8point``."""
    return _pose_errors(yfcc_pose_8point, pairs_ids, finePath, coarsePath, maskPath, rotation, R_list, T_list, K_list, org_imsizes,
                        resized_shapes, multiH, th, flowList)


def _pose_errors(pose, pairs_ids, finePath, coarsePath, maskPath, rotation, R_list, T_list, K_list, org_imsizes, resized_shapes,
                 multiH, th, flowList):
    """The per-pair loop of getResults.py:298-331 with ``pose`` = the pose estimate of one pair."""
    if flowList is None:
        flowList = [item for item in os.listdir(finePath) if "flow" in item]
    res = []
    for i, (idA, idB) in enumerate(pairs_ids):
        flow, match = getFlow_yfcc_from_files(i, finePath, flowList, coarsePath, maskPath, multiH, th)
        if len(flow) == 0:
            res.append(180)
            continue
        r = R_list[idB] @ R_list[idA].T
        t = T_list[idB] - r @ T_list[idA]
        decomposed, n = pose(flow, match, resized_shapes[idA], resized_shapes[idB], rotation[str(i)], K_list[idA], K_list[idB],
                             org_imsizes[idA], org_imsizes[idB])
        if n == 0 or decomposed is None:
            res.append(180)
        else:
            res.append(max(evaluate_R_t(r, t, decomposed[0], decomposed[1])))
    return res


# --------------------------------------------------------------------------- evalKITTI
def save_pair_kitti(outDir, i, out, It_bg=None):
    """evaluation/evalKITTI/evaluation.py:338-344 (``save_output`` :43-47): ``Homograpy_{i}_{nH}.npy`` [sic] (nH,3,3),
    ``BG_{i}_{nH}H.npy`` bool, ``Finetune_D2_{i}_{nH}.npy``, ``Finetune_Mask_{i}_{nH}.npy``, ``Finetune_{i}_{nH}.npy`` (fp32).
    ``out`` is the dict ``pipeline.align_pair_kitti`` returns.  Returns nH."""
    nH = len(out["flow"])
    if nH == 0:
        return 0
    if It_bg is None:
        It_bg = np.ones(out["size"], dtype=np.float32)
    np.save(os.path.join(outDir, "Homograpy_{}_{}.npy".format(i, nH)), np.asarray(out["H"], dtype=np.float32))
    np.save(os.path.join(outDir, "BG_" + str(i) + "_{:d}H.npy".format(nH)), np.asarray(It_bg).astype(bool))
    np.save(os.path.join(outDir, "Finetune_D2_{}_{}.npy".format(i, nH)), np.asarray(out["flow_d2"], dtype=np.float32))
    np.save(os.path.join(outDir, "Finetune_Mask_{}_{}.npy".format(i, nH)), np.asarray(out["mask"], dtype=np.float32))
    np.save(os.path.join(outDir, "Finetune_{}_{}.npy".format(i, nH)), np.asarray(out["flow"], dtype=np.float32))
    return nH


def kitti_pairs(predDir):
    """evaluation/evalKITTI/getResults.py:190-193: {pair id: nbH} from the ``BG_*`` files of a prediction directory."""
    bg = [item for item in os.listdir(predDir) if "BG" in item]
    return dict((item.split("_")[1], item.split("_")[2].split("H")[0]) for item in bg)


def getFlow_all_kitti_from_files(pairID, predDir, nbH, res_name, Ith, Itw, multiH, th, cc_th, interpolate=False):
    """evaluation/evalKITTI/getResults.py:95-141 (``warper_org`` / ``grid_org`` regenerated on the device from the ground
    truth's size): flowGlobal (1,Ith,Itw,2) CUDA."""
    ld = lambda name: np.load(os.path.join(predDir, name)).astype(np.float32)
    param = ld("Homograpy_{}_{}.npy".format(pairID, nbH))
    flowd2 = ld("{}_D2_{}_{}.npy".format(res_name, pairID, nbH))
    flow = ld("{}_{}_{}.npy".format(res_name, pairID, nbH))
    match = ld("{}_Mask_{}_{}.npy".format(res_name, pairID, nbH))
    fg, _ = pipeline.getFlow_all_kitti(param, flowd2, flow, match, Ith, Itw, th=th, cc_th=cc_th, multiH=multiH, interpolate=interpolate)
    return fg


# --------------------------------------------------------------------------- metrics
def epe(input_flow, target_flow):
    """evaluation/evalHpatch/getResults.py:147-157."""
    return torch.norm(target_flow - input_flow, p=2, dim=1).mean()


def epe_hpatches(flow_est, flow_target, minSize):
    """evaluation/evalHpatch/getResults.py:224-250: average end-point error in pixels of a ``minSize`` x ``minSize`` image
    over the pixels whose ground-truth correspondence falls inside the image.  flow_est, flow_target: (1,H,W,2) in
    normalised [-1, 1] coordinates (any device)."""
    flow_target = flow_target.to(flow_est.device)
    mask = (flow_target[..., 0].ge(-1) & flow_target[..., 0].le(1)) & (flow_target[..., 1].ge(-1) & flow_target[..., 1].le(1))
    ft = (flow_target + 1) * (minSize - 1) / (1 + 1)
    fe = (flow_est + 1) * (minSize - 1) / (1 + 1)
    ft = torch.cat((ft[..., 0][mask].unsqueeze(1), ft[..., 1][mask].unsqueeze(1)), dim=1)
    fe = torch.cat((fe[..., 0][mask].unsqueeze(1), fe[..., 1][mask].unsqueeze(1)), dim=1)
    return epe(fe, ft).item()


def alignment_error(wB, hB, wA, hA, XA, YA, XB, YB, flow, match2, pixelGrid):
    """evaluation/evalCorr/getResults.py:15-38 (host code in the reference too: a lookup at the annotated keypoints):
    number of keypoints of the target aligned within each threshold of ``pixelGrid`` (1, T) and the number of keypoints
    covered by the matchability mask.  flow (1,hB,wB,2), match2 (1,hB,wB,1) or broadcastable; CUDA tensors are copied once."""
    flow = flow.detach().cpu()
    estimX = flow.narrow(3, 1, 1).reshape(hB, wB).numpy()
    estimY = flow.narrow(3, 0, 1).reshape(hB, wB).numpy()
    estimY = (estimY + 1) * 0.5 * (wA - 1)
    estimX = (estimX + 1) * 0.5 * (hA - 1)
    match = torch.as_tensor(match2).detach().cpu().squeeze().numpy()
    xa, ya, xb, yb = XA.astype(np.int64), YA.astype(np.int64), XB.astype(np.int64), YB.astype(np.int64)
    index = np.where(match[yb, xb] > 0.5)[0]
    nbAlign = len(index)
    if nbAlign > 0:
        xa, ya, xb, yb = xa[index], ya[index], xb[index], yb[index]
        pixelDiff = ((estimY[yb, xb] - xa) ** 2 + (estimX[yb, xb] - ya) ** 2) ** 0.5
        pixelDiffT = np.sum(pixelDiff.reshape((-1, 1)) <= pixelGrid, axis=0)
    else:
        pixelDiffT = np.zeros(pixelGrid.shape[1])
    return pixelDiffT, nbAlign


def epe_kitti(flow, u, v, valid):
    """evaluation/evalKITTI/getResults.py:221-230: flow (1,Ith,Itw,2) normalised target->source grid, ground truth (u, v)
    in pixels, ``valid`` mask -> average end-point error over the valid pixels."""
    Ith, Itw = u.shape
    dev = flow.device
    gy = torch.linspace(-1, 1, steps=Ith, device=dev).view(1, -1, 1, 1).expand(1, Ith, Itw, 1)
    gx = torch.linspace(-1, 1, steps=Itw, device=dev).view(1, 1, -1, 1).expand(1, Ith, Itw, 1)
    f = flow - torch.cat((gx, gy), dim=3)                          # fp32, as the reference's numpy arrays
    upred = (f[0, :, :, 0] * (Itw - 1) / 2).double()
    vpred = (f[0, :, :, 1] * (Ith - 1) / 2).double()
    u_t, v_t = torch.as_tensor(u, dtype=torch.float64, device=dev), torch.as_tensor(v, dtype=torch.float64, device=dev)
    val = torch.as_tensor(np.asarray(valid, dtype=np.float64), device=dev)
    error = ((upred - u_t) ** 2 + (vpred - v_t) ** 2) ** 0.5
    return (torch.sum(error * val) / torch.sum(val)).item()


# --------------------------------------------------------------------------- training pairs (README §4.1)
def save_train_pair(outDir, index, out):
    """Write a kept pair of ``pipeline.align_train_pair`` as ``outDir/{index}_1.jpg`` (the resized source) and ``{index}_2.jpg``
    (the target warped into its frame), with PIL's JPEG defaults: the two images ``ImageFolder`` (data/dataloader.py:43-60)
    reads for ``index``."""
    import PIL.Image as Image
    for k, key in ((1, "I1"), (2, "I2")):
        img = out[key]
        img = img.cpu().numpy() if torch.is_tensor(img) else np.asarray(img, dtype=np.uint8)
        Image.fromarray(img).save(os.path.join(outDir, "%d_%d.jpg" % (int(index), k)))


def _load_rgb(I):
    """A path (opened as the notebook opens it, ``Image.open(path).convert('RGB')``) or an image, as a uint8 (H, W, 3) array
    or tensor."""
    import PIL.Image as Image
    if isinstance(I, (str, os.PathLike)):
        return np.asarray(Image.open(I).convert("RGB"))
    if isinstance(I, Image.Image):
        return np.asarray(I.convert("RGB"))
    return I


def write_train_pairs(aligner, pairs, outDir, chunk=8):
    """The notebook over a dataset: every (I1, I2) in ``pairs`` (paths or images) through ``aligner`` (a
    ``GraphedTrainPairAligner``, a ``ConcurrentAligner`` of them, or any callable ``aligner(I1, I2)`` returning
    ``align_train_pair``'s dict), and the kept pairs written by ``save_train_pair``.  ``ImageFolder`` counts the files
    (``nbImg = len(listdir) // 2``) and reads indices 0 .. nbImg - 1, so kept pairs are numbered contiguously from 0 and
    rejected ones leave no hole; ``outDir`` (created if missing) must hold nothing else.  Returns, per input pair, its
    output index or None.  Reading and JPEG coding are host code; ``chunk`` pairs are queued at a time through a
    ``ConcurrentAligner``."""
    os.makedirs(outDir, exist_ok=True)
    if os.listdir(outDir):
        raise ValueError("write_train_pairs: %s is not empty (ImageFolder counts every file in it)" % outDir)
    run = aligner.run if hasattr(aligner, "run") else (lambda ps: [aligner(a, b) for a, b in ps])
    pairs = list(pairs)
    index, n = [], 0
    for s in range(0, len(pairs), chunk):
        loaded = [(_load_rgb(a), _load_rgb(b)) for a, b in pairs[s:s + chunk]]
        for out in run(loaded):
            if out["kept"]:
                save_train_pair(outDir, n, out)
                index.append(n)
                n += 1
            else:
                index.append(None)
    return index
