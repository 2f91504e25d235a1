"""evalCorr getResults on the device (``corr_results``, ``rf_corr_keypoints``).

  kernel      : the merged flow and matchability at each keypoint bit for bit against the dense ``pipeline.getFlow_corr`` on
                the same device operands (``ops.warp_grid`` for getFlow_Coarse), the counts against ``results.alignment_error``
                on the dense maps, with the reference's binary map (its broadcast for a threshold > 0 on a square map), also
                with a target of the flow's pixel count in another shape (the flow read at the flat index)
  fp64        : the merged values against geometry_ref's fp64 composition of the winning hypothesis, within its allowance
  golden      : ``get_results`` over every case of tests/golden/corr_results.npz (the reference's own run): the printed lines
                and the reference's errors; per keypoint the distances within 1e-4 px of the reference's
  sync        : the dataset loop queues nothing that synchronises
  evaluate    : the in-process loop against align_pair_multi -> save_pair -> get_results under the same seed, both engines
  CLI         : ``python -m ransac_flow_b200.corr_results`` in a process of its own prints the reference's lines
"""
import contextlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ransac_flow_b200 as rf
from oracle import corr_results_oracle as CO

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "corr_results.npz"))
CASES = [str(c) for c in GOLD["cases"]]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PG = rf.corr_results.PIXEL_GRID


def _operands(rs, nH, h8, w8, nan_h=None, outside=None):
    Hs = np.stack([np.eye(3) + rs.uniform(-0.05, 0.05, (3, 3)) for _ in range(nH)]).astype(np.float32)
    if nan_h is not None:
        Hs[nan_h] = np.nan
    if outside is not None:
        Hs[outside, 0, 2] += 0.5
    flow = rs.normal(0, 0.04, (nH, 2, h8, w8)).astype(np.float32)
    match = rs.uniform(0, 1, (nH, 2, h8, w8)).astype(np.float32)
    match[0] *= 0.6                                       # later hypotheses win at th = 0.5
    return Hs, flow, match


def _kpts(rs, n, H, W, Ith, Itw):
    xb, yb = rs.randint(-W, W, n), rs.randint(-H, H, n)
    xb[:4], yb[:4] = [W - 1, 0, W - 1, -1], [H - 1, H - 1, 0, -H]
    xa, ya = rs.randint(0, Itw, n), rs.randint(0, Ith, n)
    return np.stack([xa, ya, xb, yb], axis=1).astype(np.int32)


def _dense(Hs, flow, match, multiH, th, onlyCoarse):
    H, W = flow.shape[2] * 8, flow.shape[3] * 8
    if onlyCoarse:
        return rf.ops.warp_grid(torch.from_numpy(Hs[:1]).cuda(), H, W), torch.ones(1, H, W, 1, device="cuda")
    return rf.pipeline.getFlow_corr(flow, Hs, match, th=th, multiH=multiH)


def _binary(fg, mg, t):
    """getResults.py:250 on the dense maps (the broadcast included)."""
    inside = ((fg.narrow(3, 0, 1) >= -1) * (fg.narrow(3, 0, 1) <= 1)).float() * ((fg.narrow(3, 1, 1) >= -1) * (fg.narrow(3, 1, 1) <= 1)).float()
    return (mg >= t).float() * inside.permute(0, 3, 1, 2) if t > 0 else torch.ones(mg.size(), device=mg.device)


@pytest.mark.parametrize("nH,h8,w8,multiH,nan_h,onlyCoarse,mth,transpose", [
    (1, 8, 10, True, None, False, [0], False),
    (11, 8, 10, True, None, False, [0], False),
    (11, 7, 9, True, 3, False, [0], False),           # odd h8, w8 and a NaN H
    (3, 9, 9, False, None, False, [0, 0.5], False),   # multiH off; square: the broadcast of a threshold > 0
    (4, 9, 9, True, 0, False, [0.5, 0, 0.3], False),  # hypothesis 0 NaN: the merged flow keeps NaN where it wins
    (3, 8, 10, True, None, True, [0], False),         # onlyCoarse: the homography grid points equal warp_grid's
    (3, 9, 9, True, None, True, [0, 0.5], False),     # onlyCoarse, square
    (11, 8, 10, True, None, False, [0], True),        # the target is W x H: the flow is read at the flat index
    (3, 8, 10, True, None, True, [0], True),          # the same with onlyCoarse
])
def test_kernel_against_dense(nH, h8, w8, multiH, nan_h, onlyCoarse, mth, transpose):
    rs = np.random.RandomState(nH * 100 + h8 * 10 + w8 + (nan_h or 0))
    Hs, flow, match = _operands(rs, nH, h8, w8, nan_h, outside=1 if nH > 2 else None)
    H, W = 8 * h8, 8 * w8
    Ith, Itw = (W, H) if transpose else (H, W)
    th = 0.5
    kp = _kpts(rs, 300, min(H, Ith), min(W, Itw), Ith, Itw)
    n = len(kp)
    scores = rf.corr_results.CorrScores(mth, th, multiH, onlyCoarse)
    dev = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    fo = torch.full((n, 2), -7.0, device="cuda")
    mo = torch.full((n,), -7.0, device="cuda")
    ho = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    do = torch.empty((n, len(mth)), dtype=torch.float64, device="cuda")
    f8, Hm = (dev(flow[:1]), dev(Hs[:1])) if onlyCoarse else (dev(flow), dev(Hs))
    rf.corr_results.corr_keypoints(f8, None if onlyCoarse else dev(match), Hm.reshape(-1, 9), (Ith, Itw), (Ith, Itw), dev(kp),
                                   torch.tensor([n], dtype=torch.int32, device="cuda"), scores.acc, scores.err, PG, mth,
                                   scores.slots, th, multiH, onlyCoarse, 0, fo, mo, ho, do)
    counts, err = scores.read()
    assert err is None
    fg, mg = _dense(Hs, flow, match, multiH, th, onlyCoarse)
    yb, xb = kp[:, 3] % H, kp[:, 2] % W
    ref_f = fg[0].cpu().numpy()[yb, xb]
    ref_m = mg[0, ..., 0].cpu().numpy()[yb, xb]
    np.testing.assert_array_equal(fo.cpu().numpy().view(np.int32), ref_f.view(np.int32))       # bit for bit, NaN included
    np.testing.assert_array_equal(mo.cpu().numpy().view(np.int32), ref_m.view(np.int32))
    if multiH and not onlyCoarse and nH > 1:
        assert (ho.cpu().numpy() > 0).any()                                                 # a later hypothesis wins
    for k, key in enumerate(scores.keys):
        exp_c, exp_n = np.zeros(PG.size), 0
        for t in [t for t in mth if t == key]:
            c, nb = rf.results.alignment_error(Itw, Ith, Itw, Ith, kp[:, 0].astype(np.float32), kp[:, 1].astype(np.float32),
                                               kp[:, 2].astype(np.float32), kp[:, 3].astype(np.float32), fg, _binary(fg, mg, t), PG)
            exp_c, exp_n = exp_c + c, exp_n + nb
        np.testing.assert_array_equal(counts[k, :PG.size], exp_c)
        assert counts[k, PG.size] == exp_n
    if transpose:                                         # the flat-index reading differs from the pixel (yb, xb)
        flat = (kp[:, 3] % Ith) * Itw + kp[:, 2] % Itw
        assert ((flat // W != yb) | (flat % W != xb)).any()


def test_composition_against_fp64():
    """The kernel's merged flow and matchability at each keypoint against geometry_ref's fp64 composition of the winning
    hypothesis, within its propagated sampling allowance (the matchability where the inside test is decided)."""
    import geometry_ref as G
    rs = np.random.RandomState(77)
    nH, h8, w8 = 3, 8, 10
    Hs, flow, match = _operands(rs, nH, h8, w8, outside=1)
    H, W = 8 * h8, 8 * w8
    kp = _kpts(rs, 400, H, W, H, W)
    n = len(kp)
    scores = rf.corr_results.CorrScores([0], 0.5, True, False)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    fo = torch.empty((n, 2), device="cuda")
    mo = torch.empty((n,), device="cuda")
    ho = torch.empty((n,), dtype=torch.int32, device="cuda")
    rf.corr_results.corr_keypoints(dev(flow), dev(match), dev(Hs).reshape(-1, 9), (H, W), (H, W), dev(kp),
                                   torch.tensor([n], dtype=torch.int32, device="cuda"), scores.acc, scores.err, PG, [0], [0], 0.5,
                                   True, False, 0, fo, mo, ho)
    fo, mo, ho = fo.cpu().numpy(), mo.cpu().numpy(), ho.cpu().numpy()
    yb, xb = kp[:, 3] % H, kp[:, 2] % W
    refs = [G.compose_fine_ref(flow[i], match[i, 0], match[i, 1], G.warp_grid_f32(Hs[i:i + 1], H, W)[0], H, W) for i in range(nH)]
    assert len(set(ho.tolist())) > 1
    for i in range(nH):
        sel = ho == i
        r = refs[i]
        y, x = yb[sel], xb[sel]
        G.check(fo[sel], np.clip(r["flow12"][y, x], -1, 1), r["a_flow12"][y, x], "flow12 of hypothesis %d" % i)
        d = r["decided"][y, x]
        G.check(mo[sel][d], (r["match"] * r["inside"])[y, x][d], (r["a_match"] * r["inside"])[y, x][d], "match of hypothesis %d" % i)


def _run_golden(name, root, dist_out=None):
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, name, root)
    multiH, th, mth, dataset, onlyCoarse = CO.case_args(extra)
    run = lambda: rf.corr_results.get_results(df, imgs, fine, coarse, multiH, th, mth, dataset, onlyCoarse,
                                              int(GOLD["min_size"]), dist_out=dist_out)
    return run, mth, err


@pytest.mark.parametrize("name", CASES)
def test_get_results_against_golden(name, tmp_path):
    dists = []
    run, mth, err = _run_golden(name, str(tmp_path), dists)
    if err:
        with pytest.raises(Exception) as e:
            run()
        assert type(e.value).__name__ == err.split(":")[0]
        if not err.startswith("IndexError"):
            assert "%s: %s" % (type(e.value).__name__, e.value) == err
        return
    res = run()
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        rf.corr_results.print_results(res, mth)
    assert out.getvalue().splitlines() == [str(l) for l in GOLD["%s_stdout" % name]][4:]
    # per keypoint: the golden's distances (selected keypoints, repeats collapsed) against dist_out
    k = 0
    for p, d in enumerate(dists):
        if d is None:
            continue
        for q in range(len(mth)):
            pt, gidx, gd = (GOLD["%s_call%d_%s" % (name, k, s)] for s in ("pair_th", "index", "dist"))
            assert pt[0] == p and pt[1] == mth[q]
            uniq, first = np.unique(gidx, return_index=True)
            rest = np.setdiff1d(np.arange(len(d)), uniq)
            assert np.isnan(d[rest, q]).all()                   # not selected (a selected one may have a NaN flow)
            np.testing.assert_allclose(d[uniq, q], gd[first], rtol=0, atol=1e-4, equal_nan=True)
            k += 1
    assert k == int(GOLD["%s_ncalls" % name])


def test_loop_does_not_synchronise(tmp_path):
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, "sq_mth", str(tmp_path))
    multiH, th, mth, dataset, onlyCoarse = CO.case_args(extra)
    scores = rf.corr_results.CorrScores(mth, th, multiH, onlyCoarse)
    flowList = os.listdir(fine)
    m = int(GOLD["min_size"])
    inputs = []
    for i in range(len(df)):
        kpts, (Isw, Ish), (Itw, Ith) = rf.corr_results.pair_keypoints(df, i, imgs, dataset, m)
        inputs.append((kpts, (Isw, Ish), (Itw, Ith), rf.corr_results._pair_files(i, fine, coarse, fine, flowList, onlyCoarse)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i, (kpts, (Isw, Ish), (Itw, Ith), files) in enumerate(inputs):
            if files is None:
                scores.missing(len(kpts[0]))
                continue
            flow, param, match = files
            scores.queue(flow, param, match, rf.corr_results.truncate_keypoints(*kpts), (Ith, Itw), (Ish, Isw), i)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res = scores.result()
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        rf.corr_results.print_results(res, mth)
    assert out.getvalue().splitlines() == [str(l) for l in GOLD["sq_mth_stdout"]][4:]


def test_cli_subprocess(tmp_path):
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, "md_multi", str(tmp_path))
    csv = str(tmp_path / "test.csv")
    df.to_csv(csv, index=False)
    cmd = [sys.executable, "-m", "ransac_flow_b200.corr_results"] + extra + ["--minSize", str(int(GOLD["min_size"])),
                                                                             "--finePth", fine, "--coarsePth", coarse,
                                                                             sub, "--testDir", imgs, "--testCSV", csv]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == [str(l) for l in GOLD["md_multi_stdout"]]


def _eval_dataset(root):
    """Two synthetic 96 x 128 pairs with keypoints near the identity."""
    import pandas as pd
    import PIL.Image as Image
    from oracle import synth
    os.makedirs(os.path.join(root, "imgs"), exist_ok=True)
    rs = np.random.RandomState(5)
    rows = []
    for p, seed in enumerate((21, 22)):
        src, tgt, _ = synth.make_pair(seed, 96, 128)
        Image.fromarray(src).save(os.path.join(root, "imgs", "s%d.png" % p))
        Image.fromarray(tgt).save(os.path.join(root, "imgs", "t%d.png" % p))
        xb, yb = rs.uniform(0, 127, 50), rs.uniform(0, 95, 50)
        f = lambda a: ";".join("%.3f" % v for v in a)
        rows.append(dict(scene="/", source_image="s%d.png" % p, target_image="t%d.png" % p, XA=f(xb + rs.normal(0, 2, 50)),
                         YA=f(yb + rs.normal(0, 2, 50)), XB=f(xb), YB=f(yb)))
    return pd.DataFrame(rows, dtype=str), os.path.join(root, "imgs")


@pytest.mark.parametrize("engine,begin", [("fp32", 0), ("f16x3", 0), ("fp32", 1)])
def test_evaluate_equals_files_path(engine, begin, tmp_path):
    """``begin`` = 1: pair 0 is not aligned, and is scored as getResults.py scores a row without files."""
    from oracle import synth
    df, imgs = _eval_dataset(str(tmp_path))
    mk = lambda: rf.CoarseAlignA(3, 1000, 0.05, "Homography", 96, 2, False, 2, True, False,
                                 resnet_state_dict=synth.resnet50_conv4_state(0), verbose=False)
    old = rf.model.get_engine()
    rf.model.set_engine(engine)
    try:
        net = {"netFeatCoarse": rf.model.FeatureExtractor(), "netCorr": rf.model.CorrNeigh(7),
               "netFlowCoarse": rf.model.NetFlowCoarse(7), "netMatch": rf.model.NetMatchability(7)}
        for key, sd in (("netFeatCoarse", synth.feature_extractor_state(0)), ("netFlowCoarse", synth.net_flow_coarse_state(1)),
                        ("netMatch", synth.net_matchability_state(2))):
            net[key].load_state_dict(sd)
        for m in net.values():
            m.cuda()
            m.eval()
        mth = [0, 0.0]                                   # 96 x 128: a threshold > 0 raises the reference's broadcast error
        torch.manual_seed(0)
        res = rf.corr_results.evaluate(df, imgs, mk(), net, "MegaDepth", mth, 0.5, True, maxCoarse=3, minSize=96,
                                       beginIndex=begin)
        fine, coarse = str(tmp_path / "out_Fine"), str(tmp_path / "out_Coarse")
        os.makedirs(fine)
        os.makedirs(coarse)
        c = mk()
        torch.manual_seed(0)
        import PIL.Image as Image
        with torch.no_grad():
            for i in range(begin, len(df)):
                Is = Image.open(os.path.join(imgs, df["source_image"][i])).convert("RGB")
                It = Image.open(os.path.join(imgs, df["target_image"][i])).convert("RGB")
                out = rf.pipeline.align_pair_multi(c, net, Is, It, 3, 0.01, with_match21=True)
                rf.results.save_pair(coarse, fine, i, out)
        ref = rf.corr_results.get_results(df, imgs, fine, coarse, True, 0.5, mth, "MegaDepth", minSize=96)
    finally:
        rf.model.set_engine(old)
    assert res.keys() == ref.keys()
    for k in res:
        np.testing.assert_array_equal(res[k][0], ref[k][0])
        assert res[k][1] == ref[k][1] > 0
