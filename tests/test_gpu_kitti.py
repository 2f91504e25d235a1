"""KITTI extras (SURVEY 8f-4): the two-level fine flow of evaluation/evalKITTI/evaluation.py, remove_small_cc and the
two-level recomposition of evalKITTI/getResults.py against the unmodified reference's golden outputs and the CPU oracle."""
import numpy as np
import PIL.Image as Image
import pytest
import torch

from conftest import golden
from oracle import pair_oracle as PO
from oracle import synth
from oracle import warp_oracle as WO
from test_gpu_pair import FLOW_TOL, fixed_randint, networks, oracle_net

pytestmark = pytest.mark.gpu


def test_remove_small_cc_vs_reference_golden(rf):
    g = golden("kitti_remove_small_cc")
    for key in ("out_0", "out_0.01", "out_0.05", "out_1"):
        got = rf.pipeline.remove_small_cc(g["match"], float(g["match_th"]), float(key.split("_")[1]))
        assert np.array_equal(got, g[key]), key


@pytest.mark.parametrize("h,w,seed", [(376, 1241, 0), (60, 96, 1), (33, 7, 2), (1, 50, 3), (128, 128, 4)])
def test_remove_small_cc_fuzz_vs_oracle(rf, h, w, seed):
    """Random blobs, spirals of 8-connected diagonals, a batch of three maps, several area thresholds."""
    import scipy.ndimage as nd
    rs = np.random.RandomState(seed)
    maps = []
    for j in range(3):
        raw = nd.gaussian_filter(rs.rand(h, w), 1.0 + j)
        m = ((raw - raw.min()) / max(1e-9, raw.max() - raw.min())).astype(np.float32)
        m = np.where(m > 0.5 + 0.05 * j, 1.0, m).astype(np.float32)
        if h > 8 and w > 8:
            for d in range(min(h, w) // 2):          # a diagonal line: connected only through corners
                m[d, d] = 1.0
        maps.append(m)
    batch = np.stack(maps)
    for cc_th in (0.0, 1e-4, 0.003, 0.01, 0.2):
        ref = np.stack([WO.remove_small_cc(m, 0.99, cc_th) for m in maps])
        got = rf.ops.remove_small_cc(torch.from_numpy(batch.copy()).cuda(), 0.99, cc_th).cpu().numpy()
        assert np.array_equal(got, ref), (cc_th, int((got != ref).sum()))


def test_kitti_pred_flow_mask_vs_reference(rf):
    """evaluation/evalKITTI/evaluation.py:49-81 (second level: coarse flow on 48x64, outputs on 56x80) against the
    unmodified reference's golden output, fp32 engine."""
    g = golden("kitti_pred_flow_mask")
    net = networks(rf)
    flowCoarse = rf.kornia_geometry.HomographyWarper(48, 64).warp_grid(torch.from_numpy(g["H"]).cuda())
    flow12, match, f8, m8 = rf.pipeline.PredFlowMask_kitti(torch.from_numpy(g["IsSample"]).cuda(), torch.from_numpy(g["It"]).cuda(),
                                                          flowCoarse, rf.pipeline.base_grid(56, 80), net)
    assert tuple(f8.shape) == (1, 2, 6, 8) and tuple(m8.shape) == (1, 2, 6, 8) and match.shape == (56, 80)
    assert np.abs(f8.cpu().numpy() - g["flowDown8"]).max() < FLOW_TOL and np.abs(m8.cpu().numpy() - g["matchDown8"]).max() < FLOW_TOL
    d = np.abs(flow12.cpu().numpy() - g["flow12"]).max()
    far = (np.abs(np.abs(g["flow12"]) - 1) > 1e-3).all(-1)[0]
    dm = np.abs(match - g["match"])[far].max()
    print("KITTI PredFlowMask: |flow12 - ref| %.3g, |match - ref| %.3g" % (d, dm))
    assert d < FLOW_TOL and dm < FLOW_TOL


def test_kitti_get_flow_all_vs_reference(rf):
    g = golden("kitti_get_flow_all")
    fg, mb = rf.pipeline.getFlow_all_kitti(g["H"], g["flowd2"], g["flow"], g["mask"], 48, 80, th=float(g["th"]), cc_th=float(g["cc_th"]),
                                           multiH=True)
    ref, rmb = WO.get_flow_all_kitti(g["H"], g["flowd2"], g["flow"], g["mask"], 48, 80, th=float(g["th"]), cc_th=float(g["cc_th"]), multiH=True)
    same = (mb.cpu() == rmb).all(-1)[0]                      # the merge flips only where a matchability sits on the threshold
    assert same.float().mean() > 0.99
    assert np.abs(fg.cpu().numpy() - g["flowGlobal_interp0"])[0][same.numpy()].max() < 1e-5
    # interpolate=True (evalKITTI/getResults.py:87-93): holes take the flow of the nearest matched pixel.  Exact distances;
    # the filled value equals the reference's wherever scipy picked the same (or the unique) nearest pixel
    import scipy.ndimage as nd
    fi, mbi = rf.pipeline.getFlow_all_kitti(g["H"], g["flowd2"], g["flow"], g["mask"], 48, 80, th=float(g["th"]), cc_th=float(g["cc_th"]),
                                            multiH=True, interpolate=True)
    assert torch.equal(mbi, mb)
    holes = ~mb.cpu().numpy()[0, :, :, 0]
    assert holes.any() and (~holes).any()
    d_ref, idx_ref = nd.distance_transform_edt(holes, return_distances=True, return_indices=True)
    _, idx = rf.ops.fill_nearest_matched(fg, mb, want_index=True)
    idx = idx.cpu().numpy()
    yy, xx = np.mgrid[0:48, 0:80]
    assert np.array_equal((idx[..., 0] - yy) ** 2 + (idx[..., 1] - xx) ** 2, np.round(d_ref ** 2).astype(np.int64))
    agree = (idx[..., 0] == idx_ref[0]) & (idx[..., 1] == idx_ref[1]) & same.numpy()
    assert agree.mean() > 0.9
    assert np.abs(fi.cpu().numpy() - g["flowGlobal_interp1"])[0][agree].max() < 1e-5


def test_kitti_two_level_pair_vs_oracle(rf):
    """align_pair_kitti (evaluation/evalKITTI/evaluation.py:216-344) on a KITTI-shaped 96x256 pair against the CPU oracle with
    the same RANSAC samples: identical homographies, both levels' /8 flows and the full-resolution flow within 1e-3."""
    src, tgt, _ = synth.make_pair(41, 96, 256)
    Is, It = Image.fromarray(src), Image.fromarray(tgt)
    rsd = synth.resnet50_conv4_state(0)
    oc = PO.CoarseAlignOracle(rsd, nbScale=3, nbIter=1000, tolerance=0.05, minSize=96, scaleR=1.2, variant="A", seed=1000)
    log, inner = [], oc._ransac

    def recording(m1, m2):
        r = inner(m1, m2)
        log.append(oc.last_samples)
        return r
    oc._ransac = recording
    ref = PO.align_pair_kitti(oc, oracle_net(), Is, It, fineSize=96, cc_th=0.01, maskRegionTh=0.005, maxH=2)
    c = rf.CoarseAlignA(3, 1000, 0.05, "Homography", 96, 2, False, 1.2, True, False, resnet_state_dict=rsd, verbose=False)
    with fixed_randint(log + log[-1:]):
        out = rf.pipeline.align_pair_kitti(c, networks(rf), Is, It, fineSize=96, cc_th=0.01, maskRegionTh=0.005, maxH=2)
    assert out["size"] == ref["size"] == (96, 256)
    nH = len(ref["H"])
    print("KITTI two-level pair: %d hypothesis(es) in the oracle, %d here" % (nH, len(out["H"])))
    assert nH >= 1 and len(out["H"]) == nH
    np.testing.assert_allclose(out["H"], ref["H"], atol=1e-5)
    assert out["flow_d2"].shape == ref["flow_d2"].shape and out["flow"].shape == ref["flow"].shape and out["mask"].shape == ref["mask"].shape
    assert np.abs(out["flow_d2"] - ref["flow_d2"]).max() < FLOW_TOL and np.abs(out["flow"] - ref["flow"]).max() < FLOW_TOL
    assert np.abs(out["mask"] - ref["mask"]).max() < FLOW_TOL
    for (f, m), (rfl, rm) in zip(out["maps"], ref["maps"]):
        assert np.abs(f.cpu().numpy() - rfl.numpy()).max() < FLOW_TOL
        far = (np.abs(np.abs(rfl.numpy()) - 1) > 1e-3).all(-1)[0]
        assert np.abs(m - rm)[far].max() < FLOW_TOL


def test_get_flow_from_the_drivers_files(rf, tmp_path):
    """results.getFlow_all_from_files / getFlow_all_kitti_from_files: the reference's file names (evaluation.py:254-260 and
    evalKITTI/evaluation.py:338-344) read back and composed on the device == the reference's golden getFlow_all outputs."""
    g = golden("get_flow_all")
    fine, coarse = tmp_path / "fine", tmp_path / "coarse"
    fine.mkdir()
    coarse.mkdir()
    out = dict(H=g["H"], flowDown8=g["flow"], matchDown8=g["mask"])
    assert rf.results.save_pair(str(coarse), str(fine), 0, out) == 2
    fg = rf.results.getFlow_all_from_files(0, str(fine), str(coarse), sorted(p.name for p in fine.iterdir()), True, float(g["th"]), 56, 40)
    ref, m = WO.get_flow_all(g["flow"], g["H"], g["mask"], 40, 56, th=float(g["th"]), multiH=True)
    far = (np.abs(m.numpy() - float(g["th"])) > 1e-4).all(0)[..., 0]
    assert np.abs(fg.cpu().numpy() - g["flowGlobal"])[0][far].max() < 1e-5
    assert rf.results.getFlow_all_from_files(9, str(fine), str(coarse), sorted(p.name for p in fine.iterdir()), True, 0.5, 56, 40) == []
    k = golden("kitti_get_flow_all")
    kd = tmp_path / "kitti"
    kd.mkdir()
    assert rf.results.save_pair_kitti(str(kd), 7, dict(H=k["H"], flow_d2=k["flowd2"], mask=k["mask"], flow=k["flow"], size=(48, 80))) == 2
    pid, nbH = list(rf.results.kitti_pairs(str(kd)).items())[0]
    fk = rf.results.getFlow_all_kitti_from_files(pid, str(kd), nbH, "Finetune", 48, 80, True, float(k["th"]), float(k["cc_th"]))
    d = np.abs(fk.cpu().numpy() - k["flowGlobal_interp0"])[0].max(-1)
    assert (d < 1e-5).mean() > 0.99                       # merge picks flip only where a matchability sits on the threshold


@pytest.mark.parametrize("h,w,p,seed", [(376, 1241, 0.3, 0), (376, 1241, 0.001, 1), (60, 96, 0.05, 2), (1, 40, 0.2, 3), (37, 1, 0.3, 4),
                                        (64, 64, 0.9, 5), (20, 30, 0.0, 6)])
def test_fill_nearest_matched_is_exact(rf, h, w, p, seed):
    """rf_fill_nearest_matched vs scipy's exact EDT: every pixel is filled from a MATCHED pixel at exactly the EDT distance
    (ties between equidistant pixels may be resolved differently), matched pixels keep their own flow; p = 0 (nothing
    matched) leaves the flow unchanged."""
    import scipy.ndimage as nd
    rs = np.random.RandomState(seed)
    m = rs.rand(h, w) < p
    flow = torch.from_numpy(rs.randn(1, h, w, 2).astype(np.float32)).cuda()
    out, idx = rf.ops.fill_nearest_matched(flow, torch.from_numpy(m).cuda(), want_index=True)
    out, idx, f = out.cpu().numpy(), idx.cpu().numpy().astype(np.int64), flow.cpu().numpy()
    if not m.any():
        assert np.array_equal(out, f)
        return
    d = nd.distance_transform_edt(~m)
    yy, xx = np.mgrid[0:h, 0:w]
    assert m[idx[..., 0], idx[..., 1]].all()
    assert np.array_equal((idx[..., 0] - yy) ** 2 + (idx[..., 1] - xx) ** 2, np.round(d ** 2).astype(np.int64))
    assert np.array_equal(out[0], f[0][idx[..., 0], idx[..., 1]])
    assert np.array_equal(out[0][m], f[0][m])


def test_get_flow_corr_vs_reference(rf, tmp_path):
    """pipeline.getFlow_corr / results.getFlow_from_files (evaluation/evalCorr/getResults.py:78-134) vs the reference's golden
    flowGlobal / matchGlobal, away from the merge threshold."""
    g = golden("get_flow_corr")
    fg, mg = rf.pipeline.getFlow_corr(g["flow"], g["H"], g["mask"], th=float(g["th"]), multiH=True)
    assert tuple(fg.shape) == (1, 40, 56, 2) and tuple(mg.shape) == (1, 40, 56, 1)
    far = np.abs(g["matchGlobal"][0, :, :, 0] - float(g["th"])) > 1e-3
    assert np.abs(mg.cpu().numpy() - g["matchGlobal"])[0, :, :, 0][far].max() < 1e-5
    d = np.abs(fg.cpu().numpy() - g["flowGlobal"])[0].max(-1)
    assert (d < 1e-5).mean() > 0.98
    fine, coarse = tmp_path / "fine", tmp_path / "coarse"
    fine.mkdir()
    coarse.mkdir()
    rf.results.save_pair(str(coarse), str(fine), 4, dict(H=g["H"], flowDown8=g["flow"], matchDown8=g["mask"]))
    fg2, mg2 = rf.results.getFlow_from_files(4, str(fine), sorted(p.name for p in fine.iterdir()), str(coarse), str(fine), True, float(g["th"]))
    assert np.array_equal(fg2.cpu().numpy(), fg.cpu().numpy()) and np.array_equal(mg2.cpu().numpy(), mg.cpu().numpy())
    assert rf.results.getFlow_from_files(5, str(fine), sorted(p.name for p in fine.iterdir()), str(coarse), str(fine), True, 0.5) == ([], [])
