"""The training-pair generator on the device (train/generate_coarse_aligned_pair.ipynb): the fused warp kernel bit for bit
against the composition it replaces and within its fp64 bound, ``align_train_pair`` against the notebook's own outputs
(tests/golden/train_pair_*), the writer on a rejected pair, and the graphed aligner against the eager path."""
import os

import numpy as np
import PIL.Image as Image
import pytest
import torch

from conftest import golden
from oracle import outil_oracle as OO
from oracle import pair_oracle as PO
from oracle import synth
from oracle import train_pair_oracle as TO
import geometry_ref as G
from test_gpu_parity import tie_report
from train_pair_ref import decided, warp_u8_ref

pytestmark = pytest.mark.gpu
PREC = {"fp32": 0, "f16x3": 2}


@pytest.fixture
def engine(request, rf):
    rf.model.set_engine(request.param)
    rf.outil.corr_precision = PREC[request.param]
    yield request.param
    rf.model.set_engine("fp32")
    rf.outil.corr_precision = 0


def composition(rf, H, src, h, w):
    """What ``rf_warp_sample_u8`` replaces: warp_grid -> preproc_u8(normalize=False) -> grid_sample -> (x * 255).byte()."""
    Hin, Win = src.shape[:2]
    grid = rf.ops.warp_grid(H.view(1, 3, 3), h, w)
    t = rf.ops.preproc_u8(src.reshape(-1, 3), normalize=False).view(1, Hin, Win, 3).permute(0, 3, 1, 2)
    s = rf.ops.grid_sample(t, grid)
    return (s * 255).to(torch.uint8)[0].permute(1, 2, 0).contiguous()


def homographies():
    rs = np.random.RandomState(5)
    out = {"identity": np.eye(3), "near": np.eye(3) + rs.uniform(-0.05, 0.05, (3, 3)),
           "partly_outside": np.array([[1.4, 0.1, 0.35], [-0.05, 1.3, -0.3], [0.08, -0.06, 1.0]]),     # maps beyond [-1, 1]
           "perspective": np.array([[0.9, 0.0, 0.0], [0.0, 0.9, 0.0], [0.7, 0.5, 1.0]]),              # pz crosses 0 nowhere near
           "zero": np.zeros((3, 3)),                                                                    # a failed RANSAC's H
           "nan": np.full((3, 3), np.nan), "inf": np.array([[np.inf, 0, 0], [0, 1, 0], [0, 0, 1]])}
    return {k: torch.from_numpy(v.astype(np.float32)).reshape(-1).cuda() for k, v in out.items()}


SHAPES = [((37, 53), (29, 71)), ((64, 96), (64, 96)), ((480, 720), (480, 720)), ((1, 1), (5, 3)), ((255, 257), (17, 301)),
          ((160, 240), (480, 720))]


@pytest.mark.parametrize("src_hw,out_hw", SHAPES)
def test_warp_sample_equals_its_composition(rf, src_hw, out_hw):
    """Bit for bit, on every pixel: partial 256-thread blocks, odd sizes, source and output of different shapes, homographies
    mapping partly outside the image, and non-finite ones (zeros: nothing is sampled)."""
    rs = np.random.RandomState(src_hw[0] * 1000 + out_hw[1])
    src = torch.from_numpy(rs.randint(0, 256, src_hw + (3,), dtype=np.uint8)).cuda()
    h, w = out_hw
    for name, H in homographies().items():
        got = rf.train_pairs.warp_sample_u8(H, src, h, w)
        want = composition(rf, H, src, h, w)
        torch.cuda.synchronize()
        assert got.shape == (h, w, 3) and torch.equal(got, want), (name, int((got != want).sum()))
        if name in ("nan", "inf", "zero"):
            assert int(got.max()) == 0, name


@pytest.mark.parametrize("src_hw,out_hw", SHAPES[:3] + SHAPES[4:])
def test_warp_sample_vs_fp64(rf, src_hw, out_hw):
    """Every byte differing from fp64's truncation lies within the sampling bound of tests/geometry_ref.py (at the kernel's own
    fp32 grid, so the bound is the sampling's alone) and differs by one."""
    rs = np.random.RandomState(src_hw[1] + 7)
    src_np = synth.make_pair(int(rs.randint(100)), *src_hw)[0] if min(src_hw) > 8 else rs.randint(0, 256, src_hw + (3,), dtype=np.uint8)
    src = torch.from_numpy(src_np).cuda()
    h, w = out_hw
    for name, H in homographies().items():
        if name in ("nan", "inf", "zero"):
            continue
        got = rf.train_pairs.warp_sample_u8(H, src, h, w).cpu().numpy().astype(np.int64)
        g32 = G.warp_grid_f32(H.cpu().numpy().reshape(1, 3, 3), h, w)[0]
        v, _ = warp_u8_ref(None, src_np, h, w, grid=(g32[..., 0], g32[..., 1]))
        ref, allow, _ = G.grid_sample_ref((src_np.astype(np.float32) / np.float32(255)).transpose(2, 0, 1)[None], g32[None], False)
        band = 255.0 * allow[0].transpose(1, 2, 0) + 2 * 255.0 * G.U * v
        want = np.floor(v).astype(np.int64)
        off = got != want
        assert not (off & decided(v, band)).any(), (name, int((off & decided(v, band)).sum()))
        assert np.abs(got - want).max() <= 1, name


def trunk_matches(rf, model, g):
    """The device's mutual pairs (source index, target index) on the golden's inputs, by the library calls
    ``align_train_pair`` makes (cell 9 on the ragged batch of cell 7's four images)."""
    T = rf.train_pairs
    I1, I2 = torch.from_numpy(g["src"]).cuda(), torch.from_numpy(g["tgt"]).cuda()
    sizes = [tuple(s) for s in g["sizes"]]
    imgs = [rf.ops.resize_lanczos_u8(I1, w, h) for (w, h) in sizes[:3]] + [rf.ops.resize_lanczos_u8(I2, *sizes[3])]
    feats, _ = rf.coarseAlignFeatMatch.conv4_features(model.net, imgs)
    m_src, m_tgt, cnt, idx1, idx2 = T._matches(feats)
    n = int(cnt.item())
    return m_src[:n].cpu().numpy(), m_tgt[:n].cpu().numpy(), set(zip(idx1[:n].tolist(), idx2[:n].tolist()))


@pytest.mark.parametrize("engine", ["fp32", "f16x3"], indirect=True)
def test_align_train_pair_vs_notebook(rf, engine):
    g = golden("train_pair_480")
    rsd = synth.resnet50_conv4_state(0)
    model = rf.train_pairs.TrainPairModel({"model": {"module." + k: v for k, v in rsd.items()}})     # the MoCo layout
    out = rf.pipeline.align_train_pair(model, g["src"], Image.fromarray(g["tgt"]), samples=g["samples"].astype(np.int64))
    w1, h1 = g["sizes"][1]
    assert np.array_equal(out["I1"].cpu().numpy(), np.asarray(PO.resize_img(Image.fromarray(g["src"]), 16, 480)))
    assert out["I1"].shape == out["I2"].shape == (h1, w1, 3) and out["I2"].dtype == torch.uint8
    assert out["nbMatch"] == int(g["nbMatch"]) and out["status"] == 0
    # the match list: equal up to proven arg-max ties (tests/test_gpu_parity.py's criterion, scores from the oracle's features)
    m_src, m_tgt, got_pairs = trunk_matches(rf, model, g)
    key = lambda a, b: set(map(tuple, np.concatenate([a[:, :2], b[:, :2]], 1).tolist()))
    got, ref = key(m_src, m_tgt), key(g["match2"], g["match1"])
    if got != ref:
        featp, f2 = TO.features(rsd, Image.fromarray(g["src"]), Image.fromarray(g["tgt"]), 480)[2:4]
        i1, i2 = OO.mutualMatching(featp, f2)
        ties = tie_report(featp.T @ f2, set(zip(i1.tolist(), i2.tolist())), got_pairs)
        print("[%s] match sets differ in %d pairs, all within %.3g of a tie" % (engine, len(ties), max(m for _, m in ties)))
        assert all(m <= 2 * 2e-5 + 3e-6 for _, m in ties) and len(ties) <= max(2, len(ref) // 50), ties
    else:
        np.testing.assert_array_equal(m_tgt[:, :2], g["match1"][:, :2])
        np.testing.assert_array_equal(m_src[:, :2], g["match2"][:, :2])
        np.testing.assert_allclose(out["H"], g["H"], atol=1e-5, rtol=0)
        assert np.array_equal(out["isInlier"], g["isInlier"]) and out["nbInlier"] == int(g["nbInlier"])
    assert out["kept"] == bool(g["kept"]) is True
    # the warped target: the notebook's bytes wherever fp64 puts 255 v outside the truncation band
    It = np.asarray(PO.resize_img(Image.fromarray(g["tgt"]), 16, 480))
    v, band = warp_u8_ref(g["H"], It, h1, w1)
    v2, _ = warp_u8_ref(out["H"], It, h1, w1)
    step = int(g["row_step"])
    ok = decided(v, band + np.abs(v2 - v))[::step]
    assert ok.mean() > 0.9
    assert np.array_equal(out["I2"].cpu().numpy()[::step][ok], g["I2Sample"][ok])


def test_small_pair_is_not_kept_and_writes_nothing(rf, tmp_path):
    g = golden("train_pair_small")
    model = rf.train_pairs.TrainPairModel(synth.resnet50_conv4_state(0), minSize=int(g["minSize"]))
    out = rf.pipeline.align_train_pair(model, g["src"], g["tgt"], samples=g["samples"].astype(np.int64))
    assert not out["kept"] and not bool(g["kept"])
    assert out["nbMatch"] == int(g["nbMatch"]) <= 50 and out["status"] == 0
    np.testing.assert_allclose(out["H"], g["H"], atol=1e-5, rtol=0)
    assert np.array_equal(out["isInlier"], g["isInlier"])
    aligner = rf.pipeline.GraphedTrainPairAligner(model)
    index = rf.results.write_train_pairs(aligner, [(g["src"], g["tgt"])], str(tmp_path / "pairs"))
    assert index == [None] and os.listdir(tmp_path / "pairs") == []


def same(a, b):
    for k in ("kept", "status", "nbMatch", "nbInlier"):
        assert a[k] == b[k], k
    assert np.array_equal(a["H"], b["H"]) and np.array_equal(a["isInlier"], b["isInlier"])
    assert torch.equal(a["I1"], b["I1"]) and torch.equal(a["I2"], b["I2"])


def test_graph_replays_equal_the_eager_path(rf):
    """Two input sizes through a one-graph aligner (every size change evicts and recaptures), each replay against the eager
    path drawing from an identically seeded generator."""
    rsd = synth.resnet50_conv4_state(0)
    model_g, model_e = rf.train_pairs.TrainPairModel(rsd, minSize=128), rf.train_pairs.TrainPairModel(rsd, minSize=128)
    aligner = rf.pipeline.GraphedTrainPairAligner(model_g, max_graphs=1)
    gen_g, gen_e = (torch.Generator(device="cuda") for _ in range(2))
    aligner.use_generator(gen_g)
    model_e.sample_generator = gen_e
    P = [tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(51, 96, 128)[:2]),
         tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(52, 112, 160)[:2])]
    for n, (I1, I2) in enumerate([P[0], P[1], P[0], P[0]]):
        aligner.prepare(I1, I2)
        gen_g.manual_seed(10 + n)
        gen_e.manual_seed(10 + n)
        same(aligner(I1, I2), rf.pipeline.align_train_pair(model_e, I1, I2))
        assert len(aligner.graphs) == 1


def test_two_lanes_return_what_one_lane_returns(rf):
    rsd = synth.resnet50_conv4_state(0)
    ca = rf.pipeline.ConcurrentAligner(lambda: (rf.train_pairs.TrainPairModel(rsd, minSize=128), None), lanes=2, seed=3,
                                       make_aligner=rf.pipeline.GraphedTrainPairAligner)
    P = [tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(53, 96, 128)[:2]),
         tuple(torch.from_numpy(a).cuda() for a in synth.make_pair(54, 96, 128)[:2])]
    pairs = [P[0], P[1], P[1], P[0]]
    ca.prepare(*P[0])
    ca.seed(3)
    together = ca.run(pairs)
    ca.seed(3)
    for k in range(2):
        for i in range(k, len(pairs), 2):
            same(ca.lanes[k](*pairs[i]), together[i])
