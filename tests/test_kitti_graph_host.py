"""Host parts of the graphed KITTI pair (``pipeline.align_pair_kitti_graph`` / ``GraphedKittiAligner``): the fine-level sizes,
the acceptance threshold ``kitti_region_cmin``, the unpacking of the per-hypothesis records and the C ABI export.  No GPU."""
import ctypes

import numpy as np
import PIL.Image as Image
import pytest
import torch


@pytest.mark.parametrize("minSize", [650, 325, 96, 48, 100, 7, 8, 13])
def test_fine_sizes_is_resize_img(rf, minSize):
    """Over a sweep of sizes (KITTI's, tiny, tall, wide, square), every (w, h) equals outil.resizeImg's PIL output size."""
    sizes = [(1241, 376), (1242, 375), (1224, 370), (1226, 370), (96, 256), (256, 96), (64, 64), (17, 9), (9, 17), (1000, 3)]
    rs = np.random.RandomState(minSize)
    sizes += [(int(a), int(b)) for a, b in rs.randint(1, 1500, size=(12, 2))]
    for w, h in sizes:
        I = Image.new("RGB", (w, h))
        assert rf.pipeline.fine_sizes(w, h, 8, minSize) == rf.outil.resizeImg(I, 8, minSize).size, (w, h, minSize)


def test_fine_sizes_rounds_half_to_even(rf):
    """w / ratio / 8 lands exactly on .5: Python's round goes to the even neighbour, as in utils/outil.py."""
    cases = []
    for w in range(8, 400):
        for h in (40, 80):
            q = w / (min(w / 40, h / 40)) / 8
            if q == int(q) + 0.5:
                cases.append((w, h))
    assert len(cases) >= 2
    for w, h in cases:
        got = rf.pipeline.fine_sizes(w, h, 8, 40)
        assert got == rf.outil.resizeImg(Image.new("RGB", (w, h)), 8, 40).size
    # 20 x 100 at minSize 100: 100 / 8 = 12.5 -> 12 and 500 / 8 = 62.5 -> 62 (half to even, not half up)
    assert rf.pipeline.fine_sizes(20, 100, 8, 100) == (96, 496) == rf.outil.resizeImg(Image.new("RGB", (20, 100)), 8, 100).size


def brute_cmin(n, th):
    fg = np.zeros(n, dtype=np.float32)
    for c in range(n + 1):
        m = np.zeros(n, dtype=np.float32)
        m[:c] = 1
        if ((m > 0.9999) * (1 - fg)).mean() > th:
            return c
    return n + 1


@pytest.mark.parametrize("n,th", [(1, 0.005), (7, 0.5), (200, 0.005), (1000, 0.005), (1000, 0.01), (999, 0.005), (1024, 0.25),
                                  (2000, 0.0), (300, 1.0), (4096, 0.005), (3000, 0.1)])
def test_cmin_against_brute_force(rf, n, th):
    assert rf.pipeline.kitti_region_cmin(n, th) == brute_cmin(n, th)


def test_cmin_threshold_hit_exactly(rf):
    """count / n == maskRegionTh in float32 (5 / 1000 = 0.005, 1 / 4 = 0.25): the reference's strict `>` rejects that count."""
    assert rf.pipeline.kitti_region_cmin(1000, 0.005) == 6
    assert rf.pipeline.kitti_region_cmin(1024, 0.25) == 257
    assert rf.pipeline.kitti_region_cmin(2000, 0.0) == 1
    assert rf.pipeline.kitti_region_cmin(300, 1.0) == 301


def test_cmin_at_kitti_size(rf):
    """376 x 1241 at the driver's maskRegionTh: cmin is the first count accepted, cmin - 1 is not, and the expression is
    position-independent (the ones scattered over the 2-D map give the same verdict)."""
    n, th = 376 * 1241, 0.005
    c = rf.pipeline.kitti_region_cmin(n, th)
    fg = np.zeros((376, 1241), dtype=np.float32)
    rs = np.random.RandomState(0)
    for cnt, want in ((c - 1, False), (c, True), (c + 1, True)):
        m = np.zeros(n, dtype=np.float32)
        m[rs.choice(n, cnt, replace=False)] = 1
        m = m.reshape(376, 1241)
        assert bool(((m > 0.9999) * (1 - fg)).mean() > th) is want, cnt


def records(alive, status, maxH, d2=(1, 2, 2, 3), f8=(1, 2, 3, 4)):
    nd, n8 = int(np.prod(d2)), int(np.prod(f8))
    rows = []
    for k in range(maxH):
        r = np.concatenate([[alive[k], status[k], 100 + k, 50 + k], np.arange(9) + 10 * k, np.full(nd, k + 0.25), np.full(n8, k + 0.5),
                            np.full(n8, k + 0.75)]).astype(np.float32)
        rows.append(r)
    return np.concatenate(rows), ["map%d" % k for k in range(maxH)], (376, 1241), (d2, f8)


def test_unpack_stops_at_the_first_dead_hypothesis(rf):
    host, maps, size, shapes = records([1, 1, 0, 1, 0], [0, 0, 0, 0, 1], 5)
    out = rf.pipeline._unpack_kitti(host, maps, size, shapes, 5)
    assert out["H"].shape == (2, 3, 3) and out["H"].dtype == np.float32
    assert np.array_equal(out["H"][1].reshape(-1), np.arange(9) + 10)
    assert out["flow_d2"].shape == (2, 2, 2, 3) and (out["flow_d2"][1] == 1.25).all()
    assert out["mask"].shape == (2, 2, 3, 4) and (out["mask"][0] == 0.5).all()
    assert out["flow"].shape == (2, 2, 3, 4) and (out["flow"][1] == 1.75).all()
    assert out["nbMatch"] == [100, 101] and out["nbInlier"] == [50, 51]
    assert out["maps"] == ["map0", "map1"] and out["size"] == (376, 1241) and out["capped"] is False


def test_unpack_capped_and_empty(rf):
    host, maps, size, shapes = records([1] * 4, [0] * 4, 4)
    out = rf.pipeline._unpack_kitti(host, maps, size, shapes, 4)
    assert out["capped"] is True and len(out["H"]) == 4 and len(out["maps"]) == 4
    host, maps, size, shapes = records([0, 0], [1, 0], 2)
    out = rf.pipeline._unpack_kitti(host, maps, size, shapes, 2)
    assert out["H"].shape == (0,) and out["flow"].shape == (0,) and out["maps"] == [] and out["capped"] is False


def test_unpack_raises_on_no_model_before_the_first_dead_hypothesis(rf):
    with pytest.raises(TypeError):                                         # utils/outil.py:162 in the first hypothesis
        rf.pipeline._unpack_kitti(*records([0, 0], [2, 0], 2), 2)
    with pytest.raises(TypeError):                                         # ... and in a later one the reference reaches
        rf.pipeline._unpack_kitti(*records([1, 1, 0], [0, 0, 2], 3), 3)
    out = rf.pipeline._unpack_kitti(*records([1, 0, 0], [0, 1, 2], 3), 3)   # after a stop the reference never gets there
    assert len(out["H"]) == 1


def test_kitti_region_step_is_exported(rf):
    lib = ctypes.CDLL(rf._lib.LIB_PATH)
    for s in ("rf_kitti_region_step", "rf_kitti_region_step_workspace"):
        assert hasattr(lib, s) and s in rf._lib.SIGNATURES
    assert rf._lib.lib.rf_kitti_region_step_workspace(376, 1241) >= 256 * 4 + 4
    assert rf._lib.lib.rf_kitti_region_step_workspace(1, 1) == rf._lib.lib.rf_kitti_region_step_workspace(376, 1241)


def test_kitti_region_step_refuses_host_tensors(rf):
    z = torch.zeros((4, 4))
    i = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(rf._lib.RFError):
        rf.ops.kitti_region_step(z, z, z, z, i, i, True, 1)


def test_graph_kitti_needs_a_cap(rf):
    with pytest.raises(ValueError):
        rf.pipeline.align_pair_kitti_graph(None, None, None, None, maxH=None)
