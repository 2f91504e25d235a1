"""Host side of the MegaDepth validation (train/validation.py): the resize rule against the reference's own sizes, the keypoint
scaling and ``int()`` truncation against the integers the reference indexed with, the host ``alignmentError`` mirror, the
theta and keypoint checks, and the CPU restatement (``oracle.validation_oracle``) pinned to the reference's precision vector
and per-keypoint distances (tests/golden/validation_megadepth.npz)."""
import os

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import validation_oracle as VO
from oracle.gen_validation_golden import pair_digest, pair_images


@pytest.fixture(scope="module")
def g():
    return golden("validation_megadepth")


def _rows(g):
    return [{c: str(g["%s%d" % (c, i)]) for c in ("scene", "source_image", "target_image", "XA", "YA", "XB", "YB")}
            for i in range(int(g["n_pairs"]))]


def test_size_rule_is_the_references(rf, g):
    for w, h, nw, nh in g["sweep"].tolist():
        assert rf.validation.resize_min_resolution_size(w, h) == (nw, nh), (w, h)
        assert VO.resize_size(w, h) == (nw, nh), (w, h)


def test_size_rule_floors_after_a_half_to_even_round(rf):
    # 128 x 166: 166 / (128 / 480) = 622.5 -> round() = 622 -> 608; pipeline.fine_sizes rounds 622.5 / 16 instead: 624
    assert rf.validation.resize_min_resolution_size(128, 166) == (480, 608)
    assert rf.pipeline.fine_sizes(128, 166, 16, 480) == (480, 624)
    # 500 x 333: 500 / (333 / 480) = 720.72... -> 721 -> floor to 720 (not 736)
    assert rf.validation.resize_min_resolution_size(500, 333) == (720, 480)


def test_images_regenerate(g):
    for i in range(int(g["n_pairs"])):
        assert pair_digest(*pair_images(g["spec%d" % i])) == str(g["sha%d" % i])


def test_keypoint_truncation_is_the_references(rf, g):
    V = rf.validation
    for i, row in enumerate(_rows(g)):
        ws0, hs0, wt0, ht0, _ = g["spec%d" % i].tolist()
        ws, hs = V.resize_min_resolution_size(ws0, hs0)
        wt, ht = V.resize_min_resolution_size(wt0, ht0)
        Xs, Ys = V.scale_keypoints(row["XA"], row["YA"], ws0, hs0, ws, hs)
        Xt, Yt = V.scale_keypoints(row["XB"], row["YB"], wt0, ht0, wt, ht)
        assert Xs.dtype == np.float32 and Yt.dtype == np.float32
        k = V.truncate_keypoints(Xs, Ys, Xt, Yt, ht, wt)
        assert k.dtype == np.int32
        np.testing.assert_array_equal(k, g["kpts%d" % i])


def test_the_golden_covers_its_edges(g):
    ks = [g["kpts%d" % i] for i in range(int(g["n_pairs"]))]
    assert any((k[:, 2] < 0).any() for k in ks)                       # a negative target index (torch wraps it)
    for i, k in enumerate(ks):
        ws0, hs0, wt0, ht0, _ = g["spec%d" % i].tolist()
        wt, ht = VO.resize_size(wt0, ht0)
        assert (k[:, 2] == wt - 1).any() and (k[:, 3] == ht - 1).any(), i   # last column and last row
    assert (np.abs(g["theta2"][:, 2]) > 0.25).all()                    # the partly-outside theta


def test_oracle_matches_the_reference(g):
    """The CPU restatement reproduces the reference's precision vector exactly and its distances to 1e-6 px."""
    from oracle import synth
    states = {"netFeatCoarse": synth.feature_extractor_state(int(g["feat_seed"])),
              "netFlowCoarse": synth.net_flow_coarse_state(int(g["flow_seed"]))}
    dists = []
    for i, row in enumerate(_rows(g)):
        Is, It = pair_images(g["spec%d" % i])
        d = VO.pair_distances(Is, It, g["theta%d" % i], row["XA"], row["YA"], row["XB"], row["YB"], states)
        np.testing.assert_allclose(d, g["dist%d" % i], rtol=0, atol=1e-6)
        dists.append(d)
    np.testing.assert_array_equal(VO.precision(dists), g["prec"])


def test_alignment_error_mirror(rf, g):
    """The host ``alignmentError`` on a full flow: the reference's counts, torch's index rule and its IndexError."""
    V = rf.validation
    rs = np.random.RandomState(0)
    hB, wB, hA, wA = 48, 64, 40, 56
    flow = torch.from_numpy(rs.uniform(-1.1, 1.1, (1, hB, wB, 2)).astype(np.float32))
    XB = np.array([0, 63.9, -1.2, 10.5, -64], dtype=np.float32)
    YB = np.array([0, 47.5, -48, 3.7, 5], dtype=np.float32)
    XA = rs.uniform(0, wA, 5).astype(np.float32)
    YA = rs.uniform(0, hA, 5).astype(np.float32)
    counts, n = V.alignmentError(wB, hB, wA, hA, XA, YA, XB, YB, flow, V.PIXEL_GRID)
    f = flow[0].numpy().astype(np.float32)
    want = []
    for j in range(5):
        xb, yb = int(XB[j]), int(YB[j])
        ex = (f[yb, xb, 0] + np.float32(1)) * np.float32(0.5) * np.float32(wA - 1)
        ey = (f[yb, xb, 1] + np.float32(1)) * np.float32(0.5) * np.float32(hA - 1)
        want.append(((float(ex) - int(XA[j])) ** 2 + (float(ey) - int(YA[j])) ** 2) ** 0.5)
    assert n == 5
    np.testing.assert_array_equal(counts, np.sum(np.array(want).reshape(-1, 1) < V.PIXEL_GRID, axis=0))
    with pytest.raises(IndexError):
        V.alignmentError(wB, hB, wA, hA, XA[:1], YA[:1], np.float32([64.0]), np.float32([0.0]), flow, V.PIXEL_GRID)
    with pytest.raises(IndexError):
        V.alignmentError(wB, hB, wA, hA, XA[:1], YA[:1], np.float32([0.0]), np.float32([-49.0]), flow, V.PIXEL_GRID)


def test_truncation_raises_as_the_reference(rf):
    V = rf.validation
    f = lambda *a: [np.asarray(v, dtype=np.float32) for v in a]
    np.testing.assert_array_equal(V.truncate_keypoints(*f([1.9, -0.5], [2.2, 3.99], [-1.5, 4.7], [0.2, -7.9]), 10, 10),
                                  [[1, 2, -1, 0], [0, 3, 4, -7]])
    with pytest.raises(ValueError):
        V.truncate_keypoints(*f([np.nan], [1], [1], [1]), 10, 10)
    with pytest.raises(OverflowError):
        V.truncate_keypoints(*f([1], [1], [np.inf], [1]), 10, 10)
    with pytest.raises(IndexError):            # keypoint 0's target index fails before keypoint 1's NaN, as in the reference
        V.truncate_keypoints(*f([1, np.nan], [1, 1], [12, 1], [1, 1]), 10, 10)
    with pytest.raises(IndexError):            # XA shorter than XB
        V.truncate_keypoints(*f([1], [1, 1], [1, 1], [1, 1]), 10, 10)
    assert V.truncate_keypoints(*f([], [], [], []), 10, 10).shape == (0, 4)
    big = V.truncate_keypoints(*f([3e9], [1], [-3e9], [1]), 10, 10)
    assert big[0, 0] == np.iinfo(np.int32).max and big[0, 2] == np.iinfo(np.int32).min


def test_theta_is_checked_as_the_reference(rf):
    V = rf.validation
    with pytest.raises(RuntimeError, match="same dtype"):
        V.check_theta(np.eye(2, 3))                                  # float64: grid_sample's dtype mismatch
    with pytest.raises(ValueError):
        V.check_theta(np.eye(3, dtype=np.float32))
    assert V.check_theta(np.eye(2, 3, dtype=np.float32)).dtype == torch.float32


def test_accumulator_layout(rf):
    V = rf.validation
    host = np.zeros(V.PIXEL_GRID.size + 2, dtype=np.int64)
    host[:-1] = np.arange(9)
    host[-1] = V.NO_ERROR
    counts, err = V.read_counts(host)
    assert err is None and counts.tolist() == list(range(9))
    host[-1] = 3
    assert V.read_counts(host)[1] == 3
    assert V.PIXEL_GRID.reshape(-1).tolist() == [1, 2, 3, 5, 8, 13, 22, 36]


def test_pair_inputs_check_theta_before_the_keypoints(rf, tmp_path):
    """The reference's order within a row: the images and the keypoint strings, then ``F.affine_grid`` / ``F.grid_sample``
    on theta, then ``int()`` and the indexing of the keypoints.  A row with both a bad theta and a bad keypoint raises the
    theta's error."""
    import pandas as pd
    import PIL.Image as Image
    V = rf.validation
    os.makedirs(tmp_path / "s")
    Image.fromarray(np.zeros((48, 64, 3), np.uint8)).save(tmp_path / "s" / "a.png")
    row = dict(scene="s", source_image="a.png", target_image="a.png", XA="1;2", YA="1;2", XB="nan;2", YB="1;2")
    df = pd.DataFrame([row], dtype=str)
    eye = np.eye(2, 3, dtype=np.float32)
    with pytest.raises(RuntimeError, match="same dtype"):
        V.pair_inputs(df, 0, str(tmp_path), [eye.astype(np.float64)])
    with pytest.raises(ValueError, match="floating point"):
        V.pair_inputs(df, 0, str(tmp_path), [np.eye(2, 3, dtype=np.int64)])
    with pytest.raises(ValueError, match="Nx2x3"):
        V.pair_inputs(df, 0, str(tmp_path), [np.eye(3, dtype=np.float64)])
    with pytest.raises(ValueError, match="NaN"):
        V.pair_inputs(df, 0, str(tmp_path), [eye])
    df.loc[0, "XB"] = "1;2"
    Is, It, theta, kpts = V.pair_inputs(df, 0, str(tmp_path), [eye])
    assert Is.shape == (48, 64, 3) and theta.dtype == torch.float32 and kpts.tolist() == [[10, 10, 10, 10], [20, 20, 20, 20]]


def test_module_entry_point(rf):
    """``python -m ransac_flow_b200.validation`` runs the module once, as ``__main__`` (the package imports it lazily), and
    the package still exports it."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-W", "error::RuntimeWarning", "-m", "ransac_flow_b200.validation", "--help"], cwd=root,
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "--resumePth" in r.stdout and "RuntimeWarning" not in r.stderr
    assert rf.validation.PIXEL_GRID.size == 8
