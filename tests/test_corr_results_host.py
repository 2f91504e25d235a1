"""evalCorr getResults on the host side: the CPU restatement (oracle/corr_results_oracle.py) pinned to the reference's own run
(tests/golden/corr_results.npz, oracle/gen_corr_results_golden.py), and the host rules of ``corr_results``: sizes from the
image headers, the MegaDepth filter, the int64 truncation, the threshold keys, and the command line."""
import contextlib
import io
import os

import numpy as np
import pytest

import ransac_flow_b200 as rf
from oracle import corr_results_oracle as CO

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "corr_results.npz"))
CASES = [str(c) for c in GOLD["cases"]]


def _lines(res, mth):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        rf.corr_results.print_results(res, mth)
    return out.getvalue().splitlines()


def _golden_calls(name):
    return [(GOLD["%s_call%d_pair_th" % (name, k)], GOLD["%s_call%d_index" % (name, k)], GOLD["%s_call%d_dist" % (name, k)])
            for k in range(int(GOLD["%s_ncalls" % name]))]


@pytest.mark.parametrize("name", CASES)
def test_oracle_pinned_to_golden(name, tmp_path):
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, name, str(tmp_path))
    multiH, th, mth, dataset, onlyCoarse = CO.case_args(extra)
    calls = []
    run = lambda: CO.get_results(df, imgs, fine, coarse, multiH, th, mth, dataset, onlyCoarse, int(GOLD["min_size"]), calls)
    if err:
        with pytest.raises(Exception) as e:
            run()
        assert "%s: %s" % (type(e.value).__name__, e.value) == err
    else:
        res = run()
        assert _lines(res, mth) == [str(l) for l in GOLD["%s_stdout" % name]][4:]
    gold = _golden_calls(name)
    assert len(calls) == len(gold)
    for (i, t, idx, d), (pt, gidx, gd) in zip(calls, gold):
        assert (i, t) == (pt[0], pt[1])
        np.testing.assert_array_equal(idx, gidx)
        np.testing.assert_allclose(d, gd, rtol=0, atol=1e-6)


@pytest.mark.parametrize("name", ["md_multi", "rc_multi", "sq_mth"])
def test_sizes_filter_and_truncation(name, tmp_path):
    """``pair_keypoints`` (header sizes, the MegaDepth filter) and ``truncate_keypoints`` against the restatement."""
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, name, str(tmp_path))
    dataset = CO.case_args(extra)[3]
    m = int(GOLD["min_size"])
    edge = wrap = False
    for i in range(len(df)):
        (Xs, Ys, Xt, Yt), (Isw, Ish), (Itw, Ith) = rf.corr_results.pair_keypoints(df, i, imgs, dataset, m)
        path = lambda n: rf.corr_results.image_path(imgs, df["scene"][i], n)
        import PIL.Image as Image
        with Image.open(path(df["source_image"][i])) as im:
            (w, h), xs, ys = CO.resize_keypoints(m, im.size, df["XA"][i], df["YA"][i])
        with Image.open(path(df["target_image"][i])) as im:
            (wt, ht), xt, yt = CO.resize_keypoints(m, im.size, df["XB"][i], df["YB"][i])
        assert (Isw, Ish, Itw, Ith) == (w, h, wt, ht)
        if dataset != "RobotCar":
            v = (xs > 0) * (xs < w) * (ys > 0) * (ys < h) * (xt > 0) * (xt < wt) * (yt > 0) * (yt < ht)
            assert v.sum() < len(v)                              # the golden's keypoints include some the filter drops
            xs, ys, xt, yt = xs[v], ys[v], xt[v], yt[v]
        for a, b in zip((Xs, Ys, Xt, Yt), (xs, ys, xt, yt)):
            assert a.dtype == np.float32
            np.testing.assert_array_equal(a, b)
        k = rf.corr_results.truncate_keypoints(Xs, Ys, Xt, Yt)
        np.testing.assert_array_equal(k, np.stack([a.astype(np.int64) for a in (xs, ys, xt, yt)], axis=1))
        wrap |= bool((k[:, 2] == -1).any())                      # a negative index that wraps
        edge |= bool((k[:, 2] == Itw - 1).any() and (k[:, 3] == Ith - 1).any())   # the last column and row
    assert edge and wrap == (dataset == "RobotCar")


def test_truncation_rule():
    """astype(np.int64): toward zero, negatives kept (numpy wraps them once), beyond int32 clipped out of range."""
    x = np.array([-1.5, -0.5, 0.0, 0.99, 2.5, 3e10], dtype=np.float32)
    k = rf.corr_results.truncate_keypoints(x, x, x, x)
    assert list(k[:, 0]) == [-1, 0, 0, 0, 2, 2 ** 31 - 1]


def test_header_size_only(tmp_path):
    """Sizes come from the header; a file PIL cannot open still raises."""
    import PIL.Image as Image
    p = tmp_path / "a.png"
    Image.new("RGB", (123, 77)).save(p)
    assert rf.corr_results.image_size(str(p)) == (123, 77)
    bad = tmp_path / "b.png"
    bad.write_bytes(b"not an image")
    with pytest.raises(Exception):
        rf.corr_results.image_size(str(bad))


def test_threshold_keys_and_missing_rule_keys():
    """Equal thresholds share one dict entry, as the reference's dicts do; 0 and 0.0 are one key."""
    assert rf.corr_results._keys([0, 0.5, 0.0, 0.5]) == ([0, 0.5], [0, 1, 0, 1])
    assert rf.corr_results._keys([0.5]) == ([0.5], [0])


def _drop_pair(fine, pair):
    for f in os.listdir(fine):
        if f.split("_")[1] == str(pair):
            os.remove(os.path.join(fine, f))


def test_error_order_oracle(tmp_path):
    """The first error wins, in pair order and within a pair in threshold order: every pair has an out-of-range index, so
    threshold 0 raises IndexError at pair 0 before pair 3 (no files) is reached and before threshold 0.5's broadcast
    RuntimeError (a threshold > 0 on a non-square map), which alone raises first; pair 0 without files raises KeyError
    (0 not a threshold) before anything else."""
    df, imgs, fine, coarse, extra, sub, err = CO.case_setup(GOLD, "rc_index", str(tmp_path))
    run = lambda mth: CO.get_results(df, imgs, fine, coarse, False, 0.95, mth, "RobotCar", minSize=int(GOLD["min_size"]))
    _drop_pair(fine, 3)
    with pytest.raises(IndexError):
        run([0, 0.5])
    with pytest.raises(RuntimeError, match="must match the size"):
        run([0.5, 0])
    _drop_pair(fine, 0)
    with pytest.raises(KeyError):
        run([0.5])


def test_argument_parsing():
    p = rf.corr_results.build_parser()
    a = p.parse_args(["--multiH", "--th", "0.9", "--matchabilityTH", "0", "0.5", "--finePth", "f", "--coarsePth", "c",
                      "MegaDepth", "--testDir", "d", "--testCSV", "x.csv", "--beginIndex", "3", "--endIndex", "9"])
    assert (a.multiH, a.th, a.matchabilityTH, a.subcommand, a.testDir, a.beginIndex, a.endIndex) == \
        (True, 0.9, [0.0, 0.5], "MegaDepth", "d", 3, 9)
    assert a.dataset == "MegaDepth" and a.minSize == 480 and a.onlyCoarse is False and a.resumePth is None
    a = p.parse_args(["--dataset", "RobotCar", "--onlyCoarse", "RobotCar"])
    assert (a.subcommand, a.dataset, a.onlyCoarse, a.matchabilityTH, a.th) == ("RobotCar", "RobotCar", True, [0], 0.95)
    assert a.testDir == "../../data/RobotCar/imgs/" and a.testCSV == "../../data/RobotCar/test6511.csv"
    assert not hasattr(a, "beginIndex")
    a = p.parse_args(["--resumePth", "m.pth", "--segNet", "--maxCoarse", "3", "MegaDepth"])
    assert (a.resumePth, a.segNet, a.maxCoarse, a.kernelSize, a.coarseIter, a.nbScale, a.scaleR) == ("m.pth", True, 3, 7, 10000, 7, 2)
