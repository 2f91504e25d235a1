"""Host side of the training-pair generator (train/generate_coarse_aligned_pair.ipynb): the notebook's resize rule, its keep
rule and the exceptions it would raise, the writer's layout as data/dataloader.py's ``ImageFolder`` reads it, and the CPU
restatement of the notebook (``oracle.train_pair_oracle``) pinned to the notebook's own outputs (tests/golden/train_pair_*)."""
import os

import numpy as np
import PIL.Image as Image
import pytest
import torch

from conftest import golden
from oracle import pair_oracle as PO
from oracle import synth
from oracle import train_pair_oracle as TO
from train_pair_ref import decided, warp_u8_ref


@pytest.mark.parametrize("w,h", [(720, 480), (730, 480), (480, 720), (1024, 683), (500, 333), (96, 64), (1001, 999)])
def test_sizes_are_resizeImg(rf, w, h):
    """cell 7: the three source scales (and the target at minSize) are ``outil.resizeImg``'s sizes, from the size alone."""
    I = Image.fromarray(np.zeros((h, w, 3), dtype=np.uint8))
    want = [PO.resize_img(I, 16, m).size for m in (240, 480, 960)]
    assert rf.train_pairs.train_pair_sizes(w, h, 480) == want


def test_size_rule_rounds_half_to_even(rf):
    # 720 x 480 at minSize 240: 720 / 2 / 16 = 22.5 -> round() = 22 -> 352 (not 368); 730 x 480 at 480: 736 (ResizeMinSize: 720)
    assert rf.train_pairs.train_pair_sizes(720, 480, 480)[0] == (352, 240)
    assert rf.train_pairs.train_pair_sizes(730, 480, 480)[1] == (736, 480)
    assert rf.coarseAlignFeatMatch.CoarseAlignA._target_size(type("M", (), {"resize_mode": "min", "strideNet": 16})(), 730, 480, 480) == (720, 480)


def test_keep_rule_and_notebook_exceptions(rf):
    T, OK, NONE, NO_MODEL, TOO_FEW = rf.train_pairs, 0, 1, 2, 3
    # (status, M) -> (kept, what the notebook raises)
    table = [((OK, 51), (True, None)), ((OK, 50), (False, None)), ((OK, 4), (False, None)), ((NONE, 500), (False, None)),
             ((NO_MODEL, 80), (False, "TypeError")), ((TOO_FEW, 3), (False, "TypeError")), ((TOO_FEW, 1), (False, "TypeError")),
             ((TOO_FEW, 0), (False, "RuntimeError"))]
    for (status, M), (kept, exc) in table:
        assert T.keep_pair(status, M) == kept, (status, M)
        assert T.notebook_exception(status, M) == exc, (status, M)


def test_resnet50_state_takes_both_layouts(rf):
    sd = {"conv1.weight": torch.ones(1), "layer1.0.bn1.bias": torch.zeros(2)}
    moco = {"model": {"module." + k: v for k, v in sd.items()}}
    S = rf.coarseAlignFeatMatch.resnet50_state
    assert S(sd) is sd and sorted(S(moco)) == sorted(sd)


class _Fake:
    """An aligner stand-in: pair i is kept when keep[i]; its images are filled with i."""

    def __init__(self, keep):
        self.keep, self.i = keep, 0

    def __call__(self, a, b):
        i, self.i = self.i, self.i + 1
        assert a.dtype == np.uint8 and a.ndim == 3 and b.shape[2] == 3
        img = np.full((32, 48, 3), 10 * i, dtype=np.uint8)
        return dict(kept=self.keep[i], I1=img, I2=255 - img)


def image_folder_items(imgDir):
    """data/dataloader.py:43-60 ``ImageFolder``: cycle 2 without '1_3.jpg', nbImg = len(listdir) // cycle, pair ``index`` is
    '{index}_1.jpg' and '{index}_2.jpg'."""
    cycle = 3 if os.path.exists(os.path.join(imgDir, "1_3.jpg")) else 2
    nbImg = len(os.listdir(imgDir)) // cycle
    return cycle, [(os.path.join(imgDir, "%d_1.jpg" % i), os.path.join(imgDir, "%d_2.jpg" % i)) for i in range(nbImg)]


def test_writer_numbers_kept_pairs_contiguously(rf, tmp_path):
    keep = [False, True, True, False, False, True, False]
    src, tgt, _ = synth.make_pair(0, 40, 56)
    paths = []
    for i in range(len(keep)):                                 # paths and in-memory images both accepted
        p = tmp_path / ("in_%d.png" % i)
        Image.fromarray(src).save(p)
        paths.append((str(p), Image.fromarray(tgt)) if i % 2 else (str(p), str(p)))
    out = tmp_path / "pairs"
    index = rf.results.write_train_pairs(_Fake(keep), paths, str(out), chunk=3)
    assert index == [None, 0, 1, None, None, 2, None]
    assert sorted(os.listdir(out)) == sorted("%d_%d.jpg" % (i, k) for i in range(3) for k in (1, 2))
    cycle, items = image_folder_items(str(out))
    assert cycle == 2 and len(items) == 3
    for n, src_i in enumerate(i for i, k in enumerate(keep) if k):
        a = np.asarray(Image.open(items[n][0]).convert("RGB")).astype(int)
        b = np.asarray(Image.open(items[n][1]).convert("RGB")).astype(int)
        assert a.shape == (32, 48, 3) and abs(a.mean() - 10 * src_i) < 2 and abs(b.mean() - (255 - 10 * src_i)) < 2
    with pytest.raises(ValueError):                            # ImageFolder counts every file: the directory must be empty
        rf.results.write_train_pairs(_Fake(keep), paths, str(out))


def test_oracle_is_the_notebook():
    """The CPU restatement on the notebook's inputs and RANSAC draw gives the notebook's sizes, matches, homography, inlier
    array, keep decision and warped bytes (outside the truncation band of an fp32 evaluation)."""
    rsd = synth.resnet50_conv4_state(0)
    for name in ("train_pair_480", "train_pair_small"):
        g = golden(name)
        o = TO.train_pair(rsd, Image.fromarray(g["src"]), Image.fromarray(g["tgt"]), g["samples"].astype(np.int64), int(g["minSize"]))
        assert [tuple(s) for s in g["sizes"]] == o["sizes"]
        assert o["nbMatch"] == int(g["nbMatch"])
        assert np.array_equal(o["match1"], g["match1"]) and np.array_equal(o["match2"], g["match2"])
        np.testing.assert_allclose(o["H"], g["H"], atol=1e-5, rtol=0)
        assert np.array_equal(o["isInlier"], g["isInlier"]) and o["kept"] == bool(g["kept"])
        if not o["kept"]:
            assert o["I2Sample"] is None and g["I2Sample"].size == 0
            continue
        step = int(g["row_step"])
        w1, h1 = o["sizes"][1]
        It = np.asarray(PO.resize_img(Image.fromarray(g["tgt"]), 16, int(g["minSize"])))
        v, band = warp_u8_ref(g["H"], It, h1, w1)
        v2, _ = warp_u8_ref(o["H"], It, h1, w1)
        band = band + np.abs(v2 - v)
        ok = decided(v, band)[::step]
        got = o["I2Sample"][::step]
        assert ok.mean() > 0.9
        assert np.array_equal(got[ok], g["I2Sample"][ok]) and np.array_equal(g["I2Sample"][ok], np.floor(v[::step][ok]))
