"""CPU checks of the segNet mirror: the fp32 oracle against the reference's golden masks (up to proven ties), the pass sizes, the
synthetic weights' activation range (fp16 hi planes), checkpoint key handling, the missing-weights error, the SciPy-1.2 imresize
emulation of the drop-in, the rf_layer_t mirror and the PIL BILINEAR tables."""
import ctypes
import os
import re

import numpy as np
import PIL.Image as Image
import pytest
import torch

from conftest import ROOT, golden
from oracle import seg_oracle as SO
from oracle import synth

IMAGES = ((0, 96, 128), (1, 20, 400))
VARIANTS = ((2, False), (1, True))


@pytest.fixture(scope="module")
def oracle_runs():
    enc, dec = synth.segnet_encoder_state(0), synth.segnet_decoder_state(0)
    out = {}
    for seed, h, w in IMAGES:
        img = Image.fromarray(synth.segnet_image(seed, h, w))
        stats = {}
        for segId, segFg in VARIANTS:
            out[(seed, segId, segFg)] = SO.get_sky(enc, dec, img, segId, segFg, torch.float32, stats)
        out[seed] = stats
    return out


@pytest.mark.parametrize("seed,h,w", IMAGES)
@pytest.mark.parametrize("segId,segFg", VARIANTS)
def test_oracle_matches_reference_golden_up_to_ties(oracle_runs, seed, h, w, segId, segFg):
    g = golden("segnet")
    tag = "%d_%d_%d" % (seed, segId, int(segFg))
    mask, pred, _, sizes = oracle_runs[(seed, segId, segFg)]
    assert [tuple(s) for s in g["sizes_%d" % seed]] == [tuple(s) for s in sizes]
    ref = g["mask_" + tag]
    assert 0.1 <= ref.mean() <= 0.9, "the fixture must give a mask with 10-90 % ones"
    diff = mask != ref
    assert (g["margin12_" + tag][diff] <= 1e-5).all(), (int(diff.sum()), float(g["margin12_" + tag][diff].max()))
    cdiff = pred != g["class_" + tag]
    assert (g["margin12_" + tag][cdiff] <= 1e-5).all()


def test_pass_sizes_repeat_as_documented():
    assert SO.pass_sizes(480, 640) == [(304, 400)] + [(376, 504)] * 4
    assert SO.pass_sizes(376, 1241) == [(152, 504)] * 5


def test_synthetic_weights_keep_activations_in_fp16_range(oracle_runs):
    for seed, _, _ in IMAGES:
        stats = oracle_runs[seed]
        assert len(stats) > 60
        worst = max(stats.values())
        assert worst < 1e3, sorted(stats.items(), key=lambda kv: -kv[1])[:3]


def test_weight_loading_ignores_extras_and_names_missing_keys(rf):
    from ransac_flow_b200 import segnet
    enc, dec = synth.segnet_encoder_state(0), synth.segnet_decoder_state(0)
    assert any("_tmp_running" in k for k in enc) and "conv_last_deepsup.weight" in dec and any("num_batches" in k for k in enc)
    sel = segnet._select(enc, segnet.encoder_keys(), "encoder")
    assert set(sel) == set(segnet.encoder_keys()) and all(v.dtype == torch.float32 for v in sel.values())
    assert not any(k.startswith(("cbr_deepsup", "conv_last_deepsup")) for k in segnet.decoder_keys())
    assert set(segnet.decoder_keys()) <= set(dec)
    del enc["layer3.2.conv2.weight"]
    with pytest.raises(KeyError, match="layer3.2.conv2.weight"):
        segnet._select(enc, segnet.encoder_keys(), "encoder")


def test_missing_weights_error_is_both_file_and_not_implemented(rf, monkeypatch, tmp_path):
    from ransac_flow_b200 import segnet
    assert issubclass(segnet.SegNetWeightsNotFound, FileNotFoundError)
    assert issubclass(segnet.SegNetWeightsNotFound, NotImplementedError)
    monkeypatch.delenv("RF_SEGNET_ENCODER", raising=False)
    monkeypatch.delenv("RF_SEGNET_DECODER", raising=False)
    monkeypatch.chdir(tmp_path)
    with pytest.raises(segnet.SegNetWeightsNotFound):
        segnet.segnet_weights(None)
    e, d = tmp_path / "e.pth", tmp_path / "d.pth"
    e.write_bytes(b"x")
    d.write_bytes(b"x")
    monkeypatch.setenv("RF_SEGNET_ENCODER", str(e))
    monkeypatch.setenv("RF_SEGNET_DECODER", str(d))
    assert segnet.segnet_weights(None) == (str(e), str(d), None)
    assert segnet.segnet_weights(({}, {}))[2] == ({}, {})


def _scipy12_imresize(arr, size):
    """SciPy 1.2 scipy.misc.imresize(arr, (h, w)) restated: toimage (bytescale unless uint8, mode 'L' for 2-D), PIL BILINEAR."""
    a = np.asarray(arr)
    if a.dtype != np.uint8:
        lo, hi = float(a.min()), float(a.max())
        span = (hi - lo) if hi != lo else 1.0
        a = (np.clip((a.astype(np.float64) - lo) * (255.0 / span), 0, 255) + 0.5).astype(np.uint8)
    return np.asarray(Image.fromarray(a, "L" if a.ndim == 2 else "RGB").resize((size[1], size[0]), Image.BILINEAR))


def test_imresize_shim_is_scipy12(rf):
    from ransac_flow_b200 import dropin
    rs = np.random.RandomState(3)
    cases = [(rs.rand(37, 53) > 0.5).astype(np.float32), rs.randint(0, 256, (40, 30)).astype(np.uint8),
             np.ones((21, 17), np.float32), rs.rand(25, 31).astype(np.float32) * 7 - 2, rs.randint(0, 256, (12, 14, 3)).astype(np.uint8)]
    for a in cases:
        for size in ((64, 80), (9, 11), a.shape[:2]):
            got = dropin.imresize(a, size)
            assert got.dtype == np.uint8 and got.shape[:2] == tuple(size)
            assert np.array_equal(got, _scipy12_imresize(a, size)), (a.dtype, a.shape, size)
    m = (rs.rand(30, 40) > 0.5).astype(np.float32)            # evalHpatch's use: a 0 / 1 mask becomes 0 / 255 before the test
    assert set(np.unique(dropin.imresize(m, (30, 40)))) <= {0, 255}
    assert (dropin.imresize(np.ones((8, 8), np.float32), (16, 16)) < 128).all()      # constant input: bytescale gives 0


def test_layer_struct_mirror_matches_header(rf):
    from ransac_flow_b200.program import rf_layer_t
    src = open(os.path.join(ROOT, "include", "ransacflow_b200.h")).read()
    body = re.search(r"typedef struct rf_layer \{(.*?)\} rf_layer_t;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [n.strip() for n in re.sub(r"^(const\s+)?\w+\s*\*?\s*", "", decl).split(",")]
    assert [f[0] for f in rf_layer_t._fields_] == names
    assert names[-1] == "dil"


def _pil_emulate(img, ow, oh, fn):
    cur = img
    for axis, (insz, outsz) in ((1, (img.shape[1], ow)), (0, (img.shape[0], oh))):
        if insz == outsz:
            continue
        ks = ctypes.c_int(0)
        assert fn(insz, outsz, None, None, 0, ctypes.byref(ks)) == 0
        b = np.zeros(2 * outsz, np.int32)
        kk = np.zeros(ks.value * outsz, np.int32)
        assert fn(insz, outsz, b.ctypes.data_as(ctypes.c_void_p), kk.ctypes.data_as(ctypes.c_void_p), kk.size, ctypes.byref(ks)) == 0
        kk = kk.reshape(outsz, ks.value)
        src = np.moveaxis(cur, axis, 0).astype(np.int64)
        out = np.zeros((outsz,) + src.shape[1:], np.int64)
        for o in range(outsz):
            lo, n = b[2 * o], b[2 * o + 1]
            out[o] = np.clip(((1 << 21) + np.tensordot(kk[o, :n].astype(np.int64), src[lo:lo + n], axes=(0, 0))) >> 22, 0, 255)
        cur = np.moveaxis(out.astype(np.uint8), 0, axis)
    return cur


def test_bilinear_coefficients_match_pil(rf):
    img = np.random.RandomState(1).randint(0, 256, (37, 53, 3)).astype(np.uint8)
    for (ow, oh) in [(96, 64), (20, 11), (53, 80), (400, 304)]:
        got = _pil_emulate(img, ow, oh, rf._lib.lib.rf_bilinear_coeffs_host)
        assert np.array_equal(got, np.asarray(Image.fromarray(img).resize((ow, oh), Image.BILINEAR))), (ow, oh)
