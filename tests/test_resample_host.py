"""The PIL resampling tables of the library (``rf_lanczos_coeffs_host``, ``rf_bilinear_coeffs_host``) against Pillow itself.

The tables are host arithmetic, so this runs without a GPU: an integer numpy emulation of Pillow's 8 bits-per-channel pass
(``ss = 2^21 + sum(kk * px)``, ``clip8(ss >> 22)``) driven by the library's bounds and fixed-point weights must equal
``Image.resize`` bit for bit.  The images have a few rows (or columns) only, so Pillow runs the one pass under test and the
emulation is exact for every table: exhaustively for in, out in 1..64, at every size the pipeline resizes to or from, and at a
seeded sample of pairs up to 4000.  The rows hold random bytes and 0 / 255 steps, impulses and checkerboards, which push
LANCZOS overshoot past both ends of ``clip8``.
"""
import ctypes
import math

import numpy as np
import PIL.Image as Image
import pytest

FILTERS = {"lanczos": ("rf_lanczos_coeffs_host", Image.LANCZOS, 3.0), "bilinear": ("rf_bilinear_coeffs_host", Image.BILINEAR, 1.0)}


def tables(rf, fn, insz, outsz):
    """(bounds [out][2], kk [out][ksize]) from the library."""
    f = getattr(rf._lib.lib, fn)
    ks = ctypes.c_int(0)
    assert f(insz, outsz, None, None, 0, ctypes.byref(ks)) == 0
    b = np.zeros(2 * outsz, np.int32)
    kk = np.zeros(ks.value * outsz, np.int32)
    assert f(insz, outsz, b.ctypes.data_as(ctypes.c_void_p), kk.ctypes.data_as(ctypes.c_void_p), kk.size, ctypes.byref(ks)) == 0
    return b.reshape(outsz, 2), kk.reshape(outsz, ks.value)


def emulate_pass(src, bounds, kk):
    """One 8bpc pass along axis 0 of ``src`` (uint8 [in, ...]): out[o] = clip8(2^21 + sum_j kk[o, j] src[lo_o + j])."""
    n_in = src.shape[0]
    j = np.arange(kk.shape[1])
    idx = bounds[:, :1] + j[None, :]
    used = j[None, :] < bounds[:, 1:]
    w = np.where(used, kk, 0).astype(np.int64)
    x = src.astype(np.int64)[np.clip(idx, 0, n_in - 1)]                # [out, ksize, ...]
    acc = (1 << 21) + np.einsum("ok,ok...->o...", w, x)
    return np.clip(acc >> 22, 0, 255).astype(np.uint8)


def content(rs, n, cols):
    """[n, cols] uint8 lines along the resampled axis: random, a 0 / 255 step, an impulse, a checkerboard, random 0 / 255."""
    lines = [rs.randint(0, 256, n), np.where(np.arange(n) < n // 2, 0, 255), np.eye(1, n, n // 2)[0] * 255,
             np.where(np.arange(n) % 2, 255, 0), rs.randint(0, 2, n) * 255, 255 - np.eye(1, n, (n - 1) // 3)[0] * 255]
    a = np.stack([lines[i % len(lines)] for i in range(cols)], 1)
    return a.astype(np.uint8)


def check_pair(rf, name, insz, outsz, rs, channels=3):
    """Both axes, both image modes: the horizontal pass on a (rows, in) image and the vertical pass on an (in, cols) image."""
    fn, flt, _ = FILTERS[name]
    b, kk = tables(rf, fn, insz, outsz)
    lines = content(rs, insz, 6 * channels)                                              # [in, 6 * ch]
    for axis in (0, 1):
        img = lines.reshape(insz, 6, channels) if axis == 0 else lines.reshape(insz, 6, channels).transpose(1, 0, 2)
        img = np.ascontiguousarray(img if channels == 3 else img[..., 0])
        got = emulate_pass(np.moveaxis(img, axis, 0), b, kk)
        got = np.moveaxis(got, 0, axis)
        size = (img.shape[1], outsz) if axis == 0 else (outsz, img.shape[0])
        ref = np.asarray(Image.fromarray(img, "RGB" if channels == 3 else "L").resize(size, resample=flt))
        if not np.array_equal(got, ref):
            bad = np.argwhere(got != ref)[0]
            raise AssertionError("%s %d -> %d (axis %d, %d channel(s)): first difference at %s: table %d, Pillow %d"
                                 % (name, insz, outsz, axis, channels, bad.tolist(), got[tuple(bad)], ref[tuple(bad)]))


def pipeline_resizes():
    """(filter, (w, h) in, (w, h) out, channels) of every resize the pipeline runs at the benchmark's and drivers' sizes, from
    the library's own size functions: the LANCZOS pyramids and targets of configs 2-5, the KITTI fine levels, YFCC's four
    rotated targets, segNet's BILINEAR passes and the BILINEAR sky-mask resize to each target."""
    from ransac_flow_b200 import coarseAlignFeatMatch as ca
    from ransac_flow_b200 import pipeline, segnet
    out = []
    for cls, (w, h), nbScale, scaleR, minSize in ((ca.CoarseAlignA, (640, 480), 7, 2, 480), (ca.CoarseAlignA, (1241, 376), 3, 1.2, 800),
                                                  (ca.CoarseAlignC, (640, 480), 7, 2, 480), (ca.CoarseAlignB, (640, 480), 7, 2, 480)):
        c = cls.__new__(cls)
        c.strideNet = 16
        sizes = [c._target_size(w, h, int(minSize * s)) for s in ca.scale_list(nbScale, scaleR)] + [c._target_size(w, h, minSize)]
        out += [("lanczos", (w, h), s, 3) for s in sizes]
        out.append(("bilinear", (w, h), c._target_size(w, h, minSize), 1))                        # the sky mask of the target
        if cls is ca.CoarseAlignB:                                                                 # YFCC: It rotated by 90 k
            for k in range(4):
                rw, rh = (w, h) if k % 2 == 0 else (h, w)
                out += [("lanczos", (rw, rh), c._target_size(rw, rh, minSize), 3), ("bilinear", (rw, rh), c._target_size(rw, rh, minSize), 1)]
    for fineSize in (650, 325):
        out.append(("lanczos", (1241, 376), pipeline.fine_sizes(1241, 376, 8, fineSize), 3))
    for h, w in ((480, 640), (376, 1241)):
        out += [("bilinear", (w, h), (sw, sh), 3) for sh, sw in segnet.scale_sizes(h, w)]
    return out


def pipeline_axis_pairs():
    """The distinct (filter, in, out) of one pass among ``pipeline_resizes``."""
    pairs = set()
    for name, (w, h), (ow, oh), _ in pipeline_resizes():
        pairs |= {(name, w, ow), (name, h, oh)}
    return sorted(pairs)


@pytest.mark.parametrize("name", list(FILTERS))
def test_tables_match_pillow_exhaustive_small(rf, name):
    rs = np.random.RandomState(0)
    for insz in range(1, 65):
        for outsz in range(1, 65):
            check_pair(rf, name, insz, outsz, rs)


@pytest.mark.parametrize("name", list(FILTERS))
def test_tables_match_pillow_at_pipeline_sizes(rf, name):
    rs = np.random.RandomState(1)
    pairs = [(i, o) for n, i, o in pipeline_axis_pairs() if n == name]
    assert len(pairs) >= (20 if name == "lanczos" else 8), pairs
    for insz, outsz in pairs:
        check_pair(rf, name, insz, outsz, rs)
        check_pair(rf, name, insz, outsz, rs, channels=1)


@pytest.mark.parametrize("name", list(FILTERS))
def test_tables_match_pillow_sampled_to_4000(rf, name):
    rs = np.random.RandomState(2)
    pairs = [(1241, 3), (3, 1241), (4000, 1), (1, 4000), (4000, 3999), (3999, 4000)]
    pairs += [tuple(int(v) for v in rs.randint(1, 4001, 2)) for _ in range(60)]
    pairs += [(int(i), max(1, int(i * r))) for i, r in zip(rs.randint(1, 4001, 30), rs.uniform(0.05, 3.0, 30))]
    for insz, outsz in pairs:
        check_pair(rf, name, insz, outsz, rs, channels=1 + 2 * (insz % 2))


@pytest.mark.parametrize("name", list(FILTERS))
def test_size_query_and_capacity_refusal(rf, name):
    """The size query writes Pillow's ksize = 2 ceil(support max(in / out, 1)) + 1 and touches nothing else; a kk buffer one
    entry short of ksize * out, and a zero size, are refused with a message instead of written past."""
    fn, _, support = FILTERS[name]
    f = getattr(rf._lib.lib, fn)
    for insz, outsz in ((1, 1), (1241, 3), (3, 1241), (640, 480), (480, 240), (7, 5)):
        ks = ctypes.c_int(-1)
        assert f(insz, outsz, None, None, 0, ctypes.byref(ks)) == 0
        assert ks.value == 2 * int(math.ceil(support * max(insz / outsz, 1.0))) + 1, (insz, outsz, ks.value)
        b = np.full(2 * outsz, -7, np.int32)
        kk = np.full(ks.value * outsz, -7, np.int32)
        rc = f(insz, outsz, b.ctypes.data_as(ctypes.c_void_p), kk.ctypes.data_as(ctypes.c_void_p), kk.size - 1, ctypes.byref(ks))
        assert rc != 0 and b"kk buffer too small" in rf._lib.lib.rf_last_error_string()
        assert (b == -7).all() and (kk == -7).all(), "a refused call wrote its tables"
    for insz, outsz in ((0, 5), (5, 0), (-1, 3)):
        ks = ctypes.c_int(0)
        assert f(insz, outsz, None, None, 0, ctypes.byref(ks)) != 0
        assert b"bad sizes" in rf._lib.lib.rf_last_error_string()


def test_pipeline_resize_list_follows_the_code(rf):
    """The size list the tests above and the device resampler tests walk: the benchmark's pyramids and targets are in it."""
    r = pipeline_resizes()
    assert ("lanczos", (640, 480), (1280, 960), 3) in r and ("lanczos", (640, 480), (320, 240), 3) in r
    assert any(name == "lanczos" and src == (1241, 376) and dst[0] % 16 == 0 and dst[1] % 16 == 0 for name, src, dst, _ in r)
    from ransac_flow_b200 import pipeline
    assert ("lanczos", (1241, 376), pipeline.fine_sizes(1241, 376, 8, 325), 3) in r
