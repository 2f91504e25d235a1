"""The device PIL resampler (``rf_resample_u8``: ``resample_h_kernel``, ``resample_v_kernel`` and the byte-wise fallback
``resample_u8_kernel``) bit for bit against Pillow, for LANCZOS and BILINEAR, 3 and 1 channels.

Sizes: every resize the pipeline runs (``test_resample_host.pipeline_resizes``: the configs' pyramids and targets, the KITTI
fine levels, YFCC's rotated targets, segNet's passes and the sky-mask resizes), the edges of the tables (1 x 1 to N, N to 1,
one side unchanged so its pass is skipped, 1241 <-> 3 with ksize in the thousands), and both vertical kernels: the 4-byte
kernel runs when a row is a multiple of 4 bytes and both pointers are 4-byte aligned, the fallback otherwise (RGB widths with
W mod 4 = 1, 2, 3, odd single-channel widths, a source that starts one row or one byte into its buffer).  Content: random
bytes, checkerboards, impulses and 0 / 255 steps, which drive LANCZOS overshoot into ``clip8`` at both ends.
"""
import numpy as np
import PIL.Image as Image
import pytest
import torch

from test_resample_host import pipeline_resizes

pytestmark = pytest.mark.gpu
FN = {"lanczos": ("rf_lanczos_coeffs_host", Image.LANCZOS), "bilinear": ("rf_bilinear_coeffs_host", Image.BILINEAR)}


def image(seed, h, w, ch, style):
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    if style == "random":
        a = rs.randint(0, 256, (h, w, ch))
    elif style == "checker":
        a = np.repeat((((yy + xx) % 2) * 255)[..., None], ch, 2)
    elif style == "impulse":
        a = np.zeros((h, w, ch))
        a[rs.randint(0, h, 1 + h * w // 50), rs.randint(0, w, 1 + h * w // 50)] = 255
        a[..., -1] = 255 - a[..., -1]                       # bright impulses on one channel, dark on the last
    else:                                                   # 0 / 255 steps along both axes, phase per channel
        a = np.stack([((xx // (1 + c) + yy // 3) % 2) * 255 for c in range(ch)], 2)
    return a.astype(np.uint8)


def pil(img, ow, oh, name):
    mode = "L" if img.shape[2] == 1 else "RGB"
    out = np.asarray(Image.fromarray(img[..., 0] if mode == "L" else img, mode).resize((ow, oh), resample=FN[name][1]))
    return out.reshape(oh, ow, img.shape[2])


def variant(t, ow, oh):
    """Which kernels ``_resize_u8`` launches for a source tensor ``t`` (H, W, ch): the rule of ``rf_resample_u8``."""
    H, W, ch = t.shape
    v = []
    if ow != W:
        v.append("h")
    if oh != H:
        aligned = (ow * ch) % 4 == 0 and (ow != W or t.data_ptr() % 4 == 0)
        v.append("v4" if aligned else "v-fallback")
    return "+".join(v) or "copy"


def run(rf, t, ow, oh, name):
    out = rf.ops._resize_u8(t, ow, oh, FN[name][0])
    torch.cuda.synchronize()
    return out.cpu().numpy()


def check(rf, img, ow, oh, name, t=None, what=""):
    t = torch.from_numpy(img).cuda() if t is None else t
    v = variant(t, ow, oh)
    got = run(rf, t, ow, oh, name)
    ref = pil(img, ow, oh, name)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if not np.array_equal(got, ref):
        bad = np.argwhere(got != ref)
        raise AssertionError("%s %s %s -> %dx%d (%s): %d bytes differ, first at %s: %d vs Pillow %d" % (
            what, name, img.shape, ow, oh, v, len(bad), bad[0].tolist(), got[tuple(bad[0])], ref[tuple(bad[0])]))
    return v


def test_pipeline_sizes_bit_exact(rf):
    seen = {}
    for i, (name, (w, h), (ow, oh), ch) in enumerate(pipeline_resizes()):
        for style in ("random", "steps"):
            v = check(rf, image(i, h, w, ch, style), ow, oh, name, what="pipeline")
            seen.setdefault((name, ch, v), []).append("%dx%d->%dx%d" % (w, h, ow, oh))
    for k, s in sorted(seen.items()):
        print("%s %d channel(s) %s: %s" % (k[0], k[1], k[2], ", ".join(sorted(set(s)))))
    assert ("lanczos", 3, "h+v4") in seen and ("bilinear", 3, "h+v4") in seen


EDGES = [((1, 1), (7, 5)), ((1, 1), (1, 9)), ((53, 37), (1, 1)), ((53, 37), (53, 1)), ((53, 37), (1, 37)), ((53, 37), (53, 80)),
         ((53, 37), (96, 37)), ((1241, 4), (3, 4)), ((3, 4), (1241, 4)), ((5, 1241), (5, 3)), ((5, 3), (5, 1241)), ((1241, 376), (3, 2)),
         ((2, 3), (1241, 376)), ((640, 480), (639, 481)), ((17, 9), (16, 10))]


@pytest.mark.parametrize("name", list(FN))
@pytest.mark.parametrize("ch", [3, 1])
def test_edge_sizes_bit_exact(rf, name, ch):
    for i, ((w, h), (ow, oh)) in enumerate(EDGES):
        for style in ("random", "checker", "impulse", "steps"):
            check(rf, image(100 + i, h, w, ch, style), ow, oh, name, what="edge")


@pytest.mark.parametrize("name", list(FN))
def test_both_vertical_kernels(rf, name):
    """The horizontal pass is skipped (out width = in width), so the vertical pass reads the caller's tensor: RGB widths with
    W mod 4 = 0..3 and single-channel widths 64..67 pick the 4-byte kernel only for rows that are a multiple of 4 bytes."""
    seen = set()
    for ch, widths in ((3, (64, 65, 66, 67)), (1, (64, 65, 66, 67))):
        for w in widths:
            for h, oh in ((40, 97), (97, 40), (31, 1), (1, 13)):
                for style in ("random", "checker", "steps"):
                    v = check(rf, image(w + h, h, w, ch, style), w, oh, name, what="vertical")
                    seen.add(v)
                    assert v == ("v4" if (w * ch) % 4 == 0 else "v-fallback"), (w, ch, v)
    assert seen == {"v4", "v-fallback"}


@pytest.mark.parametrize("name", list(FN))
@pytest.mark.parametrize("ch,w", [(3, 64), (3, 67), (1, 64), (1, 62)])
def test_misaligned_sources(rf, name, ch, w):
    """Sources that are views into a larger buffer: one row in (its pointer is misaligned whenever a row is not a multiple of 4
    bytes) and one byte in (always misaligned, so even 4-byte rows take the fallback)."""
    h, oh, ow = 45, 70, w
    img = image(w * ch, h, w, ch, "random")
    flat = torch.from_numpy(img).reshape(-1).cuda()
    row = torch.zeros((h + 1) * w * ch, dtype=torch.uint8, device="cuda")[w * ch:]
    row.copy_(flat)
    one = torch.zeros(h * w * ch + 1, dtype=torch.uint8, device="cuda")[1:]
    one.copy_(flat)
    for t, where in ((row.view(h, w, ch), "row"), (one.view(h, w, ch), "byte")):
        assert t.is_contiguous()
        v = check(rf, img, ow, oh, name, t=t, what="%s-offset view" % where)
        expect_v4 = (w * ch) % 4 == 0 and t.data_ptr() % 4 == 0
        assert v == ("v4" if expect_v4 else "v-fallback"), (where, v)
        assert where == "row" or v == "v-fallback"
        # both passes from the same view: the vertical pass then reads the horizontal pass's own (aligned) buffer
        check(rf, img, ow + 3, oh, name, t=t, what="%s-offset view, both passes" % where)
