"""The direct stems of engines 2 and 4 (RF_OP_STEM7: stem_kernel<k, stride, split> in csrc/gemm_tc.cu) restated for the tests
(helper of the stem tests, not a test module): the fp64 reference on the operands the kernel consumes, the launcher's work
decomposition, and which situations of that decomposition a batch of images runs into on a device with a given SM count.

The decomposition, from the kernel's documentation: the stem output of an image is cut into strips of 32 columns and steps of
4 rows (fused with the max-pool: strips of 15 pooled columns and steps of 2 pooled rows); the work units run image by image,
strip by strip, down each strip; G = min(units, CTAS x SMs) persistent CTAs take the contiguous ranges
[units b / G, units (b + 1) / G), with CTAS = 2 for the 3x3 / stride 1 stem and 1 for the 7x7 / stride 2 stem.
"""
import numpy as np
import torch

import wgmma_ref as R

GEOMETRIES = [(7, 2, 3), (3, 1, 1)]        # (k, stride, pad): the ResNet-50 stem and the FeatureExtractor stem
STRIDE = {7: 2, 3: 1}
CTAS = {7: 1, 3: 2}                         # CTAs per SM
TILE_W, TILE_H = 32, 4                      # stem columns per strip, stem rows per step
POOL_W, POOL_H = 15, 2                      # pooled columns per strip, pooled rows per step
SITUATIONS = ("three_units", "starts_mid_strip", "crosses_strip", "crosses_image_width", "partial_column", "partial_step")


# ------------------------------------------------------------------ programs and runs
def stem_args(seed, k):
    """Seeded (weight (64, 3, k, k) / sqrt(fan-in), BatchNorm2d(64) in eval mode with random statistics)."""
    g = torch.Generator().manual_seed(seed)
    weight = torch.randn(64, 3, k, k, generator=g) / np.sqrt(3 * k * k)
    bn = torch.nn.BatchNorm2d(64).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(64, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(64, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(64, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(64, generator=g) + 0.5)
    return weight, bn


def stem_program(weight, bn, device="cuda"):
    """(a LayerProgram of the stem alone, its FoldedConv); the geometry follows the weight's size."""
    from ransac_flow_b200.program import LayerProgram
    P = LayerProgram(3, device=device)
    P.stem7_fused(0, weight, bn)
    return P, P.ops[0][9]


def run_nan(rf, P, xs, engine):
    """Runs the program on the (1, 3, H, W) CPU images twice, the second time into its output buffer filled with NaN; returns
    (that output, a view valid until the program's next run; the output sizes)."""
    x = rf.ops.Ragged(R.nhwc(xs).cuda(), [(t.shape[2], t.shape[3]) for t in xs])
    out, ohw = P.run(x, engine)
    out.fill_(float("nan"))
    out, ohw = P.run(x, engine)
    torch.cuda.synchronize()
    return out, ohw


def bits(t):
    return t.view(torch.int16)


def image_part(out, ohw, i):
    """Image i's rows of a ragged fp16 [P, 64] or split [2, P, 64] output."""
    o = np.cumsum([0] + [h * w for h, w in ohw])
    return out[:, o[i]:o[i + 1]] if out.dim() == 3 else out[o[i]:o[i + 1]]


# ------------------------------------------------------------------ the fp64 reference
def packed_weights(fc, engine, k):
    """fp64 (64, 3, k, k) values of the packed operand the engine reads: the fp16 weights (engine 2) or hi + lo 2^-11 of the
    split planes (engine 4), whose rows are the taps in (r, s, c) order, zero padded."""
    w = (R.from_split(fc.w_split) if engine == 4 else fc.w_f16.double()).cpu()
    kk = k * k * 3
    assert not bool(w[:, kk:].any()), "the padding of the packed stem weights is not zero"
    return w[:, :kk].reshape(64, k, k, 3).permute(0, 3, 1, 2).contiguous()


def stem_ref(x, weight_q, bias, k, stride, pad):
    """fp64 convolution + bias + ReLU of a (1, 3, H, W) image and its absref (the same on absolute values, no ReLU).  ``x`` and
    ``weight_q`` (64, 3, k, k) hold the values the kernel consumes: wgmma_ref.operand(..., "f16" | "split") of the image, the
    packed weights."""
    assert tuple(weight_q.shape) == (64, 3, k, k) and x.shape[1] == 3
    return R.conv_ref(x, weight_q, bias, None, stride, pad, relu=True)


def output_images(out, ohw, engine):
    """The fp64 (1, 64, Ho, Wo) images an engine-2 (fp16) or engine-4 (split) output stands for."""
    return R.images(R.from_split(out) if engine == 4 else out.double(), ohw)


def check_stem(fc, k, xs, engine, out, ohw, what):
    """Every element of a stem output against stem_ref, within the output format's rounding plus the engine's accumulation
    allowance (wgmma_ref.check: split-grade on engine 4, fp16 rounding on engine 2).  Returns the worst error / allowance."""
    stride, pad = STRIDE[k], (k - 1) // 2
    kind = "split" if engine == 4 else "f16"
    hw = [(t.shape[2], t.shape[3]) for t in xs]
    assert [tuple(v) for v in ohw] == [R.out_hw(h, w, k, stride, pad) for h, w in hw]
    _, xq = R.operand(R.nhwc(xs), kind)
    wq = packed_weights(fc, engine, k).cuda()
    got = output_images(out, ohw, engine)
    worst = 0.0
    for i, xi in enumerate(R.images(xq.cuda(), hw)):
        ref, absref = stem_ref(xi, wq, fc.bias, k, stride, pad)
        worst = max(worst, R.check(got[i], ref, absref, R.R_SPLIT if engine == 4 else R.R_F16, R.ACC[kind], R.ATOL[kind],
                                   "%s image %d" % (what, i)))
    return worst


# ------------------------------------------------------------------ the work decomposition
def stem_units(sizes, k, stride, pool):
    """The work units of a batch of (H, W) images: {"images": one dict per image (stem output Hs x Ws, stored output
    Ho x Wo, strips, steps per strip, first unit), "total": units of the batch}."""
    pad = (k - 1) // 2
    images, start = [], 0
    for h, w in sizes:
        hs, ws = R.out_hw(h, w, k, stride, pad)
        ho, wo = ((hs - 1) // 2 + 1, (ws - 1) // 2 + 1) if pool else (hs, ws)        # max-pool 3 / stride 2 / pad 1
        strips = -(-wo // POOL_W) if pool else -(-ws // TILE_W)
        steps = -(-ho // POOL_H) if pool else -(-hs // TILE_H)
        images.append(dict(Hs=hs, Ws=ws, Ho=ho, Wo=wo, strips=strips, steps=steps, start=start))
        start += strips * steps
    return dict(images=images, total=start)


def cta_ranges(units, sms, k):
    """[begin, end) of the units each CTA runs."""
    g = min(units, CTAS[k] * sms)
    return [(units * b // g, units * (b + 1) // g) for b in range(g)]


def decode(un, u):
    """(image, strip, step) of unit u."""
    img = max(i for i, im in enumerate(un["images"]) if u >= im["start"])
    loc = u - un["images"][img]["start"]
    return img, loc // un["images"][img]["steps"], loc % un["images"][img]["steps"]


def describe(sizes, k, pool, sms):
    """Which situations a batch runs into on a device with ``sms`` SMs:
      three_units          a CTA runs at least 3 units: the two window buffers and the rotating output tiles wrap;
      starts_mid_strip     a CTA's range starts below the top of a strip;
      crosses_strip        a CTA goes from the bottom of a strip to the top of the next one of the same image;
      crosses_image_width  a CTA goes from one image into another of a different width (it prefetches the next image's window
                           with that image's sizes while it stores the tile of this one);
      partial_column       an image's last strip is narrower than a strip;
      partial_step         an image's last step is lower than a step."""
    un = stem_units(sizes, k, STRIDE[k], pool)
    out = dict.fromkeys(SITUATIONS, False)
    for b, e in cta_ranges(un["total"], sms, k):
        out["three_units"] |= e - b >= 3
        prev = decode(un, b)
        out["starts_mid_strip"] |= prev[2] > 0
        for u in range(b + 1, e):
            cur = decode(un, u)
            out["crosses_strip"] |= cur[0] == prev[0] and cur[1] != prev[1]
            out["crosses_image_width"] |= cur[0] != prev[0] and sizes[cur[0]][1] != sizes[prev[0]][1]
            prev = cur
    for im in un["images"]:
        out["partial_column"] |= (im["Wo"] % POOL_W if pool else im["Ws"] % TILE_W) != 0
        out["partial_step"] |= (im["Ho"] % POOL_H if pool else im["Hs"] % TILE_H) != 0
    return out


# ------------------------------------------------------------------ tap probes
def tap_of(r, s, c, k):
    return (r * k + s) * 3 + c


def probe_weight(k):
    """Integer weights (64, 3, k, k): tap t = (r k + s) 3 + c of output channel o is 1 + ((t + 5 o) mod 251).  k k 3 <= 147 <
    251, so within a channel every tap has its own value; all are exact in fp16 (hi plane only, lo plane zero)."""
    t = torch.arange(k * k * 3)
    w = 1 + ((t[None, :] + 5 * torch.arange(64)[:, None]) % 251)
    return w.reshape(64, k, k, 3).permute(0, 3, 1, 2).contiguous().float()


def tap_with_weight(value, o, k):
    """The tap of output channel o whose probe weight is ``value``, as (r, s, c), or None."""
    for t in range(k * k * 3):
        if 1 + ((t + 5 * o) % 251) == value:
            return t // (3 * k), t // 3 % k, t % 3
    return None


def impulse_images(sizes, k):
    """One (1, 3, H, W) image per size: zeros with unit impulses on a lattice of pitch k, so that no k x k window holds two and
    every output element is one weight or zero.  The lattice of image i is anchored at corner i mod 4 (so each corner of some
    image carries an impulse, and the ragged sizes shift the lattice against the tiles from image to image); the channel
    changes from impulse to impulse."""
    xs = []
    for i, (h, w) in enumerate(sizes):
        ys, cols = torch.arange(0, h, k), torch.arange(0, w, k)
        if i & 1:
            cols = w - 1 - cols
        if i & 2:
            ys = h - 1 - ys
        yy, xx = torch.meshgrid(ys, cols, indexing="ij")
        x = torch.zeros(1, 3, h, w)
        x[0, (yy // k + 2 * (xx // k) + i) % 3, yy, xx] = 1.0
        xs.append(x)
    return xs


def probed_taps(x, k):
    """(Ho, Wo) int64: the tap whose weight each output pixel of an impulse image shows (-1: none), and the number of
    impulses in each pixel's window (at most 1 by construction)."""
    stride, pad = STRIDE[k], (k - 1) // 2
    idx = (torch.arange(k * k * 3, dtype=torch.float64) + 1).reshape(1, k, k, 3).permute(0, 3, 1, 2)
    tap = torch.nn.functional.conv2d(x.double(), idx, stride=stride, padding=pad)[0, 0]
    count = torch.nn.functional.conv2d(x.double(), torch.ones_like(idx), stride=stride, padding=pad)[0, 0]
    return tap.long() - 1, count.long()


def first_mismatch(got, ref, x, k):
    """None if the (1, 64, Ho, Wo) output of an impulse image equals ``ref`` exactly, else a description of the first element
    that does not: its pixel and channel, the tap it should show, and what it holds instead - another tap's weight (two
    offsets swapped) or the right value plus another tap's weight (that tap's offset points at this pixel's impulse)."""
    bad = (got != ref).nonzero()
    if not len(bad):
        return None
    _, o, oy, ox = bad[0].tolist()
    t = int(probed_taps(x, k)[0][oy, ox])
    want = "tap (r, s, c) = %s" % ((t // (3 * k), t // 3 % k, t % 3),) if t >= 0 else "no tap"
    v, e = float(got[0, o, oy, ox]), float(ref[0, o, oy, ox])
    is_tap = tap_with_weight(v, o, k) if np.isfinite(v) else None
    extra = tap_with_weight(v - e, o, k) if np.isfinite(v) and e > 0 else None
    have = ["the weight of tap (r, s, c) = %s" % (is_tap,)] if is_tap else []
    have += ["the expected value plus the weight of tap (r, s, c) = %s" % (extra,)] if extra else []
    return ("%d of %d elements differ; first at pixel (%d, %d) channel %d: expected %s, value %r; got %r, %s" %
            (len(bad), got.numel(), oy, ox, o, want, e, v, " or ".join(have) or "no tap's weight"))
