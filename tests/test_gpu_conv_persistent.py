"""The persistent wgmma convolution: several tiles per CTA, with the ring running on across tile boundaries, the residual
TMA-loaded into the epilogue slot and fp16 / split outputs TMA-stored from it.  Every element is checked against the fp64
references of tests/wgmma_ref.py in NaN-filled outputs; the ragged case also checks that nothing is written past the
output.  Plus the CPU test of tools/conv_layer_profile.py's flop / byte model."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import wgmma_ref as R

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def size_for(tiles):
    """An (H, W) image with at least ``tiles`` 128-pixel tiles, whose last tile row and column are partial."""
    w = 367
    tw = R.pick_tw(1, w)
    h = 1
    while True:
        tw = R.pick_tw(h, w)
        th = 128 // tw
        if ((w + tw - 1) // tw) * ((h + th - 1) // th) >= tiles and h % th:
            return h, w
        h += 1


def persistent_cases():
    """(engine, cout, KI, res): KI in {1, STAGES, STAGES + 1, 2 STAGES + 1} of each instance, so that tile boundaries fall at
    different ring phases; Cout 56 (BN 64) and 200 (BN 128, partial second N tile); with and without residual (engine 5
    writes fp32 and takes none)."""
    out = []
    for engine in (2, 4, 5):
        kind = R.ENGINES[engine][0]
        for cout in (56, 200):
            s = R.stages(kind, R.bn_of(cout))
            for ki in sorted({1, s, s + 1, 2 * s + 1}):
                for res in ((False,) if engine == 5 else (False, True)):
                    out.append((engine, cout, ki, res))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("engine,cout,ki,res", persistent_cases())
def test_persistent_tiles(rf, engine, cout, ki, res):
    """Every CTA runs at least 4 tiles (2 CTAs per SM for the instances that allow it)."""
    nt = (cout + R.bn_of(cout) - 1) // R.bn_of(cout)
    hw = size_for(math.ceil(4 * 2 * sm_count() / nt))
    cin = R.BK[R.ENGINES[engine][0]] * ki
    xs, w, bias, rs = R.conv_inputs(engine * 1000 + cout + ki, cin, cout, 1, [hw], res, 1)
    R.check_conv(rf, engine, xs, w, bias, rs, 1, True, "persistent %d -> %d KI %d %s" % (cin, cout, ki, hw))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [2, 4])
@pytest.mark.parametrize("cout,k,stride", [(72, 3, 1), (136, 1, 1), (56, 3, 2)])
def test_ragged_partial_tiles_leave_guard(rf, monkeypatch, engine, cout, k, stride):
    """Images ending in partial pixel tiles (and partial N tiles): every output element right, and a guard region after the
    output buffer untouched."""
    guard = 4096
    bufs = []

    def guarded(shape, dtype):
        n = int(np.prod(shape))
        flat = torch.full((n + guard,), 1234.0, dtype=dtype, device="cuda")
        flat[:n] = float("nan")
        bufs.append((flat, n))
        return flat[:n].view(shape)
    monkeypatch.setattr(R, "nan_output", guarded)
    sizes = [(37, 53), (61, 29), (5, 131), (1, 1), (23, 70)]
    xs, w, bias, rs = R.conv_inputs(engine + cout + k, 64, cout, k, sizes, True, stride)
    R.check_conv(rf, engine, xs, w, bias, rs, stride, True, "ragged %dx%d -> %d stride %d" % (k, k, cout, stride))
    flat, n = bufs[0]
    assert bool((flat[n:] == 1234.0).all()), "the convolution wrote past its output"


@pytest.mark.gpu
@pytest.mark.parametrize("c1,c2,cout,stride2", [(128, 256, 512, 2), (64, 64, 200, 1)])
def test_dual_several_tiles_per_cta(rf, c1, c2, cout, stride2):
    from test_gpu_split import dual_check
    nt = (cout + 127) // 128
    h, w = size_for(math.ceil(4 * sm_count() / nt))
    g = torch.Generator().manual_seed(c1 + c2 + cout)
    x2s = [torch.randn(1, c2, h * stride2, w * stride2 - 1, generator=g)]
    x1s = [torch.randn(1, c1, (x2s[0].shape[2] - 1) // stride2 + 1, (x2s[0].shape[3] - 1) // stride2 + 1, generator=g)]
    w1 = torch.randn(cout, c1, generator=g) / np.sqrt(c1)
    w2 = torch.randn(cout, c2, generator=g) / np.sqrt(c2)
    bias = torch.randn(cout, generator=g)
    worst, _ = dual_check(rf, x1s, x2s, w1, w2, bias, stride2, True)
    print("dual %d + %d -> %d at %s: worst error / allowance %.3g" % (c1, c2, cout, x1s[0].shape[2:], worst))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [2, 4])
def test_two_streams_match_alone(rf, engine):
    """The same layer on two streams at once, on separate buffers: persistent CTAs of both launches share the GPU, and each
    result equals the layer run alone bit for bit."""
    kind, out = R.ENGINES[engine]
    cin, cout, k = 128, 136, 3
    hw = [size_for(4 * sm_count())]
    xs, w, bias, rs = R.conv_inputs(77 + engine, cin, cout, k, hw, True, 1)
    x = R.operand(R.nhwc(xs), kind)[0].contiguous().cuda()
    wd = R.operand(w.permute(0, 2, 3, 1).reshape(cout, -1).contiguous(), kind)[0].contiguous().cuda()
    r = R.operand(R.nhwc(rs), kind)[0].contiguous().cuda()
    b = bias.cuda()
    P = hw[0][0] * hw[0][1]
    shape = (2, P, cout) if out == "split" else (P, cout)

    def run(y):
        R.conv_call(rf, x, hw, cin, None, wd, b, r, cout, k, 1, 1, True, engine, y)
        return y
    alone = run(R.nan_output(shape, torch.float16))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ys = [[R.nan_output(shape, torch.float16) for _ in range(3)] for _ in streams]
    torch.cuda.synchronize()
    for i in range(3):
        for s, yl in zip(streams, ys):
            with torch.cuda.stream(s):
                run(yl[i])
    torch.cuda.synchronize()
    ref = alone.view(torch.int16)
    assert not bool(torch.isnan(alone).any())
    for yl in ys:
        for y in yl:
            assert torch.equal(y.view(torch.int16), ref)


def test_profile_model_trunk_floor():
    """tools/conv_layer_profile.py's model of the split trunk on one config-2 pair: the stem and 39 wg_kernel convolutions,
    477 GFLOP, 6.6 GB, and a floor of 2.39 ms at the H100 SXM data-sheet rates."""
    import conv_layer_profile as M
    hw = M.pair_sizes()
    assert hw[0] == (960, 1280) and hw[6] == (240, 320) and hw[7] == (480, 640) and len(hw) == 8
    prog = M.trunk_program()
    rows = M.convs(M.layer_model(prog.ops, hw, prog.dual))
    assert len(rows) == 40 and rows[0]["op"] == "stem7"
    assert abs(sum(r["gflop"] for r in rows) - 477.1) < 0.5
    assert abs(sum(r["bytes"] for r in rows) / 1e9 - 6.62) < 0.05
    floor = sum(r["floor_ms"] for r in rows)
    assert abs(floor - 2.39) <= 0.05 * 2.39, floor
    assert sum(r["bound"] == "hbm" for r in rows) == 21
    assert sum(r["KI"] <= 4 for r in rows[1:]) == 15
    # one layer by hand: layer1 conv3 + residual, 64 -> 256 at 1x1 on the pyramid at stride 4
    r = rows[6]
    pix = sum((h // 4) * (w // 4) for h, w in hw)
    assert (r["cin"], r["cout"], r["residual"], r["KI"]) == (64, 256, True, 1)
    assert r["gflop"] == pytest.approx(2 * pix * 64 * 256 / 1e9)
    assert r["bytes"] == 4 * pix * (64 + 256 + 256)
    assert r["floor_ms"] == pytest.approx(1e3 * r["bytes"] / 3.35e12)
