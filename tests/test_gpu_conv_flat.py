"""Flat pixel tiles of the wgmma convolution: a 1x1 / stride-1 layer runs its ragged batch as one [sum HW][C] matrix in tiles
of 128 consecutive pixels that run on across image boundaries (3x3 and strided layers keep tw x (128 / tw) rectangles inside
each image).  Every element is checked against the fp64 references of tests/wgmma_ref.py in NaN-filled outputs, each image of
a batch equals that image run alone bit for bit, and the outputs' digests equal those of the kernel with per-image rectangle
tiles.  Plus the CPU test of tools/conv_layer_profile.py's tile model."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

import wgmma_ref as R

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

# image sizes that are not multiples of 128 pixels, with a 1 x 1 image among them
RAGGED = [(37, 53), (61, 29), (5, 131), (1, 1), (23, 70)]
SIXTEEN = [(1, 128), (2, 64), (16, 8), (4, 32), (8, 16), (13, 21), (1, 1), (9, 7), (3, 40), (25, 2), (6, 6), (11, 17), (2, 3), (7, 30),
           (19, 5), (5, 12)]


def rect_tiles(hw):
    return sum(((w + R.pick_tw(h, w) - 1) // R.pick_tw(h, w)) * ((h + 128 // R.pick_tw(h, w) - 1) // (128 // R.pick_tw(h, w))) for h, w in hw)


def straddling(hw):
    """The flat tiles (pixels 128 j .. 128 j + 127 of the batch) that hold pixels of more than one image."""
    ends = np.cumsum([h * w for h, w in hw])[:-1]
    return sorted({int(e) // 128 for e in ends if e % 128})


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def part(y, o, i):
    return y[:, o[i]:o[i + 1]] if y.dim() == 3 else y[o[i]:o[i + 1]]


def test_straddling_tiles_of_the_test_batches():
    assert straddling(RAGGED) == [15, 29, 34]
    assert straddling(SIXTEEN) == [7, 8, 9, 10, 12, 13]          # the first five images are whole tiles
    assert straddling([(8, 16), (1, 128)]) == []


def test_profile_tile_model_flat_for_1x1_stride1():
    """tools/conv_layer_profile.py counts ceil(sum HW / 128) pixel tiles for 1x1 / stride-1 layers (the dual conv3 + down-sampling
    GEMM only when its second input has stride 1) and per-image rectangles for the others, as conv_impl launches them."""
    import conv_layer_profile as M
    hw = M.pair_sizes()
    prog = M.trunk_program()
    rows = M.convs(M.layer_model(prog.ops, hw, prog.dual))
    nflat = 0
    for r in rows[1:]:
        flat = r["k"] == 1 and r["stride"] == 1 and (r["op"] == "conv" or prog.dual[r["index"]][2] == 1)
        pix = sum(h * w for h, w in r["out_hw"])
        assert r["tiles"] == ((pix + 127) // 128 if flat else rect_tiles(r["out_hw"])), r
        nflat += flat
    assert nflat == 24
    by = {(r["cin"], r["cout"], r["k"], r["stride"], r["op"]): r["tiles"] for r in rows[1:]}
    assert by[(64, 256, 1, 1, "conv")] == 1784 and by[(64, 64, 3, 1, "conv")] == 1817 and by[(64, 256, 1, 1, "conv_dual")] == 1784
    assert by[(512, 128, 1, 1, "conv")] == 446 and by[(128, 128, 3, 1, "conv")] == 482 and by[(128, 512, 1, 1, "conv_dual")] == 482
    assert by[(1024, 256, 1, 1, "conv")] == 112 and by[(256, 256, 3, 1, "conv")] == 133 and by[(256, 1024, 1, 1, "conv_dual")] == 133


def flat_cases():
    """(engine, cin, cout, sizes, res, relu): engines 1, 2, 4, 5 (engine 3 runs 3x3 layers only; engine 5 takes no residual),
    Cout 56 (BN 64) and 136 (BN 128 with a partial second N tile)."""
    out = []
    for engine in (1, 2, 4, 5):
        for cout in (56, 136):
            for cin, sizes in ((256, "ragged"), (64, "sixteen")):
                for res, relu in ((True, True), (False, False), (True, False), (False, True)):
                    if not (res and engine == 5):
                        out.append((engine, cin, cout, sizes, res, relu))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("engine,cin,cout,sizes,res,relu", flat_cases())
def test_flat_1x1_vs_fp64(rf, monkeypatch, engine, cin, cout, sizes, res, relu):
    """Every output element within the fp64 allowance, and a guard region after the output untouched (the batch's last tile is
    partial)."""
    hw = RAGGED if sizes == "ragged" else SIXTEEN
    assert straddling(hw)
    guard = 4096
    bufs = []

    def guarded(shape, dtype):
        n = int(np.prod(shape))
        flat = torch.full((n + guard,), 1234.0, dtype=dtype, device="cuda")
        flat[:n] = float("nan")
        bufs.append((flat, n))
        return flat[:n].view(shape)
    monkeypatch.setattr(R, "nan_output", guarded)
    xs, w, bias, rs = R.conv_inputs(engine * 100 + cin + cout, cin, cout, 1, hw, res, 1)
    R.check_conv(rf, engine, xs, w, bias, rs, 1, relu, "flat 1x1 %d -> %d %s res %s relu %s" % (cin, cout, sizes, res, relu))
    flat, n = bufs[0]
    assert bool((flat[n:] == 1234.0).all()), "the convolution wrote past its output"


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [1, 2, 4, 5])
def test_flat_batch_equals_images_alone(rf, engine):
    """Sixteen images whose flat tiles straddle image boundaries: each image's output equals that image run alone bit for bit,
    two identical calls give identical bits, and a seventeenth image is refused."""
    assert len(straddling(SIXTEEN)) == 6
    res = engine != 5
    xs, w, bias, rs = R.conv_inputs(30 + engine, 64, 136, 1, SIXTEEN, res, 1)
    y = R.run_conv(rf, engine, xs, w, bias, rs, 1, True)[-1]
    y2 = R.run_conv(rf, engine, xs, w, bias, rs, 1, True)[-1]
    assert not bool(torch.isnan(y).any())
    assert torch.equal(bits(y), bits(y2))
    o = np.cumsum([0] + [h * w for h, w in SIXTEEN])
    for i in range(16):
        alone = R.run_conv(rf, engine, [xs[i]], w, bias, [rs[i]] if res else None, 1, True)[-1]
        assert torch.equal(bits(part(y, o, i)), bits(alone)), i
    with pytest.raises(rf._lib.RFError):
        R.run_conv(rf, engine, xs + xs[:1], w, bias, rs + rs[:1] if res else None, 1, True)


def dual_inputs(seed, sizes, c1, c2, cout, stride2):
    g = torch.Generator().manual_seed(seed)
    x2s = [torch.randn(1, c2, h * stride2, w * stride2, generator=g) for h, w in sizes]
    x1s = [torch.randn(1, c1, h, w, generator=g) for h, w in sizes]
    w1 = torch.randn(cout, c1, generator=g) / np.sqrt(c1)
    w2 = torch.randn(cout, c2, generator=g) / np.sqrt(c2)
    return x1s, x2s, w1, w2, torch.randn(cout, generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", ["ragged", "sixteen"])
@pytest.mark.parametrize("relu", [True, False])
def test_flat_dual_stride1_vs_fp64(rf, sizes, relu):
    """Layer1's conv3 + down-sampling GEMM (second input at stride 1) on flat tiles, Cout 136, against fp64."""
    from test_gpu_split import dual_check
    hw = RAGGED if sizes == "ragged" else SIXTEEN
    x1s, x2s, w1, w2, bias = dual_inputs(40, hw, 64, 128, 136, 1)
    worst, _ = dual_check(rf, x1s, x2s, w1, w2, bias, 1, relu)
    print("flat dual %s relu %s: worst error / allowance %.3g" % (sizes, relu, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("stride2", [1, 2])
def test_dual_batch_equals_images_alone(rf, stride2):
    """The dual GEMM on sixteen images, on flat tiles (stride2 = 1) and on per-image rectangles (stride2 = 2): each image alone
    gives the same bits."""
    from test_gpu_split import dual_check
    x1s, x2s, w1, w2, bias = dual_inputs(50 + stride2, SIXTEEN, 64, 64, 136, stride2)
    _, y = dual_check(rf, x1s, x2s, w1, w2, bias, stride2, True)
    o = np.cumsum([0] + [h * w for h, w in SIXTEEN])
    for i in range(16):
        _, alone = dual_check(rf, [x1s[i]], [x2s[i]], w1, w2, bias, stride2, True)
        assert torch.equal(bits(part(y, o, i)), bits(alone)), i


# ------------------------------------------------------------------ the same bits as the kernel with per-image rectangle tiles
def digest_outputs(rf):
    """SHA-256 of the output bytes of seeded layers: 1x1 stride-1 layers on flat tiles (engines 1, 2, 4, 5, with and without
    residual), 3x3 and strided layers on rectangles, and the dual GEMM at stride2 1 (flat) and 2 (rectangles)."""
    from test_gpu_split import dual_check
    out = {}

    def put(name, y):
        torch.cuda.synchronize()
        out[name] = hashlib.sha256(y.cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()
    for engine in (1, 2, 4, 5):
        for res in ((False,) if engine == 5 else (False, True)):
            xs, w, bias, rs = R.conv_inputs(60 + engine, 128, 200, 1, RAGGED + SIXTEEN[:4], res, 1)
            put("1x1 engine %d res %s" % (engine, res), R.run_conv(rf, engine, xs, w, bias, rs, 1, True)[-1])
    for engine in (2, 4):
        for k, stride in ((3, 1), (3, 2), (1, 2)):
            xs, w, bias, rs = R.conv_inputs(70 + engine + k + stride, 64, 136, k, RAGGED, True, stride)
            put("%dx%d stride %d engine %d" % (k, k, stride, engine), R.run_conv(rf, engine, xs, w, bias, rs, stride, True)[-1])
    for stride2 in (1, 2):
        x1s, x2s, w1, w2, bias = dual_inputs(80 + stride2, RAGGED, 128, 64, 200, stride2)
        put("dual stride2 %d" % stride2, dual_check(rf, x1s, x2s, w1, w2, bias, stride2, True)[1])
    return out


# recorded with the kernel that ran every layer on per-image tw x (128 / tw) rectangles, pixel tiles fastest (an H100 80GB HBM3)
RECT_DIGESTS = {
    "1x1 engine 1 res False": "7fa9e29977bbacfb571295c0117638de4710ffe40c346eb9ec3006890f334193",
    "1x1 engine 1 res True": "e7565f10b5e9f9910117a1bf93eadcb1c48bfe815dc1cd75083c626c339a4394",
    "1x1 engine 2 res False": "0bec6834148c514bdea0961a1dcc349b88886fce847dae8f54a19cae602097d6",
    "1x1 engine 2 res True": "63759d3e4a30cc1e4798bd2a14b8b5c28ab08c22efc204f577e15894fe8f90b6",
    "1x1 engine 4 res False": "9da89617855f5d0a872846c8f80e11228bb13229b4f0412852836a46c2706853",
    "1x1 engine 4 res True": "4136522da2d7433bf0d0189c6c0b5eb70a05b28b816e80f5ae449b4f226e857e",
    "1x1 engine 5 res False": "c33098e41ae7629f718f926b887075adca4459453b187ad14b02a190b0b0f56a",
    "3x3 stride 1 engine 2": "87c6957c87f94b23f64567f5d093118bc497376d0a4feaab2720ce5a5786154b",
    "3x3 stride 2 engine 2": "abfb53697fc68ebb4315700f113aba620481e6bbb5b97c0f94cb4d82f23b1ac1",
    "1x1 stride 2 engine 2": "567ceed18318ddc61591d983b99de91fae9942cbca577bc5cd050f41b20bc741",
    "3x3 stride 1 engine 4": "714eeb330d6cd57c0813f2e24edcff45177d68b01763dff5b48f582234a6239b",
    "3x3 stride 2 engine 4": "7958d727a2c505419d7a23929280cc7d94a1a4a86b944df970f786c609e7248e",
    "1x1 stride 2 engine 4": "b6a7df4eebca48c171784073844c36242d5ca24fdf3fa0b6ff840d14053c3cde",
    "dual stride2 1": "4aded6ddde608d9312565876497780bf2fdc47b97c12e7dd688f6593100e4017",
    "dual stride2 2": "9dec554dfac1f443598416a6988247f63be05269ce77a22375f1de8368e35b67",
}


@pytest.mark.gpu
def test_outputs_bit_identical_to_rectangle_tiles(rf):
    """Flat tiles and the N-tile-fastest order change which rows share a tile and when a tile runs, not the arithmetic of any
    element: every output has the bits of the rectangle-tile kernel."""
    got = digest_outputs(rf)
    print(got)
    assert got.keys() == RECT_DIGESTS.keys()
    for name in got:
        assert got[name] == RECT_DIGESTS[name], name
