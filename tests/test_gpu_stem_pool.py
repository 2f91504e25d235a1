"""The ResNet-50 stem fused with its 3x3 / stride 2 / pad 1 max-pool (RF_LAYER_STEM_POOL, engines 2 and 4) against the same
weights run unfused: a stem-only program, then a max-pool-only program on its output.  The fused kernel computes every stem
value and every window maximum with the unfused kernels' arithmetic, so the outputs must be equal bit for bit."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from stem_ref import stem_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _profile_tool():
    spec = importlib.util.spec_from_file_location("conv_layer_profile", os.path.join(ROOT, "tools", "conv_layer_profile.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _programs(seed, device="cuda"):
    """(fused stem + max-pool, stem only, max-pool only) with the same weights."""
    from ransac_flow_b200.program import LayerProgram
    weight, bn = stem_args(seed, 7)
    fused = LayerProgram(3, device=device)
    fused.maxpool(fused.stem7_fused(0, weight, bn), 3, 2, 1)
    stem = LayerProgram(3, device=device)
    stem.stem7_fused(0, weight, bn)
    pool = LayerProgram(64, device=device)
    pool.maxpool(0, 3, 2, 1)
    return fused, stem, pool


def _images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(h * w, 3, generator=g) for h, w in sizes]
    return torch.cat(xs).cuda(), sizes


def _run_nan(rf, P, data, hw, engine):
    """Runs P twice, the second time into its output buffer filled with NaN; returns a copy of that output."""
    x = rf.ops.Ragged(data, hw)
    out, ohw = P.run(x, engine)
    out.fill_(float("nan"))
    out, ohw = P.run(x, engine)
    torch.cuda.synchronize()
    return out.clone(), ohw


def _fused_vs_unfused(rf, engine, sizes, seed=5):
    fused, stem, pool = _programs(seed)
    data, hw = _images(sizes, seed + 100)
    got, ohw = _run_nan(rf, fused, data, hw, engine)
    s, shw = _run_nan(rf, stem, data, hw, engine)
    ref, rhw = _run_nan(rf, pool, s, shw, engine)
    assert [tuple(v) for v in ohw] == [tuple(v) for v in rhw]
    assert got.shape == ref.shape and torch.equal(got.view(torch.int16), ref.view(torch.int16))
    return got, ohw


# stem outputs odd and even, below, at and past multiples of the 32 x 4 stem tile and of the 15 x 2 pooled step in either
# direction (input 61 -> stem 31, 63 -> 32, 65 -> 33, 15 -> 8, 17 -> 9, 121 -> 61, 123 -> 62)
RAGGED = [(17, 35), (3, 5), (9, 33), (15, 61), (17, 63), (65, 15), (121, 123), (123, 121), (130, 97), (8, 250), (251, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [[(1, 1)], [(1, 45)], [(38, 1)], [(1, 1), (2, 2), (3, 3), (4, 4)], RAGGED],
                         ids=["1x1", "1xW", "Hx1", "tiny", "ragged"])
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_pool_fused_equals_unfused(rf, engine, sizes):
    _fused_vs_unfused(rf, engine, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_pool_fused_equals_unfused_config2_pyramid(rf, engine):
    """The trunk's batch of one config-2 pair: the 7-scale source pyramid and the 480 x 640 target."""
    _fused_vs_unfused(rf, engine, _profile_tool().pair_sizes())


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_pool_sixteen_images_equal_images_alone(rf, engine):
    sizes = [(5 + 9 * i, 7 + 13 * i) for i in range(16)]
    batch, ohw = _fused_vs_unfused(rf, engine, sizes, seed=9)
    fused, _, _ = _programs(9)
    data, hw = _images(sizes, 109)
    o = np.cumsum([0] + [h * w for h, w in hw])
    p = np.cumsum([0] + [h * w for h, w in ohw])
    for i in range(16):
        alone, _ = _run_nan(rf, fused, data[o[i]:o[i + 1]], [hw[i]], engine)
        part = batch[:, p[i]:p[i + 1]] if engine == 4 else batch[p[i]:p[i + 1]]
        assert torch.equal(part.view(torch.int16), alone.view(torch.int16)), i


@pytest.mark.gpu
@pytest.mark.parametrize("engine", [2, 4])
def test_stem_pool_two_streams(rf, engine):
    """Two fused programs on two streams at once give what each gives alone."""
    progs = [_programs(s)[0] for s in (21, 22)]
    inputs = [_images(RAGGED, 121), _images([(480, 640), (240, 320)], 122)]
    alone = [_run_nan(rf, P, d, hw, engine)[0] for P, (d, hw) in zip(progs, inputs)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    torch.cuda.synchronize()
    for _ in range(3):
        for P, (d, hw), st in zip(progs, inputs, streams):
            with torch.cuda.stream(st):
                out, _ = P.run(rf.ops.Ragged(d, hw), engine)
                outs.append(out)
    torch.cuda.synchronize()
    for k, out in enumerate(outs[-2:]):
        assert torch.equal(out.view(torch.int16), alone[k].view(torch.int16)), k


# ------------------------------------------------------------------ host side (no GPU): the compiled programs
@pytest.mark.parametrize("split", [False, True])
def test_stem_output_sizes_no_buffer(rf, split):
    """The fused pair is marked on the stem layer, the max-pool still reads the stem's nominal slot (the program's wiring),
    and the stem's full-resolution output sizes no buffer: in the trunk its slot is only as large as its other tenants."""
    from ransac_flow_b200.program import RF_LAYER_STEM_POOL
    tool = _profile_tool()
    hw = tool.pair_sizes()
    P = tool.trunk_program("cpu") if split else _trunk_f16()
    c = P._compile(hw, torch.device("cpu"), not split, split)
    L = c["layers"]
    assert L[0].flags & RF_LAYER_STEM_POOL and not any(L[i].flags & RF_LAYER_STEM_POOL for i in range(1, len(P.ops)))
    assert (L[1].op, L[1].src, L[1].k, L[1].stride, L[1].pad) == (1, L[0].dst, 3, 2, 1) and L[1].dst != L[0].dst
    esz = 4 if split else 2

    def nbytes(t, P=P):
        hws = [list(hw)]
        for o in P.ops:
            k, s, p = o[5], o[6], o[7]
            hws.append([((h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1) for h, w in hws[o[1]]])
        return sum(h * w for h, w in hws[t]) * P.chan[t] * esz
    others = [i + 1 for i in range(1, len(P.ops)) if L[i].dst == L[0].dst]
    assert c["bufs"][L[0].dst].numel() == max(16, max([nbytes(t) for t in others], default=0))
    # a program of just the pair: the stem's slot holds nothing
    fused, _, _ = _programs(3, "cpu")
    c = fused._compile(hw, torch.device("cpu"), not split, split)
    assert c["bufs"][c["layers"][0].dst].numel() == 16 and c["out_slot"] == c["layers"][1].dst
    assert c["bufs"][c["out_slot"]].numel() == nbytes(2, fused) and nbytes(1, fused) > 3 * nbytes(2, fused)


def _trunk_f16():
    import synthdata
    from ransac_flow_b200.coarseAlignFeatMatch import ResNet50Conv4
    net = ResNet50Conv4.__new__(ResNet50Conv4)
    net.device = torch.device("cpu")
    net._sd = {k: v.detach().float() for k, v in synthdata.resnet50_conv4_state(0).items() if torch.is_tensor(v) and v.dtype.is_floating_point}
    return net._build(64)
