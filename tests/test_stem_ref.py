"""tests/stem_ref.py without a GPU: its fp64 reference against torch, its unit arithmetic against the layer model of
tools/conv_layer_profile.py, and - the point - that the batches of the stem's GPU tests run into the situations they were
chosen for on 132 and 114 SMs (H100 SXM and PCIe), so that a batch that stops biting fails here instead of passing there."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

import stem_ref as S
import test_gpu_stem_geometry as G
import test_gpu_stem_pool as GP
import wgmma_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _profile_tool():
    spec = importlib.util.spec_from_file_location("conv_layer_profile", os.path.join(ROOT, "tools", "conv_layer_profile.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def union(batches, k, pool, sms):
    out = dict.fromkeys(S.SITUATIONS, False)
    for sizes in batches:
        for s, v in S.describe(sizes, k, pool, sms).items():
            out[s] |= v
    return out


# ------------------------------------------------------------------ the GPU tests' batches bite
@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("k", [7, 3])
def test_unpooled_batches_run_into_every_situation(k, sms):
    many = S.describe(G.in_sizes(G.MANY_UNITS, k), k, False, sms)
    assert all(many[s] for s in ("three_units", "starts_mid_strip", "crosses_strip", "crosses_image_width")), many
    batches = [G.in_sizes(v, k) for v in G.OUT_SIZES.values()] + [G.in_sizes(G.MANY_UNITS, k), G.PROBE_SIZES]
    got = union(batches, k, False, sms)
    assert all(got.values()), got
    # the guard-band batch has a partial last strip and a partial last step in one image
    guard = S.describe(G.GUARD_SIZES, 3, False, sms)
    assert guard["partial_column"] and guard["partial_step"]


@pytest.mark.parametrize("sms", [132, 114])
def test_pooled_batches_run_into_every_situation(sms):
    """The batches of tests/test_gpu_stem_pool.py, for the 7x7 stem fused with its max-pool."""
    pair = _profile_tool().pair_sizes()
    got = union([GP.RAGGED, pair, [(5 + 9 * i, 7 + 13 * i) for i in range(16)]], 7, True, sms)
    assert all(got.values()), got
    d = S.describe(pair, 7, True, sms)
    assert all(d[s] for s in ("three_units", "starts_mid_strip", "crosses_strip", "crosses_image_width")), d


def test_one_unit_per_cta_sizes_are_what_they_are():
    """97 x 131 at the 3x3 stem is one unit per CTA (the window prefetch and the tile rotation never run); 480 x 640 is nine."""
    for sms in (132, 114):
        r = S.cta_ranges(S.stem_units([(97, 131)], 3, 1, False)["total"], sms, 3)
        assert len(r) == 125 and all(e - b == 1 for b, e in r)
        assert not S.describe([(97, 131)], 3, False, sms)["three_units"]
    r = S.cta_ranges(S.stem_units([(480, 640)], 3, 1, False)["total"], 132, 3)
    assert len(r) == 264 and sorted({e - b for b, e in r}) == [9, 10] and r[0] == (0, 9) and r[-1][1] == 2400


def test_describe_on_hand_made_batches():
    # 2 strips of 2 steps, then one unit of another width: 5 units
    sizes = [(8, 64), (4, 32)]
    un = S.stem_units(sizes, 3, 1, False)
    assert un["total"] == 5 and [im["start"] for im in un["images"]] == [0, 4]
    assert [S.decode(un, u) for u in range(5)] == [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0)]
    d = S.describe(sizes, 3, False, 132)                                      # 5 CTAs of one unit
    assert [s for s in S.SITUATIONS if d[s]] == ["starts_mid_strip"]
    assert S.cta_ranges(5, 1, 3) == [(0, 2), (2, 5)] and S.cta_ranges(5, 1, 7) == [(0, 5)]
    d = S.describe(sizes, 3, False, 1)                                        # [0, 2) and [2, 5)
    assert d == dict(three_units=True, starts_mid_strip=False, crosses_strip=False, crosses_image_width=True,
                     partial_column=False, partial_step=False)
    d = S.describe([(9, 65), (4, 65)], 3, False, 2)                           # 3 strips of 3 steps, then 3 of 1: four CTAs of 3 units
    assert d == dict(three_units=True, starts_mid_strip=False, crosses_strip=True, crosses_image_width=False,
                     partial_column=True, partial_step=True)
    d = S.describe([(9, 65)], 3, False, 1)                                    # [0, 4) and [4, 9)
    assert d["starts_mid_strip"] and d["crosses_strip"]
    # pooled: 29 x 29 -> stem 15 x 15 -> pooled 8 x 8: 1 strip of 4 steps; 61 x 61 -> 31 -> 16: 2 strips of 8 steps
    un = S.stem_units([(29, 29), (61, 61)], 7, 2, True)
    assert [(im["Hs"], im["Ho"], im["strips"], im["steps"]) for im in un["images"]] == [(15, 8, 1, 4), (31, 16, 2, 8)] and un["total"] == 20


def test_units_agree_with_the_layer_model():
    """Output sizes of both stems on the config-2 pair sizes, against tools/conv_layer_profile.py's layer_model."""
    tool = _profile_tool()
    hw = tool.pair_sizes()
    for k, stride, pad in S.GEOMETRIES:
        P, _ = S.stem_program(S.stem_args(1, k)[0], None, device="cpu")
        row = tool.layer_model(P.ops, hw)[0]
        un = S.stem_units(hw, k, stride, False)
        assert row["op"] == "stem7" and row["out_hw"] == [(im["Hs"], im["Ws"]) for im in un["images"]]
        assert all((im["Ho"], im["Wo"]) == (im["Hs"], im["Ws"]) for im in un["images"])
        assert un["total"] == sum(-(-h // 4) * -(-w // 32) for h, w in row["out_hw"])
    P, _ = S.stem_program(S.stem_args(1, 7)[0], None, device="cpu")
    P.maxpool(1, 3, 2, 1)
    rows = tool.layer_model(P.ops, hw)
    assert rows[1]["out_hw"] == [(im["Ho"], im["Wo"]) for im in S.stem_units(hw, 7, 2, True)["images"]]


# ------------------------------------------------------------------ the reference
@pytest.mark.parametrize("k,stride,pad", S.GEOMETRIES)
@pytest.mark.parametrize("size", [(1, 1), (2, 3), (9, 14)])
def test_stem_ref_is_conv2d(k, stride, pad, size):
    g = torch.Generator().manual_seed(k + size[1])
    x = torch.randn(1, 3, *size, generator=g, dtype=torch.float64)
    w = torch.randn(64, 3, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(64, generator=g, dtype=torch.float64)
    ref, absref = S.stem_ref(x, w, b, k, stride, pad)
    assert ref.shape == (1, 64) + R.out_hw(*size, k, stride, pad)
    assert torch.equal(ref, F.relu(F.conv2d(x, w, b, stride=stride, padding=pad)))
    assert torch.equal(absref, F.conv2d(x.abs(), w.abs(), b.abs(), stride=stride, padding=pad))
    # by hand at the top-left pixel: taps (r, s) >= pad only
    hand = sum(float(x[0, c, r - pad, s - pad]) * float(w[5, c, r, s]) for c in range(3) for r in range(pad, min(k, pad + size[0]))
               for s in range(pad, min(k, pad + size[1]))) + float(b[5])
    assert abs(max(hand, 0.0) - float(ref[0, 5, 0, 0])) < 1e-12


def test_packed_weights_are_the_operands():
    """stem7_fused packs the folded weights in (r, s, c) order, zero padded; packed_weights reads them back as (64, 3, k, k)."""
    for k, _, _ in S.GEOMETRIES:
        weight, bn = S.stem_args(3, k)
        _, fc = S.stem_program(weight, bn, device="cpu")
        scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).detach()
        folded = weight * scale.view(-1, 1, 1, 1)
        assert torch.equal(S.packed_weights(fc, 2, k), folded.half().double())
        assert torch.equal(S.packed_weights(fc, 4, k), R.operand(folded, "split")[1])
        # without BatchNorm the weights go in as they are and there is no bias: the tap probes rely on it
        _, fc = S.stem_program(S.probe_weight(k), None, device="cpu")
        assert fc.bias is None and torch.equal(S.packed_weights(fc, 4, k), S.probe_weight(k).double())


# ------------------------------------------------------------------ the tap probes
@pytest.mark.parametrize("k", [7, 3])
def test_probe_weights_name_their_tap(k):
    w = S.probe_weight(k)
    assert float(w.min()) >= 1 and float(w.max()) <= 251 and torch.equal(w.half().float(), w)
    for o in (0, 17, 63):
        assert len(set(w[o].flatten().tolist())) == k * k * 3
        for r, s, c in ((0, 0, 0), (k - 1, k - 1, 2), (k // 2, 0, 1)):
            assert w[o, c, r, s] == 1 + (S.tap_of(r, s, c, k) + 5 * o) % 251
            assert S.tap_with_weight(float(w[o, c, r, s]), o, k) == (r, s, c)
    assert S.tap_with_weight(0.0, 0, k) is None
    small = (w - 1) % 17 - 8
    assert float(small.abs().max()) == 8 and k * k * 3 * 64 < 2 ** 22


@pytest.mark.parametrize("k", [7, 3])
def test_impulse_images_probe_every_tap_and_the_seams(k):
    """No window holds two impulses; over the batch every tap is shown; on either side of a strip seam (output columns 31 |
    32) every window column s is, on either side of a step seam (output rows 3 | 4) every window row r; the four corners of
    the input carry impulses, and - for stride 2 - even and odd input columns do."""
    xs = S.impulse_images(G.PROBE_SIZES, k)
    assert len(xs) <= 16
    taps, corners, parity = set(), set(), set()
    seen = {name: set() for name in ("col31", "col32", "row3", "row4")}
    for x in xs:
        tap, count = S.probed_taps(x, k)
        assert int(count.max()) == 1 and tap.shape == R.out_hw(x.shape[2], x.shape[3], k, S.STRIDE[k], (k - 1) // 2)
        taps |= set(tap[tap >= 0].tolist())
        for name, sl, part in (("col31", tap[:, 31:32], lambda t: t // 3 % k), ("col32", tap[:, 32:33], lambda t: t // 3 % k),
                               ("row3", tap[3:4], lambda t: t // (3 * k)), ("row4", tap[4:5], lambda t: t // (3 * k))):
            seen[name] |= {part(t) for t in sl[sl >= 0].tolist()}
        h, w = x.shape[2:]
        corners |= {c for c, (y, xx) in enumerate(((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1))) if x[0, :, y, xx].any()}
        parity |= set((x[0].sum(0).nonzero()[:, 1] % 2).tolist())
        # the tap probed_taps reports is the tap whose probe weight the convolution shows
        y = F.conv2d(x.double(), S.probe_weight(k).double(), stride=S.STRIDE[k], padding=(k - 1) // 2)
        oy, ox = (tap >= 0).nonzero()[int((tap >= 0).sum()) // 2].tolist()
        t = int(tap[oy, ox])
        assert S.tap_with_weight(float(y[0, 9, oy, ox]), 9, k) == (t // (3 * k), t // 3 % k, t % 3)
    assert taps == set(range(k * k * 3)), sorted(set(range(k * k * 3)) - taps)
    assert all(v == set(range(k)) for v in seen.values()), seen
    assert corners == {0, 1, 2, 3} and parity == {0, 1}


def test_first_mismatch_names_the_taps():
    k = 3
    x = S.impulse_images([(7, 40)], k)[0]
    w = S.probe_weight(k).double()
    ref = F.conv2d(x.double(), w, stride=1, padding=1)
    assert S.first_mismatch(ref.clone(), ref, x, k) is None
    tap, _ = S.probed_taps(x, k)
    oy, ox = [int(v) for v in (tap >= 0).nonzero()[0]]
    t = int(tap[oy, ox])
    other = (t + 4) % 27
    got = ref.clone()
    got[0, 2, oy, ox] = 1 + (other + 10) % 251                 # channel 2 holds another tap's weight
    msg = S.first_mismatch(got, ref, x, k)
    assert "pixel (%d, %d) channel 2" % (oy, ox) in msg
    assert "expected tap (r, s, c) = %s" % ((t // 9, t // 3 % 3, t % 3),) in msg
    assert "the weight of tap (r, s, c) = %s" % ((other // 9, other // 3 % 3, other % 3),) in msg
    extra = (t + 7) % 27
    got[0, 2, oy, ox] = ref[0, 2, oy, ox] + 1 + (extra + 10) % 251      # another tap's offset points at this impulse too
    assert "plus the weight of tap (r, s, c) = %s" % ((extra // 9, extra // 3 % 3, extra % 3),) in S.first_mismatch(got, ref, x, k)
    got[0, 2, oy, ox] = float("nan")
    assert "no tap's weight" in S.first_mismatch(got, ref, x, k)
