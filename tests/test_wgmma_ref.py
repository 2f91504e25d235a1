"""CPU checks of the reference side of the tensor-core tests (tests/wgmma_ref.py): key decoding, TF32 truncation, the
element-wise bound, and that the convolution tests' parameter lists run every tile width at both strides."""
import numpy as np
import pytest
import torch

import wgmma_ref as R


def test_argmax_key_round_trip_and_order():
    scores = np.array([0.0, -0.0, 1.0, -1.0, 3.5e-8, -2.25, 1e30, -1e-30, 0.7071067], dtype=np.float32)
    idx = np.array([0, 1, 2, 3, 4, 5, 6, 7, 4294967294], dtype=np.uint64)
    keys = R.encode_key(scores, idx)
    s, i = R.decode_key(keys)
    assert np.array_equal(s.view(np.uint32), scores.view(np.uint32)) and np.array_equal(i, idx.astype(np.int64))
    # max over keys = max score, ties to the smallest index; negative scores order below positive ones
    k = R.encode_key(np.array([0.5, 0.5, -0.25, 0.25], np.float32), np.array([9, 3, 0, 1]))
    assert R.decode_key(k.max())[1] == 3
    k = R.encode_key(np.array([-0.5, -0.25, -0.75], np.float32), np.array([0, 7, 2]))
    assert R.decode_key(k.max())[1] == 7
    assert R.decode_key(np.array([0], np.uint64))[1][0] == -1          # an unwritten key


def test_tf32_truncation():
    x = torch.tensor([1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -12, -3.0 - 2 ** -9 - 2 ** -13, 2 ** -130])
    t = R.tf32_trunc(x)
    assert t.tolist()[:5] == [1.0, 1.0 + 2 ** -10, 1.0, 1.0 + 2 ** -10, -3.0 - 2 ** -9]
    assert bool(R.is_tf32(t).all()) and not bool(R.is_tf32(x[2:3]).any())
    g = torch.Generator().manual_seed(0)
    y = torch.randn(10000, generator=g)
    rel = ((y - R.tf32_trunc(y)) / y).abs()
    assert float(rel.max()) < 2 ** -10 and float(rel.mean()) > 2 ** -13        # truncation: one TF32 ulp at most, biased
    r = R.tf32_round(y)
    assert bool(R.is_tf32(r).all()) and float(((y - r) / y).abs().max()) <= 2 ** -11
    assert R.tf32_round(torch.tensor([1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11])).tolist() == [1.0, 1.0 + 2 ** -9]   # ties to even


def test_split_operand_is_22_bit():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(10000, generator=g) * 10
    s, q = R.operand(x, "split")
    assert s.shape == (2, 10000) and s.dtype == torch.float16
    assert float(((q - x.double()) / x.double()).abs().max()) <= 2 ** -22
    h, qh = R.operand(x, "f16")
    assert float(((qh - x.double()) / x.double()).abs().max()) <= 2 ** -11


def test_bound_accepts_rounding_and_rejects_nan_and_11_bit_errors():
    g = torch.Generator().manual_seed(2)
    x, w = torch.randn(1, 64, 9, 7, generator=g), torch.randn(72, 64, 3, 3, generator=g) / 24
    b = torch.randn(72, generator=g)
    ref, absref = R.conv_ref(x, w, b, None, 1, 1, True)
    ratio = R.check(ref.float(), ref, absref, R.R_F32, R.ACC["tf32"])         # fp32 rounding of the exact result passes
    assert ratio <= 1.0
    R.check(ref.half(), ref, absref, R.R_F16, R.ACC["f16"], R.ATOL["f16"])  # so does fp16 rounding with its r_out
    bad = ref.clone()
    bad[0, 3, 8, 6] = float("nan")                                             # an element the kernel never wrote
    with pytest.raises(AssertionError):
        R.check(bad, ref, absref, R.R_F32, R.ACC["tf32"])
    # 11-bit operands (TF32 truncation / fp16 rounding of the weights only) against the fp32 bound: must fail
    coarse, _ = R.conv_ref(x, R.tf32_trunc(w), b, None, 1, 1, True)
    with pytest.raises(AssertionError):
        R.check(coarse, ref, absref, R.R_SPLIT, R.ACC["split"], R.ATOL["split"])
    with pytest.raises(AssertionError):
        R.check(ref.half(), ref, absref, R.R_SPLIT, R.ACC["split"], R.ATOL["split"])


def test_ring_depths_mirror_the_kernel_configuration():
    # WgCfg: 4 / 3 stages for TF32 / fp16 at BN 64 / 128, 2 / 3 for split, 3 for the correlation kinds
    assert [R.stages(k, bn) for k in ("tf32", "f16", "split") for bn in (64, 128)] == [4, 3, 4, 3, 2, 3]
    assert R.stages("tf32x3", 128) == 3
    kis = sorted({cin // R.BK["split"] for cin, cout, k, _ in R.ring_cases("split") if R.bn_of(cout) == 64})
    assert kis == [1, 2, 3, 4, 5]


def test_pick_tw_mirror_and_tile_width_coverage():
    assert R.pick_tw(1, 128) == 128 and R.pick_tw(2, 64) == 64 and R.pick_tw(16, 8) == 8 and R.pick_tw(60, 80) in R.TILE_WIDTHS
    import test_gpu_split
    import test_gpu_tc
    for name, cases in (("TF32", test_gpu_tc.TF32_CASES), ("F16", test_gpu_tc.F16_CASES), ("SPLIT", test_gpu_split.SPLIT_CASES),
                        ("SPLIT_OUT32", test_gpu_split.SPLIT_OUT32_CASES)):
        cov = R.widths_covered([(k, sizes) for _, _, k, sizes in cases], (1, 2))
        print(name, {s: sorted(v) for s, v in cov.items()})
        for s in (1, 2):
            assert cov[s] == set(R.TILE_WIDTHS), (name, s, sorted(cov[s]))
    # the 256-pixel TMA box: stride 2 with tw = 128 in the dual kernel's second input
    assert any(s2 == 2 and R.pick_tw((h - 1) // 2 + 1, (w - 1) // 2 + 1) == 128
               for _, _, _, s2, sizes in test_gpu_split.DUAL_CASES for h, w in sizes)


def test_partial_n_tiles_on_every_engine():
    import test_gpu_split
    import test_gpu_tc
    for name, cases in (("TF32", test_gpu_tc.TF32_CASES), ("F16", test_gpu_tc.F16_CASES), ("SPLIT", test_gpu_split.SPLIT_CASES),
                        ("SPLIT_OUT32", test_gpu_split.SPLIT_OUT32_CASES)):
        couts = {c for _, c, _, _ in cases}
        assert {72, 136, 200} <= couts, name
        if name in ("TF32", "SPLIT_OUT32"):          # fp32 outputs: odd Cout switches the float2 store to the scalar one
            assert {65, 97, 129} <= couts, name


def test_tf32_rna_rounds_ties_away_from_zero():
    x = torch.tensor([1.0 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 3 * 2 ** -11, 1.0 + 2 ** -11 - 2 ** -23, 0.0, 2 ** -140 + 2 ** -149])
    r = R.tf32_rna(x).tolist()
    assert r[:5] == [1.0 + 2 ** -10, -(1.0 + 2 ** -10), 1.0 + 2 ** -9, 1.0, 0.0]      # ties up in magnitude; below a tie: down
    assert R.tf32_round(x[:1]).tolist() == [1.0]                                       # ties to even differs exactly there
    g = torch.Generator().manual_seed(3)
    y = torch.randn(10000, generator=g) * 100
    t = R.tf32_rna(y)
    assert bool(R.is_tf32(t).all()) and float(((y - t) / y).abs().max()) <= 2 ** -11
    tie = (y.view(torch.int32) & 0x1FFF) == 0x1000
    assert torch.equal(t[~tie], R.tf32_round(y)[~tie])


def _layer_images(seed, c, sizes):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(1, c, h, w, generator=g) * 3 for h, w in sizes]


@pytest.mark.parametrize("stride", [1, 2])
def test_blur_and_poolblur_refs_match_the_oracle(stride):
    """blur_ref == MO.blur_downsample and poolblur_ref == MO.blur_downsample(max_pool2d(x, 2, 1), 2) within the fp32
    rounding of the oracle's own 9-term sums (gamma_9 of the filter on |x|), at the smallest sizes and odd / even ones."""
    import torch.nn.functional as F
    from oracle import model_oracle as MO
    for x in _layer_images(stride, 6, [(2, 2), (3, 3), (2, 9), (9, 2), (7, 8), (8, 7), (16, 24)]):
        ref, absref = R.blur_ref(x, stride)
        R.check(MO.blur_downsample(x, stride), ref, absref, 0.0, R.gamma(9), what="blur")
        if stride == 2 and min(x.shape[2:]) >= 3:
            ref, absref = R.poolblur_ref(x)
            R.check(MO.blur_downsample(F.max_pool2d(x, 2, 1), 2), ref, absref, 0.0, R.gamma(9), what="poolblur")
    # replicate instead of reflect padding is outside the bound
    x = _layer_images(9, 4, [(5, 6)])[0]
    ref, absref = R.blur_ref(x, stride)
    a = torch.tensor([1.0, 2.0, 1.0])
    f = (a[:, None] * a[None, :] / 16)[None, None].repeat(4, 1, 1, 1)
    with pytest.raises(AssertionError):
        R.check(F.conv2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), f, stride=stride, groups=4), ref, absref, 0.0, R.gamma(9))


def test_maxpool_and_im2col_refs_match_torch():
    import torch.nn.functional as F
    for x in _layer_images(4, 5, [(1, 1), (1, 7), (6, 1), (9, 12), (13, 8)]):
        assert torch.equal(R.maxpool_ref(x, 3, 2, 1), F.max_pool2d(x, 3, 2, 1).double())
        if min(x.shape[2:]) >= 2:
            assert torch.equal(R.maxpool_ref(x, 2, 1, 0), F.max_pool2d(x, 2, 1, 0).double())
        for k, s, p, kpad in ((7, 2, 3, 160), (3, 1, 1, 32), (7, 1, 3, 160), (3, 2, 1, 64), (5, 1, 2, 128)):
            if k * k * x.shape[1] > kpad:
                continue
            ho, wo = R.out_hw(x.shape[2], x.shape[3], k, s, p)
            u = F.unfold(x, k, padding=p, stride=s)[0]                                  # (C * k * k, L) in (c, r, s) order
            u = u.view(x.shape[1], k * k, ho * wo).permute(2, 1, 0).reshape(ho * wo, -1)  # -> (r, s, c)
            got = R.im2col_ref(x, k, s, p, kpad)
            assert got.shape == (ho * wo, kpad) and torch.equal(got[:, :u.shape[1]], u) and not bool(got[:, u.shape[1]:].any())


def test_l2norm_ref_matches_f_normalize():
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(5)
    C = 132
    x = torch.randn(40, C, generator=g) * torch.logspace(-3, 3, 40).view(-1, 1)
    x[3] = 0
    x[7] = x[7] / x[7].norm() * 3e-14                 # below the eps: x / 1e-12
    ref = R.l2norm_ref(x)
    R.check(F.normalize(x), ref, ref, R.gamma(C) / 2 + 2 * R.U, 0.0)            # the kernels' bound
    assert not bool(ref[3].any()) and abs(float(ref[7].norm()) - 0.03) < 1e-6
    mask = torch.ones(40, dtype=torch.uint8)
    mask[::3] = 0
    m = R.l2norm_ref(x, mask)
    assert not bool(m[::3].any()) and torch.equal(m[1::3], ref[1::3])


@pytest.mark.parametrize("k", [3, 5, 7])
def test_softmax_flow_ref_matches_net_flow_coarse(k, monkeypatch):
    """softmax_flow_ref == MO.net_flow_coarse with its convolution trunk replaced by the identity (the epilogue alone), within
    the bound the kernel is held to."""
    from oracle import model_oracle as MO
    monkeypatch.setattr(MO, "_trunk", lambda corr, sd: corr)
    g = torch.Generator().manual_seed(k)
    logits = torch.randn(2, k * k, 5, 9, generator=g) * 3
    ref, absf = R.softmax_flow_ref(logits, k)
    R.check(MO.net_flow_coarse(logits, None, k), ref, absf, R.U, (k * k + 8) * R.U)
