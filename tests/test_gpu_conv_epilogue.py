"""The epilogue slot of the wgmma convolutions with fp16 and split outputs: bias, residual (TMA-loaded into the slot), ReLU
and conversion, written back in place and TMA-stored, with the loads of each group of channel pairs issued together
(EPI_JC in csrc/gemm_tc.cu).  Every element is held to fp64 with the bounds of tests/wgmma_ref.py in NaN-filled outputs
with guard bands, and every output to the digest of the kernel that loaded bias and residual one channel pair at a time
(the operations and their order are the same, so the bits are too).  The cases: split BN = 128 (one CTA per SM) at 1, 2,
4 and 8 K blocks with and without a residual, Cout 192 (the second N tile's second box is outside the layer), a partial
last flat tile, fewer tiles than CTAs and more than 3 tiles per CTA, strided 1x1 rectangles, the dual conv3 +
down-sampling GEMM, the two-CTA instances (split BN = 64, fp16 BN = 64 and 128), and three launches on three streams at
once.  Plus the CPU test of tools/conv_tile_timeline.py's phase arithmetic."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

import wgmma_ref as R

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

# 39 945 pixels: 313 flat tiles, the last one of 9 pixels; x 2 N tiles = 626 tiles, more than 3 per CTA on 132 SMs
MANY = [(131, 197), (67, 211), (1, 1)]
FEW = [(5, 9)]                    # one pixel tile: fewer tiles than CTAs
GUARD = 4096


def cases():
    """(name, engine, cin, cout, sizes, res, stride): 1x1 layers, K blocks = cin / 64."""
    out = []
    for cin in (64, 128, 256, 512):
        for res in (True, False):
            out.append(("ki%d %s 256 many" % (cin // 64, "res" if res else "nores"), 4, cin, 256, "many", res, 1))
    for res in (True, False):
        out.append(("ki4 %s 192 many" % ("res" if res else "nores"), 4, 256, 192, "many", res, 1))
        out.append(("ki8 %s 256 few" % ("res" if res else "nores"), 4, 512, 256, "few", res, 1))
    out.append(("ki4 res 256 stride2", 4, 256, 256, "many", True, 2))
    for engine, cout in ((4, 56), (2, 56), (2, 136)):
        for res in (True, False):
            out.append(("engine%d ki2 %s %d many" % (engine, "res" if res else "nores", cout), engine, 128, cout, "many", res, 1))
    return out


def dual_cases():
    """(name, c1, c2, cout, stride2): the conv3 + down-sampling GEMM, K blocks (c1 + c2) / 64."""
    return [("dual ki2 stride1", 64, 64, 256, 1), ("dual ki6 stride2", 128, 256, 192, 2)]


def sizes_of(name):
    return MANY if name == "many" else FEW


def digest(y):
    torch.cuda.synchronize()
    return hashlib.sha256(y.cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def layer_inputs(case):
    name, engine, cin, cout, sizes, res, stride = case
    return R.conv_inputs(hash_seed(name), cin, cout, 1, sizes_of(sizes), res, stride)


def hash_seed(name):
    return int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)


def dual_inputs(case):
    name, c1, c2, cout, stride2 = case
    g = torch.Generator().manual_seed(hash_seed(name))
    x2s = [torch.randn(1, c2, h * stride2, w * stride2, generator=g) for h, w in MANY]
    x1s = [torch.randn(1, c1, h, w, generator=g) for h, w in MANY]
    w1 = torch.randn(cout, c1, generator=g) / np.sqrt(c1)
    w2 = torch.randn(cout, c2, generator=g) / np.sqrt(c2)
    return x1s, x2s, w1, w2, torch.randn(cout, generator=g)


@pytest.fixture
def guarded(monkeypatch):
    """Outputs of R.run_conv / dual_check: NaN-filled, with GUARD elements of 1234 after them that must stay untouched."""
    bufs = []

    def make(shape, dtype):
        n = int(np.prod(shape))
        flat = torch.full((n + GUARD,), 1234.0, dtype=dtype, device="cuda")
        flat[:n] = float("nan")
        bufs.append((flat, n))
        return flat[:n].view(shape)
    monkeypatch.setattr(R, "nan_output", make)
    return bufs


def check_guards(bufs):
    for flat, n in bufs:
        assert bool((flat[n:] == 1234.0).all()), "the convolution wrote past its output"


@pytest.mark.gpu
@pytest.mark.parametrize("case", cases(), ids=[c[0] for c in cases()])
def test_epilogue_vs_fp64_and_digest(rf, guarded, case):
    name, engine, cin, cout, sizes, res, stride = case
    xs, w, bias, rs = layer_inputs(case)
    _, y = R.check_conv(rf, engine, xs, w, bias, rs, stride, True, name)
    check_guards(guarded)
    assert digest(y) == DIGESTS[name], name


@pytest.mark.gpu
@pytest.mark.parametrize("case", dual_cases(), ids=[c[0] for c in dual_cases()])
def test_epilogue_dual_vs_fp64_and_digest(rf, guarded, case):
    from test_gpu_split import dual_check
    x1s, x2s, w1, w2, bias = dual_inputs(case)
    worst, y = dual_check(rf, x1s, x2s, w1, w2, bias, case[4], True)
    print("%s: worst error / allowance %.3g" % (case[0], worst))
    check_guards(guarded)
    assert digest(y) == DIGESTS[case[0]], case[0]


def test_cases_cover_the_tile_counts():
    """MANY gives a partial last flat tile and more than 3 tiles per CTA on 132 SMs at both N-tile counts; FEW one pixel tile."""
    pix = sum(h * w for h, w in MANY)
    assert pix % 128 == 9 and (pix + 127) // 128 == 313
    assert 313 * 2 >= 3 * 132
    assert sum(h * w for h, w in FEW) <= 128


@pytest.mark.gpu
def test_many_tiles_per_cta_on_this_gpu(rf):
    assert 2 * ((sum(h * w for h, w in MANY) + 127) // 128) >= 3 * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_epilogue_two_streams(rf):
    """Three layers launched on three streams at once, each with its own output: each gives its digest."""
    picks = [c for c in cases() if c[0] in ("ki4 res 256 many", "ki8 nores 256 few", "ki2 res 256 many")]
    calls = []
    for case in picks:
        name, engine, cin, cout, sizes, res, stride = case
        xs, w, bias, rs = layer_inputs(case)
        hw = [(x.shape[2], x.shape[3]) for x in xs]
        P = sum(h * ww for h, ww in hw)
        xd, _ = R.operand(R.nhwc(xs), "split")
        wd, _ = R.operand(w.permute(0, 2, 3, 1).reshape(cout, cin).contiguous(), "split")
        rd = R.operand(R.nhwc(rs), "split")[0].contiguous().cuda() if res else None
        y = torch.full((2, P, cout), float("nan"), dtype=torch.float16, device="cuda")
        calls.append((name, xd.contiguous().cuda(), hw, cin, wd.contiguous().cuda(), bias.cuda(), rd, cout, y))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in calls]
    for _ in range(3):
        for s, (name, xd, hw, cin, wd, b, rd, cout, y) in zip(streams, calls):
            with torch.cuda.stream(s):
                y.fill_(float("nan"))
                R.conv_call(rf, xd, hw, cin, None, wd, b, rd, cout, 1, 1, 0, True, 4, y)
        torch.cuda.synchronize()
        for name, *_, y in calls:
            assert digest(y) == DIGESTS[name], name


def test_timeline_phases():
    """tools/conv_tile_timeline.py: per-tile phases from the stamps (ns), the next tile of a CTA gridDim tiles on."""
    import conv_tile_timeline as T
    st = np.zeros((3, T.TL_WORDS), dtype=np.int64)
    st[0, :5] = [1000, 3000, 9000, 9500, 12000]
    st[0, 14] = 4000
    st[1, :5] = [2000, 2500, 8000, 8000, 9000]
    st[2, :5] = [13000, 14000, 20000, 21000, 22000]
    ph = T.tile_phases(st, 3, 2)
    assert ph[0] == {"wait_k0": 2.0, "k_loop": 6.0, "resid": 0.5, "epi": 2.5, "tile": 12.0, "lead": 5.0}
    assert ph[1]["tile"] == 7.0 and ph[2]["tile"] == 9.0


def record():
    """The digests of every case on the library in use (run with the kernel whose bits these tests hold)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from test_gpu_split import dual_check
    import ransac_flow_b200 as rf
    out = {}
    for case in cases():
        xs, w, bias, rs = layer_inputs(case)
        out[case[0]] = digest(R.run_conv(rf, case[1], xs, w, bias, rs, case[6], True)[-1])
    for case in dual_cases():
        x1s, x2s, w1, w2, bias = dual_inputs(case)
        out[case[0]] = digest(dual_check(rf, x1s, x2s, w1, w2, bias, case[4], True)[1])
    return out


# recorded with the kernel that loaded the bias and the residual one channel pair at a time (an H100 80GB HBM3)
DIGESTS = {
    "ki1 res 256 many": "cf09fcfd1eeffc53ee86ef46f4304ce7da126092670916ee5b190d2716869535",
    "ki1 nores 256 many": "f3272f9ba97ee33b49421e97daccb6cfeacc8985e11b00523dc1073ec56e76be",
    "ki2 res 256 many": "efd93099488538caac09ed8c9ddddcbde1a080fc29446c259364e5d413e0f1aa",
    "ki2 nores 256 many": "bdfe8402cf0b15b0c8365123d2e76b00e97eb8c2ce8ce864fbc4dda8729be35e",
    "ki4 res 256 many": "f811225875fe6d520753b30a27e7d477a39969a390f5d278bb359a0f79c3b240",
    "ki4 nores 256 many": "e2777280eeebd8af6bd62f4a89248ccc0c6e1c902279368077dc932252f70451",
    "ki8 res 256 many": "bd23150b0fcaa894f519ad082425174111424666e9ffceff33841477dfc2bb15",
    "ki8 nores 256 many": "cb7387607bb8869032ac7b9ac77fafe1bbf6fe8382b4380289f1badff26ee542",
    "ki4 res 192 many": "e4875075f219324b1ab15243044d560b9aaff9a2683d09d1130ddb34061fc6f9",
    "ki8 res 256 few": "9b79667ea5288b1b54f4a3410536639b026dfa43a5bcb5a8ee0135bee16f8e29",
    "ki4 nores 192 many": "9a2369447c00138172e914a5c8c1a84a6cd1362515270127e10bde76e89ff3b1",
    "ki8 nores 256 few": "9ec26ff257d21743d0d5215705f4dee6e5cd1e9468cc85d03dbdc5bd6d136776",
    "ki4 res 256 stride2": "82ff4760d1bebf8540300d16b514c74c389b84a677182437c8d2fa00b673f537",
    "engine4 ki2 res 56 many": "703d9fbb45f941e8635767c6a6cbc37509a00d4fbe64298e5ca01b331d6a40ca",
    "engine4 ki2 nores 56 many": "11ac9f96ad9f8a46a7e45fe4975f4dcc4cce34124664792356517b0e908849da",
    "engine2 ki2 res 56 many": "4965a1471e19efa7e799a91ae15b20e1166cbe582c570f0df28464120540940c",
    "engine2 ki2 nores 56 many": "02fae46113e3e54e4c4ed2debed47269ce96e2d99ff94c5d83c5db3a63d71307",
    "engine2 ki2 res 136 many": "a872196cc88e0b3a9d67e86f50b5006eccfc2006a583d0689483e0b5f2aa5e55",
    "engine2 ki2 nores 136 many": "7bdcdbbdc478aef3849bf5f72b31980cf376fa30a653cddd807f60efc0ada50e",
    "dual ki2 stride1": "d39f1c2d915f236d6ab2290acef660c44097c2b89656da25bb5de67b025c84f8",
    "dual ki6 stride2": "72cbe50c21f5120e1f707d14e38c4b830be0c6f684b1eb61378fb5dc8ee0a0d5",
}


if __name__ == "__main__":
    import json
    print(json.dumps(record(), indent=1))
