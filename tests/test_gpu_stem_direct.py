"""The direct stems of engines 2 and 4 (RF_OP_STEM7): the ResNet-50 stem (7x7 / 2 / pad 3, fused with its 3x3 / 2 max-pool)
and the FeatureExtractor stem (3x3 / 1 / pad 1) in one kernel that gathers each thread's wgmma A fragments from the staged
input window.  It issues the same three split MMAs per k16 step on the same operand values as the kernels before it (the
ResNet stem's patch tile in shared memory; for the FeatureExtractor, im2col + a 1x1 convolution) and skips only k16 steps
whose products are all zero, so every output keeps the bits of those kernels: SHA-256 digests recorded with them.  A digest
says that bits changed, not that they are wrong: the numerical reference of both stems is tests/test_gpu_stem_geometry.py, and
the digests are re-recorded after a deliberate change of arithmetic only once that file passes."""
import hashlib
import importlib.util
import os

import pytest
import torch

from stem_ref import stem_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# odd sizes on both sides of the 32 x 4 stem tile and the 15 x 2 pooled step
RAGGED = [(17, 35), (3, 5), (9, 33), (15, 61), (65, 15), (121, 123), (130, 97), (251, 7)]
FE_SIZES = {"480x640": [(480, 640)], "97x131": [(97, 131)]}


def _profile_tool():
    spec = importlib.util.spec_from_file_location("conv_layer_profile", os.path.join(ROOT, "tools", "conv_layer_profile.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.cat([torch.randn(h * w, 3, generator=g) for h, w in sizes]).cuda()


def _digest(y):
    torch.cuda.synchronize()
    return hashlib.sha256(y.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def resnet_stem_pool(seed=1):
    from ransac_flow_b200.program import LayerProgram
    P = LayerProgram(3, device="cuda")
    P.maxpool(P.stem7_fused(0, *stem_args(seed, 7)), 3, 2, 1)
    return P


def fe_stem(seed=3):
    from ransac_flow_b200.program import LayerProgram
    P = LayerProgram(3, device="cuda")
    P.stem7_fused(0, *stem_args(seed, 3))
    return P


def feature_extractor():
    import ransac_flow_b200 as rf
    from oracle import synth
    net = rf.model.FeatureExtractor()
    net.load_state_dict(synth.feature_extractor_state(0))
    return net.cuda().eval()


def digest_outputs(rf, stems=(resnet_stem_pool, fe_stem)):
    """SHA-256 of the output bytes on engines 2 and 4: the ResNet stem + max-pool on the config-2 batch of one pair and on odd
    sizes, the FeatureExtractor stem alone and the whole FeatureExtractor at 480 x 640 and 97 x 131."""
    resnet, fe = stems
    out = {}
    for engine, name in ((2, "f16"), (4, "f16x3")):
        for sname, sizes in (("config2", _profile_tool().pair_sizes()), ("ragged", RAGGED)):
            out["resnet stem+pool %s engine %d" % (sname, engine)] = _digest(resnet().run(rf.ops.Ragged(_images(sizes, 2), sizes), engine)[0])
        net = feature_extractor()
        for sname, sizes in FE_SIZES.items():
            x = rf.ops.Ragged(_images(sizes, 4), sizes)
            out["fe stem %s engine %d" % (sname, engine)] = _digest(fe().run(x, engine)[0])
            rf.model.set_engine(name)
            try:
                out["feature extractor %s engine %d" % (sname, engine)] = _digest(net.forward_ragged(x).data)
            finally:
                rf.model.set_engine("fp32")
    return out


# recorded with the kernels before the register-A stem (an H100 80GB HBM3)
DIGESTS = {
    "resnet stem+pool config2 engine 2": "5013cd113c9fecbaefffaa1cfef786d248e5a1ac21d17d9a1a2bb6322d5c80ad",
    "resnet stem+pool ragged engine 2": "7fe2bfecc3280941f9ba1810bcd83b8f44b3e8e396e5514db8aec8c3a673d3d7",
    "fe stem 480x640 engine 2": "a8f10f43252fdeb9258f5ee87e0bc625d77ac4736cb099a2c874eaba6a7fd00c",
    "feature extractor 480x640 engine 2": "c4d7e0644edc4529ccead7a9f4d6782ff3041d6c021b02df644ed43ebd5a44d8",
    "fe stem 97x131 engine 2": "a6545c5accf228203be248cccf925f21ac972857d40145b080e27e14b84a60f4",
    "feature extractor 97x131 engine 2": "9ec0fa445c29f8332e50eff5caa5928bd207e7cb0f9853bd372052a1aaa1fbc4",
    "resnet stem+pool config2 engine 4": "4891d79489d840896238963b4e1ac63ffdade168260820fe720217445c0deb97",
    "resnet stem+pool ragged engine 4": "f624027e71e3a3222186f1cbc60531922f23e5c29bd1e53a8904c0f081ff85cb",
    "fe stem 480x640 engine 4": "f285677d03510f3035860a166618a4af3311e1d1591d6c71032eeb089c05bc49",
    "feature extractor 480x640 engine 4": "cbd0a94c96d2eb2767e653d8f4c383719a5d28ab57b9ba955508cf2be45be234",
    "fe stem 97x131 engine 4": "e43615fc602f2d300beb82e7279b7a0859de0027fc689266e7dbccf373f480fa",
    "feature extractor 97x131 engine 4": "1577a7c03e1b3a3bcea73a1a8dbe94ac98e7041ad41d16ad66ae366d077ba68b",
}


@pytest.mark.gpu
def test_stems_bit_identical_to_previous_kernels(rf):
    got = digest_outputs(rf)
    print(got)
    assert got.keys() == DIGESTS.keys()
    for name in got:
        assert got[name] == DIGESTS[name], name


@pytest.mark.parametrize("engine", [2, 4])
def test_feature_extractor_program_has_no_im2col(engine):
    """Engines 2 and 4 run the FeatureExtractor stem as one RF_OP_STEM7 op on the fp32 image: no im2col matrix."""
    import ransac_flow_b200 as rf
    from ransac_flow_b200.program import RF_OP_IM2COL, RF_OP_STEM7
    net = rf.model.FeatureExtractor()
    ops = [o[0] for o in net._folded(engine).ops]
    assert ops[0] == RF_OP_STEM7 and RF_OP_IM2COL not in ops
    assert tuple(net._folded(engine).ops[0][5:8]) == (3, 1, 1)
    rows = _profile_tool().layer_model(net._folded(engine).ops, [(480, 640)])
    assert rows[0]["op"] == "stem7" and rows[0]["out_hw"] == [(480, 640)] and rows[0]["K"] == 27 and rows[0]["KI"] == 1
    assert rows[0]["bytes"] == 480 * 640 * (3 * 4 + 64 * 4) and rows[0]["bound"] == "hbm"
