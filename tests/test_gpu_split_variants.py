"""The split engine under the kernel-selection switches of earlier builds (RF_SPLIT_*, RF_CORR_MMA3; the wgmma engine has one
kernel for all of them) and the fused / plain down-sampling topology (RF_FUSE_DOWNSAMPLE).  Every variant runs
tests/split_variant_probe.py in its own process on the same seeded inputs.  The selection switches must not change any output
element: BIT-identical.  The fused down-sampling branch accumulates in one fp32 chain what the plain topology rounds to 22 bits
twice: fp32-grade tolerance."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CACHE = {}


def probe(tmp_path_factory, **env):
    key = tuple(sorted(env.items()))
    if key not in _CACHE:
        out = tmp_path_factory.mktemp("probe") / "out.npz"
        e = dict(os.environ)
        for k in [k for k in e if k.startswith(("RF_SPLIT_", "RF_FUSE_", "RF_CORR_MMA3"))]:
            del e[k]
        e.update({k: str(v) for k, v in env.items()})
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "split_variant_probe.py"), str(out)], env=e, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        _CACHE[key] = dict(np.load(out))
    return _CACHE[key]


def halves(u16):
    """split planes (uint16 views of fp16 hi / lo * 2^11) -> float64 values"""
    h = u16.view(np.float16).astype(np.float64)
    return h[0] + h[1] / 2048.0


LAYERS = ["halo128", "halo256res", "halo64", "shallow_ds", "shallow_res", "res_k256", "tap_deep", "tap_s2"]


@pytest.mark.parametrize("env", [dict(RF_SPLIT_EPW=4), dict(RF_SPLIT_HALO_BN=64), dict(RF_SPLIT_SHALLOW=0), dict(RF_SPLIT_RES_BN=64),
                                 dict(RF_SPLIT_RES2=0), dict(RF_SPLIT_BN=64), dict(RF_SPLIT_BN_MIN=128)])
def test_tile_shape_variants_are_bit_identical(tmp_path_factory, env):
    base, var = probe(tmp_path_factory), probe(tmp_path_factory, **env)
    for name in LAYERS:
        assert np.array_equal(base[name], var[name]), (env, name)
    assert np.array_equal(base["trunk"], var["trunk"]), env


def test_two_instruction_split_step_is_fp32_grade_equal_to_three(tmp_path_factory):
    base, var = probe(tmp_path_factory), probe(tmp_path_factory, RF_SPLIT_DBG=16, RF_CORR_MMA3=1)
    for name in LAYERS:
        a, b = halves(base[name]), halves(var[name])
        assert np.abs(a - b).max() <= 1e-6 * max(1.0, np.abs(b).max()), name
    assert np.abs(base["trunk"] - var["trunk"]).max() <= 2e-5 * np.abs(var["trunk"]).max()
    # random unit rows: score gaps are far above 1e-6, the mutual matches cannot move
    assert np.array_equal(base["corr_i1"], var["corr_i1"]) and np.array_equal(base["corr_i2"], var["corr_i2"]) and len(base["corr_i1"]) > 10


def test_fused_downsampling_is_fp32_grade_equal_to_two_convolutions(tmp_path_factory):
    base, var = probe(tmp_path_factory), probe(tmp_path_factory, RF_FUSE_DOWNSAMPLE=0)
    assert np.abs(base["trunk"] - var["trunk"]).max() <= 2e-5 * np.abs(var["trunk"]).max()
    for name in LAYERS:                      # the stand-alone layers do not depend on the topology switch
        assert np.array_equal(base[name], var[name]), name
