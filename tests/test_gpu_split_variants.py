"""The split engine under the fused / plain down-sampling topology (RF_FUSE_DOWNSAMPLE, read when the trunk's split program is built).  Each variant
runs tests/split_variant_probe.py in its own process on the same seeded inputs.  The fused down-sampling branch accumulates in
one fp32 chain what the plain topology rounds to 22 bits twice: fp32-grade tolerance on the trunk, and the stand-alone layers,
which do not depend on the switch, bit-identical."""
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
        for k in [k for k in e if k.startswith("RF_FUSE_")]:
            del e[k]
        e.update({k: str(v) for k, v in env.items()})
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "split_variant_probe.py"), str(out)], env=e, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        _CACHE[key] = dict(np.load(out))
    return _CACHE[key]


LAYERS = ["halo128", "halo256res", "halo64", "shallow_ds", "shallow_res", "res_k256", "tap_deep", "tap_s2"]


def test_fused_downsampling_is_fp32_grade_equal_to_two_convolutions(tmp_path_factory):
    base, var = probe(tmp_path_factory), probe(tmp_path_factory, RF_FUSE_DOWNSAMPLE=0)
    assert np.abs(base["trunk"] - var["trunk"]).max() <= 2e-5 * np.abs(var["trunk"]).max()
    for name in LAYERS:                      # the stand-alone layers do not depend on the topology switch
        assert np.array_equal(base[name], var[name]), name
