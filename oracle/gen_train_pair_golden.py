"""Generate tests/golden/train_pair_*.npz by running the code cells of the reference's
train/generate_coarse_aligned_pair.ipynb, read from its JSON at run time, on the CPU:

    python -m oracle.gen_train_pair_golden          # needs the reference checkout ($RF_REFERENCE)

Harness-side shims only (``gen_golden.cpu_as_cuda`` / ``replay_randint``; ``%`` magic lines dropped; matplotlib stubbed; kornia,
absent, served by the oracle's ``warp_grid``): ``torch.load`` returns seeded ``synthdata.resnet50_conv4_state`` weights in the
MoCo checkpoint layout the notebook loads (cell 2), and ``Image.open`` returns the synthetic ``synthdata.make_pair`` images.
No reference source is stored; only inputs and outputs (of ``I2Sample``, every ``ROW_STEP``-th row: the synthetic texture does
not compress, and the warp kernel is checked on every pixel against its own composition and fp64 elsewhere).

  train_pair_480   : the notebook's settings (minSize 480, nbIter 10000) on a 240 x 160 pair (resized to 720 x 480): kept
  train_pair_small : minSize 64 on a 96 x 64 pair: M <= 50, not kept
"""
import contextlib
import json
import os
import sys
import types

import numpy as np
import PIL.Image as Image
import torch

from . import synth
from . import warp_oracle as WO
from .gen_golden import REF, cpu_as_cuda, replay_randint, save

NOTEBOOK = os.path.join(REF, "train", "generate_coarse_aligned_pair.ipynb")
ROW_STEP = 4
CASES = {"train_pair_480": dict(pair=3, h=160, w=240, minSize=480), "train_pair_small": dict(pair=4, h=64, w=96, minSize=64)}


def code_cells():
    nb = json.load(open(NOTEBOOK))
    cells = [c for c in nb["cells"] if c["cell_type"] == "code"]
    return ["\n".join(l for l in "".join(c["source"]).splitlines() if not l.lstrip().startswith("%")) for c in cells]


class _Warper:                          # kornia is absent: the oracle's restatement stands in
    def __init__(self, h, w):
        self.h, self.w = h, w

    def warp_grid(self, H):
        return WO.warp_grid(H, self.h, self.w)


@contextlib.contextmanager
def notebook_shims(images, resnet_sd):
    plt = types.ModuleType("matplotlib.pyplot")
    for name in ("figure", "subplot", "axis", "imshow", "show"):
        setattr(plt, name, lambda *a, **k: None)
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    kornia = types.ModuleType("kornia")
    kornia.geometry = types.SimpleNamespace(HomographyWarper=_Warper)
    stubs = {"matplotlib": mpl, "matplotlib.pyplot": plt, "kornia": kornia, "kornia.geometry": kornia.geometry}
    saved_mods = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    real_open, real_load = Image.open, torch.load
    it = iter(images)
    Image.open = lambda path, *a, **k: Image.fromarray(next(it))
    torch.load = lambda *a, **k: {"model": {"module." + k: v for k, v in resnet_sd.items()}}
    sys.path[:0] = [os.path.join(REF, "utils"), os.path.join(REF, "model")]
    try:
        with cpu_as_cuda():
            yield
    finally:
        Image.open, torch.load = real_open, real_load
        del sys.path[:2]
        for k, v in saved_mods.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def full_resnet50_state():
    """The notebook's ``resNetfeat.load_state_dict`` is strict: seeded conv4 weights plus the (unused) layer4 / fc entries of a
    fresh model."""
    sys.path.insert(0, os.path.join(REF, "model"))
    try:
        from resnet50 import resnet50
    finally:
        sys.path.pop(0)
    torch.manual_seed(0)
    sd = resnet50().state_dict()
    sd.update(synth.resnet50_conv4_state(0))
    return sd, synth.resnet50_conv4_state(0)


def run_case(name, pair, h, w, minSize):
    src, tgt, _ = synth.make_pair(pair, h, w)
    full, _ = full_resnet50_state()
    cells = code_cells()
    ns = {"__name__": "__notebook__"}
    rec = []
    with notebook_shims([src, tgt], full), torch.no_grad():
        exec(compile(cells[0], NOTEBOOK + ":cell0", "exec"), ns)
        ns["minSize"] = minSize
        for i, code in enumerate(cells[1:], 1):
            if i == len(cells) - 2:                                      # the RANSAC cell: record its draw
                torch.manual_seed(1000)
                with replay_randint(None, rec):
                    exec(compile(code, NOTEBOOK + ":cell%d" % i, "exec"), ns)
            else:
                exec(compile(code, NOTEBOOK + ":cell%d" % i, "exec"), ns)
        from torchvision import transforms
        kept = len(ns["match1Inlier"]) > 50
        I2Sample = np.asarray(transforms.ToPILImage()(ns["I2Sample"].squeeze().cpu())) if kept else np.zeros((0, 0, 3), np.uint8)
        sizes = np.array([ns[k].size for k in ("I1Down2", "I1", "I1Up2", "I2")], dtype=np.int64)
        save(name, src=src, tgt=tgt, minSize=np.int64(minSize), nbIter=np.int64(ns["nbIter"]), sizes=sizes,
             nbMatch=np.int64(len(ns["match1"])), samples=rec[0][1].astype(np.int32),
             match1=ns["match1"].numpy(), match2=ns["match2"].numpy(), H=np.asarray(ns["bestParam"], dtype=np.float32),
             isInlier=np.asarray(ns["match1Inlier"], dtype=bool), nbInlier=np.int64(ns["bestInlier"]), kept=np.bool_(kept),
             I2Sample=I2Sample[::ROW_STEP], row_step=np.int64(ROW_STEP))


def main():
    for name, case in CASES.items():
        if len(sys.argv) < 2 or name in sys.argv[1:]:
            run_case(name, **case)


if __name__ == "__main__":
    main()
