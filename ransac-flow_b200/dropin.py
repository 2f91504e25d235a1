"""Run a reference driver script unchanged on top of this package.

    python -m ransac_flow_b200.dropin /path/to/RANSAC-Flow/quick_start/align2images.py --img1 ... --img2 ...

The reference's scripts import their collaborators by bare module name after ``sys.path.append``
(quick_start/align2images.py:2-7, evaluation/evalHpatch/evaluation.py:1-10).  ``install()`` puts this
package's mirrors into ``sys.modules`` under those names *before* the script runs, so
``from coarseAlignFeatMatch import CoarseAlign``, ``import outil``, ``import model`` and
``import kornia.geometry as tgm`` resolve here; the script itself is executed byte-for-byte
(``runpy.run_path``) from its own directory.  The CoarseAlign variant is chosen from the script's
location (quick_start -> C, evalYFCC -> B, other evaluation dirs -> A).
"""
import os
import runpy
import sys
import types


def variant_for(script_path):
    p = os.path.abspath(script_path).replace("\\", "/")
    if "/quick_start/" in p:
        return "C"
    if "/evalYFCC/" in p:
        return "B"
    return "A"


def install(variant="A"):
    from . import coarseAlignFeatMatch as ca
    from . import kornia_geometry, model, outil
    mod = types.ModuleType("coarseAlignFeatMatch")
    mod.CoarseAlign = {"A": ca.CoarseAlignA, "B": ca.CoarseAlignB, "C": ca.CoarseAlignC}[variant]
    mod.__doc__ = "ransac_flow_b200 drop-in (variant %s)" % variant
    sys.modules["coarseAlignFeatMatch"] = mod
    sys.modules["outil"] = outil
    sys.modules["model"] = model
    kornia = types.ModuleType("kornia")
    kornia.geometry = kornia_geometry
    sys.modules["kornia"] = kornia
    sys.modules["kornia.geometry"] = kornia_geometry
    try:                                     # removed from SciPy >= 1.3 but still imported by the evaluation scripts
        import scipy.misc as misc
        if not hasattr(misc, "imresize"):
            misc.imresize = imresize
    except Exception:  # noqa: BLE001
        pass
    return mod


def imresize(arr, size, interp="bilinear"):
    """``scipy.misc.imresize`` of SciPy <= 1.2 for an (h, w) ``size``, the form the drivers use
    (evaluation/evalHpatch/evaluation.py:180 ``imresize(It_bg, (h, w)) < 128``): an array that is not uint8 is first
    byte-scaled to 0..255 like ``scipy.misc.bytescale`` ((x - min) * 255 / (max - min), span 1 when constant, + 0.5, truncated),
    so a 0 / 1 float mask becomes 0 / 255; then a PIL resize to (w, h) with the chosen filter.  Returns uint8."""
    import numpy as np
    import PIL.Image as Image
    a = np.asarray(arr)
    if a.dtype != np.uint8:
        cmin, cmax = a.min(), a.max()
        cscale = cmax - cmin
        if cscale == 0:
            cscale = 1
        scale = float(255 - 0) / cscale
        a = ((a - cmin) * scale + 0).clip(0, 255) + 0.5
        a = a.astype(np.uint8)
    resample = {"nearest": Image.NEAREST, "lanczos": Image.LANCZOS, "bilinear": Image.BILINEAR, "bicubic": Image.BICUBIC,
                "cubic": Image.BICUBIC}[interp]
    return np.asarray(Image.fromarray(a).resize((int(size[1]), int(size[0])), resample))


def select_engine(name=None):
    """The conv / correlation engine the mirrored modules run on: ``$RF_ENGINE`` or 'f16x3' - the fp32-grade tensor-core engine
    (fp16 hi / lo split operands), whose results reproduce the reference's fp32 arg-max; 'fp32' = exact-FMA SIMT kernels."""
    from . import model, outil
    name = name or os.environ.get("RF_ENGINE", "f16x3")
    model.set_engine(name)
    outil.corr_precision = {"fp32": 0, "tf32": 1}.get(name, 2)
    return name


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit(__doc__)
    script = os.path.abspath(argv[0])
    install(variant_for(script))
    select_engine()
    sys.argv = [script] + argv[1:]
    os.chdir(os.path.dirname(script))
    sys.path.insert(0, os.path.dirname(script))
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
