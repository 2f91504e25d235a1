"""ransac_flow_b200: H100-native (sm_90a) implementation of RANSAC-Flow's per-pair inference
hot path behind the reference's own Python API (SURVEY.md section 8).

Modules mirror the reference's module names: ``outil`` (utils/outil.py), ``model``
(model/model.py), ``coarseAlignFeatMatch`` (the CoarseAlign variants), ``kornia_geometry``
(kornia.geometry.HomographyWarper), plus ``pipeline`` (PredFlowMask / pair loop / getFlow / KITTI two-level flow),
``results`` (the drivers' .npy formats and the getResults metrics),
``shard`` (pair sharding over GPUs) and ``dropin`` (run the reference's scripts unchanged).
All arithmetic is in ``libransacflow_b200.so`` (C ABI: include/ransacflow_b200.h).
Importing fails if that library is missing; compute calls fail without a CUDA device.
"""
from . import _lib  # noqa: F401  (loads the C-ABI library or raises)
from . import ops, outil, model, kornia_geometry, coarseAlignFeatMatch, pipeline, results  # noqa: F401
from .coarseAlignFeatMatch import CoarseAlign, CoarseAlignA, CoarseAlignB, CoarseAlignC  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    """``validation`` (train/validation.py on the device) and ``corr_results`` (evalCorr/getResults.py on the device) are
    imported on first use, so that ``python -m ransac_flow_b200.validation`` (``.corr_results``) runs the module once, as
    ``__main__``, instead of after a package-level import of it."""
    if name in ("validation", "corr_results"):
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
