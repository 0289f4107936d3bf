"""goslam_b200 — H100-native (sm_90a) drop-in for GO-SLAM's per-keyframe dense-update path.

Hot path only (SURVEY.md §8): correlation-volume build + radius-3 lookup, on-the-fly
windowed correlation, dense Gauss-Newton bundle adjustment, frame distance / reprojection
and the fused hash-grid neural-surface ray marcher, as hand-written CUDA behind a C-ABI
(include/goslam_b200.h), bound to PyTorch under the reference's own operator names.

    import goslam_b200
    goslam_b200.install()            # registers `droid_backends` and `lietorch` in sys.modules
    import droid_backends            # -> goslam_b200.droid_backends

The on-disk package directory is `go-slam_b200/` (not an importable identifier); the
`goslam_b200/` stub at the repo root aliases it.
"""
import sys as _sys

__version__ = "0.1.0"


def install(force=True):
    """Register the reference's native-module names so its Python imports resolve to us
    (src/modules/corr.py:4, src/depth_video.py:2-3, src/geom/projective_ops.py:2)."""
    from . import droid_backends as _db
    from . import lietorch as _lt
    for name, mod in (("droid_backends", _db), ("lietorch", _lt)):
        if force or name not in _sys.modules:
            _sys.modules[name] = mod
    return _db, _lt


def __getattr__(name):
    """goslam_b200.FactorGraph / DepthVideo / MultiviewFilter / MotionFilter / CorrBlock / AltCorrBlock / BasicEncoder /
    InstantNeuS, imported on first use"""
    import importlib
    where = {"FactorGraph": ".factor_graph", "DepthVideo": ".depth_video",
             "MultiviewFilter": ".multiview_filter", "MotionFilter": ".motion_filter", "CorrBlock": ".modules.corr",
             "AltCorrBlock": ".modules.corr", "BasicEncoder": ".modules.extractor", "InstantNeuS": ".neus"}
    if name in where:
        return getattr(importlib.import_module(where[name], __name__), name)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))


def build_library(verbose=False, force=False):
    """compile csrc/*.cu for sm_90a into go-slam_b200/libgoslam_b200.so"""
    import importlib
    _b = importlib.import_module(__name__ + '.build')
    return _b.build(verbose=verbose, force=force)
