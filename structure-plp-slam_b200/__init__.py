"""structure-plp-slam_b200 -- H100-native (sm_90a) hot path of Structure-PLP-SLAM.

The product is the C-ABI shared library ``libplpslam_b200.so`` (see ``include/plpslam_b200.h``)
built from ``csrc/*.cu``.  This Python package is only a thin ctypes binding used by the tests
and ``bench.py``; it never computes anything itself and there is no CPU fallback: loading fails
loudly if the library has not been built, and every compute call raises if no CUDA device exists.

The directory name contains '-' so it is loaded by path (see ``load_package`` in tests/conftest.py).
"""
from .capi import (  # noqa: F401
    Context,
    OrbExtractor,
    LineFeatureTracker,
    BowVocabulary,
    StereoRectifier,
    KP_DTYPE,
    KEYLINE_DTYPE,
    PT_OBS_DTYPE,
    LINE_OBS_DTYPE,
    PlpError,
    lib,
    lib_path,
    declared_symbols,
)
