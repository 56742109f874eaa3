"""plsvo_b200 — H100-native (sm_90a) implementation of PL-SVO's per-frame optimisation path.

Package directory is `pl-svo_b200/` (hyphenated, as the repo contract names it); import it through
the `plsvo_b200` shim module at the repo root.
"""
from . import abi, dist, synth  # noqa: F401
from .api import (ATANCamera, Context, DepthFilter, Matcher, PinholeCamera, SparseImgAlign, createImgPyramid, default_context, feature_alignment,  # noqa: F401
                  optimizeStructure, pose_optimizer, track_raw)

__version__ = "0.1.0"
