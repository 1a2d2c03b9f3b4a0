"""pyscenedetect_b200 - H100-native (sm_90a) per-frame content-score engine for PySceneDetect.

Only the hot path is here: the four fast-cut detectors' `process_frame` arithmetic and the
SceneManager downscale, as sm_90a CUDA kernels behind a C-ABI (include/psd_b200.h).
Importing the package does not need a GPU; constructing an engine does (no CPU fallback).
"""

from .compat import FlashFilter, FrameTimecode, SceneDetector, StatsManager

__version__ = "0.1.0"
__all__ = ["FlashFilter", "FrameTimecode", "SceneDetector", "StatsManager", "__version__"]
