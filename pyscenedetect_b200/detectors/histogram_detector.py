"""Drop-in for scenedetect.detectors.HistogramDetector (histogram_detector.py:27-168)."""

from __future__ import annotations

import typing as ty

import numpy as np

from .._capi import F_YHIST
from ._base import EngineDetector, frame_format


class HistogramDetector(EngineDetector):
    """YUV-Y histogram per frame (fused GPU pass) + Pearson correlation with the previous
    frame's histogram (trailing device scan, cv2.normalize / HISTCMP_CORREL arithmetic)."""

    METRIC_KEYS: ty.ClassVar[list[str]] = ["hist_diff"]
    FEATURES = F_YHIST

    def __init__(self, threshold: float = 0.20, bins: int = 128, min_scene_len=15):
        super().__init__()
        self._threshold = max(0.0, min(1.0, 1.0 - threshold))
        if not 1 <= int(bins) <= 256:
            raise ValueError("bins must be in [1, 256] (8-bit luma)")
        self._bins = bins
        self._min_scene_len = min_scene_len
        self._last_cut = None
        self._metric_key = f"hist_diff [bins={self._bins}]"
        self._halo = False

    def get_metrics(self) -> list[str]:
        return [self._metric_key]

    def _validate(self, frames) -> None:
        shape, uint8 = frame_format(frames, self._frames_device())
        if not uint8:
            raise ValueError("Image must be 8-bit rgb for HistogramDetector")
        if shape[-1] != 3:
            raise ValueError("Image must have three color channels for HistogramDetector")

    def set_halo(self, frame_img: np.ndarray) -> None:
        eng = self._ensure_engine(self._as_batch(frame_img))
        eng.set_halo(frame_img)
        self._halo = True

    def _consume(self, timecodes: list, first: int) -> list:
        diffs = self._engine.scan_hist_correl(self._bins, first=first, n=len(timecodes))
        cuts = []
        for i, timecode in enumerate(timecodes):
            if not self._last_cut:  # histogram_detector.py:87-88 (a FrameTimecode is always truthy)
                self._last_cut = timecode
            if (first + i) == self._base_index and not self._halo:
                continue  # first frame: nothing to compare with yet
            hist_diff = diffs[i]
            if hist_diff <= self._threshold and (
                    (timecode - self._last_cut) >= self._min_scene_len):
                cuts.append(timecode)
                self._last_cut = timecode
            if self.stats_manager is not None:
                self.stats_manager.set_metrics(timecode, {self._metric_key: hist_diff})
        return cuts
