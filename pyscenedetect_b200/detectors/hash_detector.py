"""Drop-in for scenedetect.detectors.HashDetector (hash_detector.py:27-158): same constructor, metric key
and cut rule; the perceptual hash of every frame (gray, INTER_AREA square, DCT low band > median) and the
Hamming distance between consecutive hashes are computed on the GPU."""

from __future__ import annotations

import math

import numpy as np

from .._capi import F_HASH
from ._base import EngineDetector


class HashDetector(EngineDetector):
    """Detects cuts using a perceptual hashing algorithm (DCT + median threshold)."""

    FEATURES = F_HASH

    def __init__(self, threshold: float = 0.35, size: int = 8, lowpass: int = 2, min_scene_len=15):
        super().__init__()
        if not (int(size) >= 1 and int(lowpass) >= 1):
            raise ValueError("HashDetector needs size >= 1 and lowpass >= 1")
        self._threshold = threshold
        self._min_scene_len = min_scene_len
        self._size = size
        self._size_sq = float(size * size)
        self._factor = lowpass
        self._last_scene_cut = None
        self._metric_key = f"hash_dist [size={self._size} lowpass={self._factor}]"
        self._halo = False

    def get_metrics(self):
        return [self._metric_key]

    def engine_kwargs(self) -> dict:
        return {"hash_size": int(self._size), "hash_lowpass": int(self._factor)}

    def set_halo(self, frame_img: np.ndarray) -> None:
        eng = self._ensure_engine(self._as_batch(frame_img))
        eng.set_halo(frame_img)
        self._halo = True

    def _consume(self, timecodes: list, first: int) -> list:
        dists = self._engine.scan_hash_dist(first=first, n=len(timecodes))
        cuts = []
        for i, timecode in enumerate(timecodes):
            if self._last_scene_cut is None:  # hash_detector.py:79-80
                self._last_scene_cut = timecode
            hash_dist_norm = dists[i]
            if math.isnan(hash_dist_norm):
                continue  # first frame: nothing to compare with yet (hash_detector.py:83)
            if self.stats_manager is not None:
                self.stats_manager.set_metrics(timecode, {self._metric_key: float(hash_dist_norm)})
            if hash_dist_norm >= self._threshold and (
                    (timecode - self._last_scene_cut) >= self._min_scene_len):
                cuts.append(timecode)
                self._last_scene_cut = timecode
        return cuts
