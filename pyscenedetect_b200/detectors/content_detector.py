"""Drop-in for scenedetect.detectors.ContentDetector (content_detector.py:49-243): same
constructor, metric keys, cut semantics; the HSV conversion, |frame[t]-frame[t-1]| means,
Canny/dilate edge delta and the weighted score run on the GPU."""

from __future__ import annotations

import typing as ty

import numpy as np

from .._capi import F_EDGES, F_HSV
from ..compat import FlashFilter
from ._base import EngineDetector


class ContentDetector(EngineDetector):
    """Detects fast cuts using changes in colour and intensity between frames (HSV space)."""

    class Components(ty.NamedTuple):
        """Components that make up a frame's score, and their default values
        (content_detector.py:58-71)."""

        delta_hue: float = 1.0
        delta_sat: float = 1.0
        delta_lum: float = 1.0
        delta_edges: float = 0.0

    DEFAULT_COMPONENT_WEIGHTS = Components()
    LUMA_ONLY_WEIGHTS = Components(delta_hue=0.0, delta_sat=0.0, delta_lum=1.0, delta_edges=0.0)
    FRAME_SCORE_KEY = "content_val"
    METRIC_KEYS: ty.ClassVar[list[str]] = [FRAME_SCORE_KEY, *Components._fields]

    def __init__(
        self,
        threshold: float = 27.0,
        min_scene_len=15,
        weights: "ContentDetector.Components" = DEFAULT_COMPONENT_WEIGHTS,
        luma_only: bool = False,
        kernel_size: int | None = None,
        filter_mode: FlashFilter.Mode = FlashFilter.Mode.MERGE,
    ):
        super().__init__()
        self._threshold: float = threshold
        self._weights = ContentDetector.Components(*weights)
        if luma_only:
            self._weights = ContentDetector.LUMA_ONLY_WEIGHTS
        self._kernel_size = 0
        if kernel_size is not None:
            if kernel_size < 3 or kernel_size % 2 == 0:
                raise ValueError("kernel_size must be odd integer >= 3")
            self._kernel_size = int(kernel_size)
        self._frame_score: float | None = None
        self._flash_filter = FlashFilter(mode=filter_mode, length=min_scene_len)
        self._scores: list = []  # every frame's score, frame 0 included (0.0)

    def get_metrics(self):
        return ContentDetector.METRIC_KEYS

    def required_features(self, stats: bool = False) -> int:
        # content_detector.py:158: edges are computed when weighted OR a StatsManager is attached
        calculate_edges = (self._weights.delta_edges > 0.0) or self.stats_manager is not None or stats
        return F_HSV | (F_EDGES if calculate_edges else 0)

    def edge_kernel_size_arg(self) -> int:
        return self._kernel_size

    @property
    def event_buffer_length(self) -> int:
        return self._flash_filter.max_behind

    # -- per-batch logic --
    def _score_batch(self, timecodes: list, first: int):
        """Device scan -> (scores, components); writes stats rows like content_detector.py:183-186."""
        n = len(timecodes)
        val, comps = self._engine.scan_content(self._weights, first=first, n=n)
        scores = []
        for i in range(n):
            is_first = (first + i) == self._base_index and not self._has_halo()
            if is_first:
                # content_detector.py:161-164: no previous frame -> 0.0, no metrics row
                scores.append(0.0)
                continue
            score = val[i]
            if self.stats_manager is not None:
                metrics = {self.FRAME_SCORE_KEY: score}
                metrics.update(dict(zip(ContentDetector.Components._fields, comps[i])))
                self.stats_manager.set_metrics(timecodes[i], metrics)
            scores.append(score)
        return scores

    def _has_halo(self) -> bool:
        return getattr(self, "_halo", False)

    def set_halo(self, frame_img: np.ndarray) -> None:
        """Time-shard support: `frame_img` is the frame preceding this detector's first frame."""
        eng = self._ensure_engine(self._as_batch(frame_img))
        eng.set_halo(frame_img)
        self._halo = True

    def _consume(self, timecodes: list, first: int) -> list:
        cuts = []
        for tc, score in zip(timecodes, self._score_batch(timecodes, first)):
            self._frame_score = score
            self._scores.append(score)
            above_threshold = bool(score >= self._threshold)
            cuts += self._flash_filter.filter(timecode=tc, above_threshold=above_threshold)
        return cuts
