"""Shared machinery of the drop-in detectors: lazy engine creation, strict (one frame per
call, as SceneManager drives it: scene_manager.py:426-428) and batched submission."""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .. import _dlpack
from .._capi import F_EDGES
from ..compat import SceneDetector
from ..engine import Engine


@dataclass(frozen=True)
class PixelGroup:
    """What a detector needs from the fused pixel pass: the Engine arguments of detectors (or sweep cells) that
    can share one score pass."""

    features: int
    edge_kernel_size: int
    engine_kwargs: tuple  # sorted (name, value) pairs

    def make_engine(self, src_width: int, src_height: int, width: int, height: int, device: int = 0,
                    max_batch: int = 64) -> Engine:
        return Engine(src_width, src_height, self.features, width=width, height=height, device=device,
                      max_batch=max_batch, edge_kernel_size=self.edge_kernel_size, **dict(self.engine_kwargs))


def pixel_group_of(detector, stats: bool = False) -> PixelGroup:
    """The features a detector needs, its dilation kernel size argument when it uses the edge component
    (content_detector.py:135-138; 0 otherwise) and its extra Engine arguments (the hash geometry).  `stats`: as if a
    StatsManager were attached (the detector itself is not changed)."""
    feats = detector.required_features(stats)
    return PixelGroup(feats, detector.edge_kernel_size_arg() if feats & F_EDGES else 0,
                      tuple(sorted(detector.engine_kwargs().items())))


def frame_format(frames, device: int = 0) -> tuple[tuple, bool]:
    """(shape, whether the samples are uint8) of numpy frames, or of CUDA frames of `device` read from their DLPack
    view (ValueError for frames on another device)."""
    if _dlpack.is_dlpack(frames):
        return _dlpack.frame_format(frames, device)
    return frames.shape, frames.dtype == np.uint8


class EngineDetector(SceneDetector):
    """Base class: owns (or borrows) a `psd_engine` and feeds it frames.

    `process_frame(timecode, frame_img)` keeps the reference signature and semantics
    (detector.py:48-60).  `process_batch(timecodes, frames)` is the same computation for B
    frames per call; both produce identical cuts and metrics because the per-frame state
    machines below run on the same device-computed metric arrays.
    """

    #: PSD_F_* bits this detector needs from the fused pass
    FEATURES = 0

    def __init__(self):
        super().__init__()
        self._engine: Engine | None = None
        self._owns_engine = True
        self._device = 0
        self._max_batch = 16  # strict mode submits one frame per call; staging is sized by this
        self._scored_size: tuple[int, int] | None = None  # (width, height) detectors see
        self._base_index = 0  # engine frame index of this detector's first frame

    # -- configuration hooks used by SceneManager's batched fast path --
    def required_features(self, stats: bool = False) -> int:
        """PSD_F_* bits of the fused pass; `stats`: also what the per-frame metrics of a StatsManager need."""
        return self.FEATURES

    def edge_kernel_size_arg(self) -> int:
        return 0

    def engine_kwargs(self) -> dict:
        """Extra `Engine(...)` arguments this detector needs (e.g. the hash geometry)."""
        return {}

    def configure(self, device: int = 0, max_batch: int = 64,
                  scored_size: tuple[int, int] | None = None) -> None:
        """Select device / batch size / on-device downscale target before the first frame."""
        self._device = device
        self._max_batch = max_batch
        self._scored_size = scored_size

    def attach_engine(self, holder) -> None:
        """Share one fused pass between several detectors (SceneManager does this).  `holder` holds this
        detector's results: an Engine, a `SlotView` of one (`Engine.view`) or gathered results."""
        self._engine = holder
        self._owns_engine = False
        self._base_index = holder.frame_count

    def _ensure_engine(self, frames) -> Engine:
        if self._engine is None:
            h, w = frame_format(frames, self._device)[0][-3:-1]
            sw, sh = self._scored_size if self._scored_size else (w, h)
            self._engine = pixel_group_of(self).make_engine(w, h, sw, sh, device=self._device,
                                                            max_batch=self._max_batch)
            self._owns_engine = True
            self._base_index = 0
        return self._engine

    def _frames_device(self) -> int:
        """The CUDA device that device frames must be on: the engine's."""
        return getattr(self._engine, "device", self._device)

    @staticmethod
    def _as_batch(frame_img):
        """A numpy frame or batch as a batch; CUDA frames (any DLPack exporter) as they are: `Engine.submit` takes
        one frame or a batch."""
        if _dlpack.is_dlpack(frame_img):
            return frame_img
        if not isinstance(frame_img, np.ndarray):
            raise ValueError("frame_img must be a numpy.ndarray or a CUDA array that exports DLPack")
        return frame_img[None] if frame_img.ndim == 3 else frame_img

    # -- the two entry points --
    def process_frame(self, timecode, frame_img) -> list:
        return self.process_batch([timecode], self._as_batch(frame_img))

    def process_batch(self, timecodes, frames, first: int | None = None) -> list:
        """Score `frames` (N,H,W,3) and run this detector's per-frame logic over them.
        `first` = engine frame index of frames[0] when a shared engine already holds them
        (SceneManager submits once for all detectors); None = submit them here."""
        frames = self._as_batch(frames)
        self._validate(frames)
        engine = self._ensure_engine(frames)
        if first is None:
            if not self._owns_engine:
                raise RuntimeError("shared engine: frames must be submitted by its owner")
            engine.submit(frames)
            first = engine.frame_count - len(timecodes)
        return self._consume(list(timecodes), first)

    def consume_results(self, timecodes, first: int) -> list:
        """Run the per-frame logic over results the attached scan provider already holds
        (frames [first, first+len(timecodes)) ) - used by the multi-GPU gather path."""
        return self._consume(list(timecodes), first)

    def _validate(self, frames) -> None:
        pass

    def _consume(self, timecodes: list, first: int) -> list:  # pragma: no cover - abstract
        raise NotImplementedError

    def close(self) -> None:
        if self._engine is not None and self._owns_engine:
            self._engine.close()
        self._engine = None
