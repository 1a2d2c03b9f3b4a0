"""Shared machinery of the drop-in detectors: lazy engine creation, strict (one frame per
call, as SceneManager drives it: scene_manager.py:426-428) and batched submission."""

from __future__ import annotations

import numpy as np

from ..compat import SceneDetector
from ..engine import Engine


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
        self._edge_slot = 0   # the engine's slots of this detector's kernel size / hash geometry (attach_engine)
        self._hash_slot = 0

    # -- configuration hooks used by SceneManager's batched fast path --
    def required_features(self) -> int:
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

    def attach_engine(self, engine: Engine, edge_slot: int = 0, hash_slot: int = 0) -> None:
        """Share one fused pass between several detectors (SceneManager does this).  `edge_slot` / `hash_slot`:
        the engine's slot that holds this detector's dilation kernel size / hash geometry."""
        self._edge_slot, self._hash_slot = int(edge_slot), int(hash_slot)
        self._engine = engine.view(edge_slot, hash_slot) if (edge_slot or hash_slot) else engine
        self._owns_engine = False
        self._base_index = engine.frame_count

    def _ensure_engine(self, frames: np.ndarray) -> Engine:
        if self._engine is None:
            h, w = frames.shape[-3], frames.shape[-2]
            sw, sh = self._scored_size if self._scored_size else (w, h)
            self._engine = Engine(w, h, self.required_features(), width=sw, height=sh,
                                  device=self._device, max_batch=self._max_batch,
                                  edge_kernel_size=self.edge_kernel_size_arg(), **self.engine_kwargs())
            self._owns_engine = True
            self._base_index = 0
            self._edge_slot = self._hash_slot = 0
        return self._engine

    @staticmethod
    def _as_batch(frame_img) -> np.ndarray:
        if not isinstance(frame_img, np.ndarray):
            raise ValueError("frame_img must be a numpy.ndarray")
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

    def _validate(self, frames: np.ndarray) -> None:
        pass

    def _consume(self, timecodes: list, first: int) -> list:  # pragma: no cover - abstract
        raise NotImplementedError

    def close(self) -> None:
        if self._engine is not None and self._owns_engine:
            self._engine.close()
        self._engine = None
