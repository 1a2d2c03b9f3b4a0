"""Minimal in-memory `VideoStream`-shaped source (the reference's interface at
scenedetect/video_stream.py:79-222) for decoded BGR24 frames.  Video decoding itself is out
of scope (SURVEY.md §2 #9): the hot path starts at decoded frames."""

from __future__ import annotations

from fractions import Fraction

import numpy as np

from . import _dlpack
from .compat import FrameTimecode, _to_fraction


class ArrayVideoStream:
    """Forward-only stream over an (N,H,W,3) uint8 array: numpy (optionally page-locked), or CUDA memory of any
    DLPack exporter, strided views such as `nchw.permute(0, 2, 3, 1)` included.  `channel_order` "rgb": the last
    axis is R, G, B.  `read` / `read_batch` return views of `frames`: for numpy, in BGR order; for CUDA frames, in
    `channel_order` (the `channel_order` property), which SceneManager passes on to the engine."""

    BACKEND_NAME = "array"

    def __init__(self, frames, fps=30.0, pinned: bool = False, repeat: int = 1, channel_order: str = "bgr"):
        if channel_order not in ("bgr", "rgb"):
            raise ValueError(f"channel_order must be 'bgr' or 'rgb', not {channel_order!r}")
        if _dlpack.is_dlpack(frames):
            if not _dlpack.on_cuda(frames):
                raise ValueError("DLPack frames must be in CUDA memory (host frames are numpy arrays)")
            shape, uint8 = _dlpack.frame_format(frames)
        else:
            shape, uint8 = frames.shape, frames.dtype == np.uint8
            if channel_order == "rgb":
                frames, channel_order = frames[..., ::-1], "bgr"
        if not uint8 or len(shape) != 4 or shape[3] != 3:
            raise ValueError("frames must be (N,H,W,3) uint8")
        self._frames = frames
        self._shape = tuple(int(d) for d in shape)   # (N, H, W, 3), read from the DLPack view for CUDA frames
        self._channel_order = channel_order
        self._fps: Fraction = _to_fraction(fps)
        self._pinned = pinned
        self._total = self._shape[0] * int(repeat)
        self._n = 0

    path = property(lambda self: "array")
    name = property(lambda self: "array")
    is_seekable = property(lambda self: False)
    frame_rate = property(lambda self: self._fps)
    frame_size = property(lambda self: (self._shape[2], self._shape[1]))
    aspect_ratio = property(lambda self: 1.0)
    frame_number = property(lambda self: self._n)
    is_pinned = property(lambda self: self._pinned)
    channel_order = property(lambda self: self._channel_order)

    def __dlpack_device__(self):
        """The DLPack device of the frames (SceneManager reads CUDA streams as views, never through the host)."""
        return self._frames.__dlpack_device__()

    @property
    def base_timecode(self):
        return FrameTimecode(0, self._fps)

    @property
    def duration(self):
        return FrameTimecode(self._total, self._fps)

    @property
    def position(self):
        return FrameTimecode(max(0, self._n - 1), self._fps)

    @property
    def position_ms(self) -> float:
        return 0.0 if self._n == 0 else 1000.0 * (self._n - 1) / float(self._fps)

    def read(self, decode: bool = True):
        if self._n >= self._total:
            return False
        frame = self._frames[self._n % self._shape[0]]
        self._n += 1
        return frame if decode else True

    def read_batch(self, max_frames: int):
        """Zero-copy view of up to `max_frames` consecutive frames (None at EOF)."""
        if self._n >= self._total:
            return None
        base = self._shape[0]
        i = self._n % base
        k = min(max_frames, self._total - self._n, base - i)
        self._n += k
        return self._frames[i:i + k]

    def reset(self):
        self._n = 0

    def seek(self, target):
        raise NotImplementedError("ArrayVideoStream is forward-only")
