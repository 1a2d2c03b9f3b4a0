"""Image sequences decoded on the GPU: a `VideoStream`-shaped source (scenedetect/video_stream.py:79-222) over a list
of JPEG files or a `%0Nd` pattern, whose frames are what `cv2.imread(path)` gives, byte for byte, decoded by
psd_jpeg_decode into CUDA tensors.

A pattern resolves as the reference's `open_video(pattern)` does (cv2.VideoCapture, whose FFmpeg image2 demuxer
takes the first index from 0 to 4 that exists, then every consecutive index up to the first missing one).  The frames
differ from what that capture decodes, though: FFmpeg decodes JPEG with its own IDCT and colour conversion, while this
stream gives imread's frames (DESIGN.md §4.9)."""

from __future__ import annotations

import ctypes as C
import os
import re
from fractions import Fraction

import numpy as np

from . import _capi
from .compat import FrameTimecode, _to_fraction

_PATTERN = re.compile(r"%(0?\d*)d")
FIRST_INDEXES = 5   # FFmpeg image2 start_number_range: the first file is looked for at indexes 0 to 4


def resolve_pattern(pattern: str) -> list[str]:
    """The files a `%d` / `%0Nd` pattern names, as FFmpeg's image2 demuxer finds them: the first existing index in
    0..4, then consecutive indexes up to the first gap.  ValueError when none of 0..4 exists (the reference cannot open
    such a sequence either)."""
    if len(_PATTERN.findall(pattern)) != 1:
        raise ValueError(f"{pattern!r} is not an image sequence pattern with one %d or %0Nd")

    def path(i):
        return _PATTERN.sub(lambda m: ("%" + m.group(1) + "d") % i, pattern)

    first = next((i for i in range(FIRST_INDEXES) if os.path.isfile(path(i))), None)
    if first is None:
        raise ValueError(f"{pattern!r}: no file at index 0 to {FIRST_INDEXES - 1}")
    out, i = [], first
    while os.path.isfile(path(i)):
        out.append(path(i))
        i += 1
    return out


def probe(data) -> _capi.PsdJpegInfo:
    """psd_jpeg_probe of one file's bytes (host only)."""
    buf = np.frombuffer(data, np.uint8)
    info = _capi.PsdJpegInfo()
    _capi.check(_capi.load().psd_jpeg_probe(buf.ctypes.data, buf.size, C.byref(info)), "psd_jpeg_probe")
    return info


def check_file(data, where: str) -> _capi.PsdJpegInfo:
    """The file's psd_jpeg_info, or ValueError naming `where` and the reason the decoder refuses it."""
    info = probe(data)
    if info.refusal:
        raise ValueError(f"{where}: cannot decode this JPEG on the device: "
                         f"{_capi.JPEG_REFUSALS.get(info.refusal, info.refusal)}")
    return info


class DeviceDecoder:
    """psd_jpeg_decode into torch CUDA tensors on torch's current stream: the files of a batch in one page-locked
    buffer, one host-to-device copy, one decode call."""

    def __init__(self, device=None, workspace_cap: int = 0):
        import torch
        self._torch = torch
        self.workspace_cap = int(workspace_cap)   # bytes of decoder workspace per sub-batch (0: 512 MiB)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
        self._pinned = None
        self._dev = None

    def dlpack_device(self):
        return (2, self.device.index)

    def allocate(self, n, height, width):
        return self._torch.empty((n, height, width, 3), dtype=self._torch.uint8, device=self.device)

    def decode(self, datas, names, out, channel_order: str = "bgr"):
        """Decode the files `datas` (bytes) into `out`, an (n, H, W, 3) uint8 CUDA tensor of any strides (a
        `permute` of NCHW included), channels in `channel_order`."""
        torch = self._torch
        n = len(datas)
        if n == 0:
            return out
        for d, name in zip(datas, names):
            info = check_file(d, name)
            if (info.width, info.height) != (out.shape[2], out.shape[1]):
                raise ValueError(f"{name}: {info.width}x{info.height}, the other frames are "
                                 f"{out.shape[2]}x{out.shape[1]}")
        sizes = [len(d) for d in datas]
        offs = np.concatenate([[0], np.cumsum([(s + 15) // 16 * 16 for s in sizes])]).astype(np.int64)
        total = int(offs[-1])
        if self._pinned is None or self._pinned.numel() < total:
            self._pinned = torch.empty(total + total // 4, dtype=torch.uint8, pin_memory=True)
            self._dev = torch.empty(self._pinned.numel(), dtype=torch.uint8, device=self.device)
        host = self._pinned.numpy()
        for d, o in zip(datas, offs):
            host[o:o + len(d)] = np.frombuffer(d, np.uint8)
        self._dev[:total].copy_(self._pinned[:total], non_blocking=True)
        srcs = (_capi.PsdJpegSource * n)()
        imgs = (_capi.PsdJpegImage * n)()
        hp, dp = self._pinned.data_ptr(), self._dev.data_ptr()
        s = out.stride()
        for i in range(n):
            srcs[i].host, srcs[i].device, srcs[i].size = hp + int(offs[i]), dp + int(offs[i]), sizes[i]
            ch = -s[3] if channel_order == "rgb" else s[3]
            base = out[i, 0, 0, 2 if channel_order == "rgb" else 0].data_ptr()
            imgs[i].base = base
            imgs[i].layout = _capi.PsdFrameLayout(s[0], s[1], s[2], ch)
            imgs[i].width, imgs[i].height = out.shape[2], out.shape[1]
        flags = torch.empty(n, dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _capi.check(_capi.load().psd_jpeg_decode(self.device.index, srcs, n, imgs, self.workspace_cap, flags.data_ptr(), stream),
                    "psd_jpeg_decode")
        bad = np.nonzero(flags.cpu().numpy())[0]   # waits for the decode (and so for the copy out of _pinned)
        if len(bad):
            raise ValueError(f"{names[bad[0]]}: its entropy-coded data does not decode (corrupt JPEG)")
        return out


class ImageSequenceStream:
    """Seekable stream over JPEG files (a list of paths, or a `%0Nd` pattern), decoded on the GPU.

    `read` / `read_batch` return CUDA tensors (H, W, 3) / (n, H, W, 3) uint8 BGR, decoded on torch's current stream.
    Batches come from a pool of `pool` (at least three) buffers of `batch_size` frames used in turn, so a batch stays
    unchanged until two more have been read (SceneManager's FrameBatches contract).  Every file must have the first
    one's size.  `decoder` is what turns file bytes into frames (a DeviceDecoder by default)."""

    BACKEND_NAME = "image_sequence"

    def __init__(self, source, frame_rate=25.0, batch_size: int = 64, pool: int = 3, decoder=None):
        if isinstance(source, (str, os.PathLike)):
            source = os.fspath(source)
            self._paths = resolve_pattern(source) if _PATTERN.search(source) else [source]
            self._path = source
        else:
            self._paths = [os.fspath(p) for p in source]
            if not self._paths:
                raise ValueError("an image sequence needs at least one file")
            self._path = self._paths[0]
        if pool < 3:
            raise ValueError("pool must hold at least three batches")
        self._fps: Fraction = _to_fraction(frame_rate)
        self._batch = int(batch_size)
        self._decoder = decoder if decoder is not None else DeviceDecoder()
        with open(self._paths[0], "rb") as f:
            info = check_file(f.read(), self._paths[0])
        self._size = (int(info.width), int(info.height))
        self._pool = [None] * int(pool)
        self._slot = 0
        self._n = 0

    path = property(lambda self: self._path)
    paths = property(lambda self: list(self._paths))
    is_seekable = property(lambda self: True)
    frame_rate = property(lambda self: self._fps)
    frame_size = property(lambda self: self._size)
    aspect_ratio = property(lambda self: 1.0)
    frame_number = property(lambda self: self._n)
    channel_order = property(lambda self: "bgr")
    # how many batches `read` / `read_batch` hand out before one's memory is decoded into again: a reader that keeps
    # CUDA frames in flight (an engine not yet synchronised) must retire them before reading this many more
    batches_kept = property(lambda self: len(self._pool))

    @property
    def name(self) -> str:
        """The file name without its extension, cut at the `%` of a pattern (backends/opencv.py:178-186)."""
        name = os.path.splitext(os.path.basename(self._path))[0]
        return name[:name.rfind("%")] if "%" in name else name

    def __dlpack_device__(self):
        return self._decoder.dlpack_device()

    @property
    def base_timecode(self):
        return FrameTimecode(0, self._fps)

    @property
    def duration(self):
        return FrameTimecode(len(self._paths), self._fps)

    @property
    def position(self):
        return FrameTimecode(max(0, self._n - 1), self._fps)

    @property
    def position_ms(self) -> float:
        return 0.0 if self._n == 0 else 1000.0 * (self._n - 1) / float(self._fps)

    def _decode(self, first: int, k: int):
        slot = self._pool[self._slot]
        if slot is None:
            w, h = self._size
            slot = self._pool[self._slot] = self._decoder.allocate(self._batch, h, w)
        self._slot = (self._slot + 1) % len(self._pool)
        names = self._paths[first:first + k]
        datas = []
        for p in names:
            with open(p, "rb") as f:
                datas.append(f.read())
            info = check_file(datas[-1], p)
            if (info.width, info.height) != self._size:
                raise ValueError(f"{p}: {info.width}x{info.height}, the sequence's frames are "
                                 f"{self._size[0]}x{self._size[1]}")
        return self._decoder.decode(datas, names, slot[:k])

    def read(self, decode: bool = True):
        if self._n >= len(self._paths):
            return False
        if not decode:
            self._n += 1
            return True
        return self.read_batch(1)[0]

    def read_batch(self, max_frames: int):
        """Up to min(max_frames, batch_size) next frames, decoded into the next pool buffer (None at the end)."""
        if self._n >= len(self._paths):
            return None
        k = min(int(max_frames), self._batch, len(self._paths) - self._n)
        frames = self._decode(self._n, k)
        self._n += k
        return frames

    def reset(self):
        self._n = 0

    def seek(self, target):
        """Position the stream so that the next frame read is frame `target` (a frame number, a FrameTimecode or
        seconds as a float), clamped to the sequence."""
        if isinstance(target, FrameTimecode):
            frame = target.frame_num
        elif isinstance(target, float):
            frame = int(round(target * float(self._fps)))
        else:
            frame = int(target)
        if frame < 0:
            raise ValueError("seek target must be non-negative")
        self._n = min(frame, len(self._paths))
