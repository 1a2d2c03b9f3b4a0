"""Scene detection over many clips in one pass: one engine stream per group of clips, one automaton launch for all
their cuts.

Dataset-curation pipelines split millions of short clips, and the reference's benchmark harness loops `detect()`
once per video (benchmark/__main__.py:44-61).  One `SceneManager.detect_scenes` per clip pays a fixed cost per clip:
a new engine (device allocations, result arrays that grow through synchronising reallocations), per-frame Python
state machines, and a device teardown.  `detect_clips` instead:

* groups the clips by (frame size, host or CUDA, channel order) and builds one engine per group through
  `shared_engine`, with every detector's edge and hash slots, exactly as SceneManager does for one video;
* scores a group's clips back to back into that engine.  The fused pass scores a frame from that frame and its
  predecessor only, so every integer result is the clip's own except at the clip edges;
* finishes a pass with one psd_scan_* per distinct metric array, each followed by psd_clip_fill, which gives every
  clip's edge entries what a one-clip engine's scan writes there (`device_cuts.scan_metric` with a clip table),
  then ONE psd_clip_cuts for every (detector, clip) automaton and one download of the compact cut lists.

Host frames are copied into page-locked batches that run across clip boundaries, so the number of fused-pass
launches follows the total frame count, not the clip count.  CUDA frames are submitted as views of each clip's
stream, as SceneManager reads them: at least one submission per clip.

A pass is finished, and the engine reset, once it holds `MAX_PASS_FRAMES` frames, at the next clip boundary; so the
per-frame result memory does not grow with the number of clips (a single longer clip is held whole).

Results are those of a fresh `SceneManager(batch_size=...)` with the same `auto_downscale` / `downscale` and fresh
detectors, running `detect_scenes` on each clip: cut list, scene lists and frame count.  Frame numbers are
clip-local, frame-number timecodes at the clip's constant frame rate (as `DeviceCuts` gives them).
"""

from __future__ import annotations

from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from . import _capi, _dlpack
from ._capi import check
from .compat import FrameTimecode
from .detectors._base import EngineDetector, pixel_group_of
from .device_cuts import scan_metric
from .engine import DeviceBuffer
from .scene_manager import FrameBatches, SceneManager, get_scenes_from_cuts, shared_engine
from .sweep import _KIND, plan_cell

MAX_PASS_FRAMES = 1 << 16     # frames an engine holds before its pass is finished at the next clip boundary
FIRST_CUTS_PER_FRAME = 0.25   # first cut buffer of a pass, in cuts per frame held; grown once if the cuts need more


@dataclass
class ClipResult:
    """One clip's detection: what `SceneManager.get_cut_list` / `get_scene_list` / `detect_scenes` give."""

    fps: Fraction
    frames: int = 0                           # what detect_scenes returns: frames read from the stream
    cut_frames: list = field(default_factory=list)  # sorted unique cut frame numbers
    start: FrameTimecode | None = None       # position of the first frame scored (None: the clip had no frames)
    end: FrameTimecode | None = None         # the stream's position after the last frame

    def cut_list(self) -> list:
        return [FrameTimecode(c, self.fps) for c in self.cut_frames]

    def scene_list(self, start_in_scene: bool = False) -> list:
        if self.start is None:
            return []
        cuts = self.cut_list()
        if not cuts and not start_in_scene:
            return []
        return sorted(get_scenes_from_cuts(cuts, self.start, self.end + 1))


class _ClipChain:
    """A group's streams read one after the other as one stream, for `FrameBatches`: `read()` moves on to the next
    clip when one ends, and records each clip's positions and frame count.  At a clip boundary, once the pass holds
    `bound` frames, it reports an end (`paused`) until `resume()`."""

    def __init__(self, clips, bound: int, on_cuda: bool):
        self._clips = clips       # [(input index, stream)]
        self._k = -1
        self._on_cuda = on_cuda
        self.bound = bound
        self.paused = False
        self.held = 0             # frames read in this pass
        self.done = []            # (input index, ClipResult, frames scored) of every clip finished in this pass
        self._result = None
        self._start_num = self._scored = 0
        self._next()

    frame_number = property(lambda self: self.held)   # FrameBatches only reads positions relative to its start
    frame_rate = property(lambda self: self._result.fps if self._result else Fraction(30))

    @property
    def position(self):
        return self._clips[self._k][1].position if self._k < len(self._clips) else None

    def _next(self):
        self._k += 1
        if self._k < len(self._clips):
            video = self._clips[self._k][1]
            self._start_num = video.frame_number
            self._result = ClipResult(fps=video.frame_rate)
            self._scored = 0

    def _end_clip(self) -> None:
        """Close the current clip; pause if the pass holds enough frames and another clip follows."""
        index, video = self._clips[self._k]
        r = self._result
        r.frames = video.frame_number - self._start_num
        if r.start is not None:
            r.end = video.position
        self.done.append((index, r, self._scored))
        self._next()
        if self.held >= self.bound and self._k < len(self._clips):
            self.paused = True

    def _took(self, n: int, first_pos) -> None:
        if self._result.start is None:
            self._result.start = first_pos
        self._scored += n
        self.held += n

    def read(self, decode: bool = True):
        while not self.paused and self._k < len(self._clips):
            video = self._clips[self._k][1]
            frame = video.read()
            if frame is not False:
                if _dlpack.is_dlpack(frame) != self._on_cuda:
                    raise ValueError("a stream's frames are not where its group's are (host or CUDA)")
                self._took(1, video.position)
                return frame
            self._end_clip()
        return False

    def resume(self) -> None:
        self.paused = False
        self.held = 0
        self.done = []


class _DeviceClipChain(_ClipChain):
    """The chain over CUDA streams with `read_batch`: views of one clip at a time, as SceneManager reads them."""

    def __dlpack_device__(self):
        return self._clips[min(self._k, len(self._clips) - 1)][1].__dlpack_device__()

    def read_batch(self, max_frames: int):
        while not self.paused and self._k < len(self._clips):
            video = self._clips[self._k][1]
            pos0 = video.frame_number
            chunk = video.read_batch(max_frames)
            if chunk is not None:
                self._took(int(chunk.shape[0]), FrameTimecode(pos0, video.frame_rate))
                return chunk
            self._end_clip()
        return None


class _Pass:
    """The device half of a `detect_clips` call: the detectors' cells and metric keys, the metric arrays, clip table
    and cut buffers (reused pass after pass and group after group; they only grow), and the step that turns an
    engine's pass into every clip's cut list."""

    def __init__(self, detectors, device: int):
        self._lib = _capi.load()
        self.device = device
        self.groups, gi = [], {}
        self.cells = []
        for d in detectors:
            g = pixel_group_of(d)
            if g not in gi:
                gi[g] = len(self.groups)
                self.groups.append(g)
            self.cells.append(plan_cell(d, gi[g]))
        self.keys = []  # metric keys in order of first use: content_val before the adaptive ratio that reads it
        for c in self.cells:
            for key in (c.metric2, c.metric):
                if key is not None and key not in self.keys:
                    self.keys.append(key)
        self._bufs = {}

    def _buf(self, name, nbytes: int) -> DeviceBuffer:
        b = self._bufs.get(name)
        if b is None or b.nbytes < nbytes:
            if b is not None:
                b.close()
            b = self._bufs[name] = DeviceBuffer(max(8, int(nbytes)), self.device)
        return b

    def close(self) -> None:
        for b in self._bufs.values():
            b.close()
        self._bufs = {}

    def finish(self, engine, holders, clips: list) -> None:
        """Every clip of `clips` ((ClipResult, frames scored) of the frames `engine` holds, in order) gets its cut
        frames."""
        lib = self._lib
        scored = [r for r, m in clips if m]
        n = engine.frame_count
        if not scored:
            return
        c, k = len(scored), len(self.cells)
        sizes = np.array([m for _, m in clips if m], dtype=np.int64)
        if int(sizes.sum()) != n:
            raise RuntimeError(f"the engine holds {n} frames, the clips {int(sizes.sum())}")
        table = np.concatenate([
            np.concatenate([[0], np.cumsum(sizes)]),
            [r.start.frame_num for r in scored],
            [cell.min_frames(r.fps) for cell in self.cells for r in scored]]).astype(np.int64)
        tbuf = self._buf("table", table.nbytes)
        tbuf.upload(table)
        offsets, first, min_frames = tbuf.ptr, tbuf.ptr + (c + 1) * 8, tbuf.ptr + (2 * c + 1) * 8
        arrays = {key: self._buf(key, n * 8) for key in self.keys}
        for key in self.keys:
            val = arrays[("content_val",) + key[1:3]].ptr if key[0] == "adaptive_ratio" else None
            scan_metric(lib, holders[key[1]], (key[0],) + key[2:], arrays[key].ptr, val, clips=(offsets, c))
        cells = (_capi.PsdSweepCell * k)()
        for i, cell in enumerate(self.cells):
            cells[i] = _capi.PsdSweepCell(
                kind=_KIND[cell.kind], mode=cell.mode, metric=arrays[cell.metric].ptr,
                metric2=arrays[cell.metric2].ptr if cell.metric2 is not None else None, threshold=cell.threshold,
                min_content_val=cell.min_content_val, fade_bias=cell.fade_bias, min_frames=0, window=cell.window,
                add_final_scene=cell.add_final_scene)
        obuf = self._buf("cut_offsets", (k * c + 1) * 8)
        cap = max(1, int(n * FIRST_CUTS_PER_FRAME)) if FIRST_CUTS_PER_FRAME > 0 else 0
        cuts = self._buf("cuts", cap * 8)
        cap = cuts.nbytes // 8
        st = engine.compute_stream
        for attempt in range(2):
            check(lib.psd_clip_cuts(cells, k, offsets, first, c, min_frames, cuts.ptr, cap, obuf.ptr, st),
                  "psd_clip_cuts")
            engine.sync()
            offs = obuf.download((k * c + 1) * 8).view(np.int64)
            total = int(offs[-1])
            if total <= cap:
                break
            if attempt:
                raise RuntimeError(f"psd_clip_cuts needs {total} cuts after growing its buffer to {cap}")
            cuts = self._buf("cuts", total * 8)
            cap = cuts.nbytes // 8
        got = cuts.download(total * 8).view(np.int64).tolist() if total else []
        offs = offs.tolist()
        for j, r in enumerate(scored):  # (cell i, clip j) is list i * c + j: SceneManager.get_cut_list per clip
            r.cut_frames = sorted({f for i in range(k) for f in got[offs[i * c + j]:offs[i * c + j + 1]]})


def _group_key(video) -> tuple:
    """(frame size, CUDA frames, read as views of `read_batch`, channel order of the CUDA frames)"""
    on_cuda = _dlpack.on_cuda(video)
    return (tuple(video.frame_size), on_cuda, on_cuda and hasattr(video, "read_batch"),
            getattr(video, "channel_order", "bgr") if on_cuda else "bgr")


def detect_clips(videos, detectors, auto_downscale: bool = True, downscale: int = 1, device: int = 0,
                 batch_size: int = 64) -> list[ClipResult]:
    """Detect scenes in every stream of `videos` with every detector of `detectors`: for each clip, in input order,
    what a fresh `SceneManager(device=device, batch_size=batch_size)` with these `auto_downscale` / `downscale` and
    fresh copies of the detectors give from `detect_scenes(video)`.  Streams are anything `detect_scenes` reads
    (`ArrayVideoStream` over numpy or CUDA arrays of any layout and channel order, a reference `VideoStream`) and may
    differ in length, frame rate and frame size; a stream is read from its current position to its end.

    The detectors are configuration only: they are not attached to an engine or otherwise changed.  ValueError for
    an empty detector list or a detector with a `stats_manager` (this path produces no per-frame metric rows)."""
    detectors = list(detectors)
    if not detectors:
        raise ValueError("No detectors added")
    for d in detectors:
        if not isinstance(d, EngineDetector):
            raise TypeError("detect_clips drives the GPU detectors of this package")
        if d.stats_manager is not None:
            raise ValueError("detect_clips produces no per-frame metrics: detectors must not have a stats_manager")
    if downscale < 1:
        raise ValueError("Downscale factor must be a positive integer >= 1!")
    geometry = SceneManager(device=device, batch_size=batch_size)
    geometry._auto_downscale, geometry._downscale = bool(auto_downscale), int(downscale)
    videos = list(videos)
    groups: dict = {}
    for i, v in enumerate(videos):
        groups.setdefault(_group_key(v), []).append((i, v))
    results: list = [None] * len(videos)
    device_pass = _Pass(detectors, device)
    try:
        for (size, on_cuda, views, order), clips in groups.items():
            box, (w, h), (sw, sh) = geometry._geometry(*size)
            engine, holders = shared_engine(device_pass.groups, w, h, sw, sh, device=device, max_batch=batch_size)
            chain = (_DeviceClipChain if views else _ClipChain)(clips, MAX_PASS_FRAMES, on_cuda)
            gather = FrameBatches(chain, box, (w, h), batch_size)
            try:
                while True:
                    item = gather.next()  # overlaps the GPU's work on the previous batch
                    engine.sync()         # retire the previous batch before its buffer is reused
                    if item is None:
                        device_pass.finish(engine, holders, [(r, m) for _, r, m in chain.done])
                        for index, r, _ in chain.done:
                            results[index] = r
                        if not chain.paused:
                            break
                        engine.reset()
                        chain.resume()
                        gather.resume()
                        continue
                    _tcs, frames, pinned = item
                    if isinstance(frames, np.ndarray):
                        engine.submit(frames, pinned=pinned)
                    else:  # CUDA frames: a view of one clip, or a list of frames from streams without read_batch
                        for f in (frames if isinstance(frames, list) else [frames]):
                            engine.submit(f, channel_order=order)
            finally:
                gather.close()
                engine.close()
    finally:
        device_pass.close()
    return results


__all__ = ["detect_clips", "ClipResult", "MAX_PASS_FRAMES"]
