"""Batched counterpart of the reference `SceneManager` for the detectors in this package.

Mirrors the part of scenedetect/scene_manager.py that is on (or immediately around) the hot
path: `add_detector`, `detect_scenes`, `get_scene_list` / cut list, `auto_downscale` /
`downscale` / `crop`, StatsManager injection.  Differences by design:

* the reference hands one frame at a time to `detector.process_frame`
  (scene_manager.py:410-435); here frames are gathered into batches of `batch_size`, pushed
  through ONE fused GPU pass shared by all attached detectors, and each detector then runs
  its per-frame state machine over the device-computed metrics.  Cuts can therefore be
  emitted up to one batch late, which the reference's contract allows (cuts are sorted and
  de-duplicated at scene_manager.py:403-408; `post_process` is the final flush, :621);
* the `cv2.resize` downscale of the decode thread (scene_manager.py:670-678) runs on the
  device (exact fixed-point restatement) instead of on the host.

The resulting cut list and scene list are identical to the reference's, and so is every integer-derived
column of the StatsManager CSV (`content_val`, `delta_*`, `average_rgb`, `adaptive_ratio`); `hist_diff`
agrees to 1e-9 (cv2.compareHist's SIMD summation order is not reproduced; BASELINE tolerance 1e-4).
"""

from __future__ import annotations

import logging

import numpy as np

from . import _dlpack
from .compat import FrameTimecode, StatsManager
from .detectors._base import EngineDetector, pixel_group_of
from ._capi import F_EDGES, F_HASH
from .engine import DeviceBuffer, Engine, PinnedBuffer, download_bgr

DEFAULT_MIN_WIDTH = 256
logger = logging.getLogger("pyscenedetect_b200")


def compute_downscale_factor(frame_width: int, effective_width: int = DEFAULT_MIN_WIDTH) -> float:
    """scene_manager.py:123-140."""
    assert frame_width > 0 and effective_width > 0
    if frame_width < effective_width:
        return 1
    return frame_width / float(effective_width)


def get_scenes_from_cuts(cut_list, start_pos, end_pos):
    """scene_manager.py:171-210: contiguous (start, end) pairs from a sorted cut list."""
    scene_list = []
    if not cut_list:
        scene_list.append((start_pos, end_pos))
        return scene_list
    last_cut = start_pos
    for cut in cut_list:
        scene_list.append((last_cut, cut))
        last_cut = cut
    scene_list.append((last_cut, end_pos))
    return scene_list


def shared_engine(groups, src_width: int, src_height: int, width: int, height: int, device: int = 0,
                  max_batch: int = 64):
    """One Engine for several `PixelGroup`s: the union of their features, the first edge user's kernel size and
    the first hash user's geometry in the configuration, and every other distinct effective kernel size and
    geometry as a further slot, in order of appearance (the engine deduplicates).  -> (engine, one result holder
    per group: `engine.view` of the group's slots); a group that does not use the edge component or the hash
    reads slot 0 for it."""
    features = 0
    for g in groups:
        features |= g.features
    k0 = next((g.edge_kernel_size for g in groups if g.features & F_EDGES), 0)
    geo0 = next((dict(g.engine_kwargs) for g in groups if g.features & F_HASH), {})
    engine = Engine(src_width, src_height, features, width=width, height=height, device=device, max_batch=max_batch,
                    edge_kernel_size=k0, **geo0)
    holders = []
    for g in groups:
        # the configured kernel size argument and geometry are slot 0 without asking, so a scorer with one slot of
        # each (tests/fake_engine.py) needs no slot calls for a mix that has nothing else
        kw = dict(g.engine_kwargs)
        edge_slot = (engine.add_edge_kernel_size(g.edge_kernel_size)
                     if g.features & F_EDGES and g.edge_kernel_size != k0 else 0)
        hash_slot = (engine.add_hash_geometry(kw["hash_size"], kw["hash_lowpass"])
                     if g.features & F_HASH and kw != geo0 else 0)
        holders.append(engine.view(edge_slot, hash_slot) if edge_slot or hash_slot else engine)
    return engine, holders


def check_window(duration=None, end_time=None, frame_skip: int = 0, stats: bool = False) -> None:
    """The argument checks of detect_scenes (scene_manager.py:500-515)."""
    if frame_skip > 0 and stats:
        raise ValueError("frame_skip must be 0 when using a StatsManager.")
    if duration is not None and end_time is not None:
        raise ValueError("duration and end_time cannot be set at the same time!")
    if duration is not None and isinstance(duration, (int, float)) and duration < 0:
        raise ValueError("duration must be greater than or equal to 0!")
    if end_time is not None and isinstance(end_time, (int, float)) and end_time < 0:
        raise ValueError("end_time must be greater than or equal to 0!")


def base_timecode_of(video) -> FrameTimecode:
    """The stream's base timecode, or frame 0 at its rate."""
    base = getattr(video, "base_timecode", None)
    return base if base is not None else FrameTimecode(0, video.frame_rate)


def window_end_frame(base, start_frame: int, duration=None, end_time=None) -> int | None:
    """scene_manager.py:543-547: end_time is absolute, duration is relative to the position the loop starts at
    (`start_frame`); frames with position + 1 >= the result are the last ones processed (scene_manager.py:686-689).
    None: read to the end."""
    if end_time is not None:
        return (base + end_time).frame_num
    if duration is not None:
        return ((base + duration) + start_frame).frame_num
    return None


class StreamWindow:
    """Which frames of one stream the detection loop processes (scene_manager.py:650-689), from the stream's position
    when the window is made: every (frame_skip + 1)-th frame, each followed by the frame_skip frames it skips (read,
    not decoded), until a processed frame leaves the position + 1 >= `end_frame`; the first frame is processed in
    any case.  `read()` for a stream read frame by frame, `read_views()` for a stream read with `read_batch`; a window
    is read one way only."""

    def __init__(self, video, frame_skip: int = 0, end_frame: int | None = None):
        self.video = video
        self.step = int(frame_skip) + 1
        self.end_frame = end_frame
        self.start = video.frame_number
        self.processed = 0
        self.done = False
        self.position = None  # read(): the position of the last frame processed

    @staticmethod
    def frames_read(step: int, start: int, end_frame: int | None) -> int | None:
        """How many frames a window of `step` made at frame number `start` reads, if the stream does not end first:
        frames start + i * step for every i with that frame < end_frame (and i = 0 in any case) are processed, each
        followed by its step - 1 skipped reads.  None without an end frame: the window reads to the end."""
        if end_frame is None:
            return None
        return step * max(1, -(-(end_frame - start) // step))

    def read(self):
        """The next frame to process, after which the frames it skips are read; False at the end."""
        if self.done:
            return False
        video = self.video
        frame = video.read()
        if frame is False:
            self.done = True
            return False
        self.position = video.position
        self.processed += 1
        for _ in range(self.step - 1):  # scene_manager.py:682-685
            if not video.read(decode=False):
                break
        if self.end_frame is not None and not (video.position.frame_num + 1) < self.end_frame:
            self.done = True
        return frame

    def read_views(self, max_frames: int):
        """Up to `max_frames` frames to process from one `read_batch`, with the frames each skips (and those still to
        skip after the previous call's last one): (frame number of the first, count, view `chunk[skip::step]`), or
        None at the end."""
        video, end_frame, step = self.video, self.end_frame, self.step
        while not self.done:
            pos = video.frame_number
            skip = (self.start - pos) % step   # frames still to skip after the last processed one
            count = max_frames
            if end_frame is not None:
                count = min(count, max(-(-(end_frame - pos - skip) // step), 1 if self.processed == 0 else 0))
            want = skip + count * step
            chunk = video.read_batch(want) if want > 0 else None
            if chunk is None:
                self.done = True
                return None
            k = len(range(skip, chunk.shape[0], step))
            if k == 0:
                continue
            self.processed += k
            return pos + skip, k, (chunk if step == 1 else chunk[skip::step])
        return None


class FrameBatches:
    """The frame-gathering half of the detection loop (scene_manager.py:650-689): reads `video` in batches of
    up to `batch_size` frames, cropped to `box` = (x0, y0, x1, y1) of size `size` = (w, h), through a `StreamWindow`.
    `box` may instead be a function that gives the box of the frames `video` has just returned (clips.py's chain of
    clips, each with its own crop to the same size).
    A stream with `read_batch` and no crop / frame skip is read zero-copy; otherwise frames are copied into one of two
    page-locked buffers, so that a batch can be gathered while the GPU scores the previous one.

    Frames on the GPU (the stream's or the frames' `__dlpack_device__` says CUDA) never go through the host.  A
    stream with `read_batch` yields views `[o::frame_skip + 1, y0:y1, x0:x1]` of what it returns; a stream with
    only `read` yields a list of cropped frame views, which the engine takes one at a time.  Either way the frames,
    their positions and the frames read past the last one are those of the host path.  Unlike host frames, CUDA
    frames are not copied as they are read: what `read` / `read_batch` return must stay unchanged until the batch
    after the one it belongs to has been scored (a decoder that recycles its output surfaces needs a pool of more
    than two batches, or must return copies).

    `next()` returns (timecodes, frames, pinned) or None at the end.  The frames of a batch stay valid until
    the batch after the next one is gathered: the caller must have synchronised the engines that read a batch
    before asking for the batch two after it.  `close()` frees the buffers, after the last batch is done."""

    def __init__(self, video, box, size, batch_size: int, cropped: bool = False, frame_skip: int = 0,
                 end_frame: int | None = None):
        self._video = video
        self._box, self._size = (box if callable(box) else lambda: box), size
        self._batch_size = int(batch_size)
        self._window = StreamWindow(video, frame_skip, end_frame)
        self._device_views = hasattr(video, "read_batch") and _dlpack.on_cuda(video)
        self._zero_copy = hasattr(video, "read_batch") and not cropped and frame_skip == 0 and not self._device_views
        self._pinned = [None, None]
        self._which = 0
        self._done = False

    def _next_views(self):
        """The next batch of a stream read with `read_batch`: CUDA views, or a zero-copy host view."""
        got = self._window.read_views(self._batch_size)
        if got is None:
            self._done = True
            return None
        first, k, chunk = got
        fps, step = self._video.frame_rate, self._window.step
        tcs = [FrameTimecode(first + j * step, fps) for j in range(k)]
        if self._zero_copy:
            return tcs, chunk, bool(getattr(self._video, "is_pinned", False))
        x0, y0, x1, y1 = self._box()
        return tcs, chunk[:, y0:y1, x0:x1], False

    def next(self):
        if self._done:
            return None
        if self._device_views or self._zero_copy:
            return self._next_views()
        window = self._window
        w, h = self._size
        tcs, batch = [], None
        which = self._which
        buf, views = None, []
        k = 0
        while k < self._batch_size:
            frame = window.read()
            if frame is False:
                self._done = True
                break
            x0, y0, x1, y1 = self._box()
            if _dlpack.is_dlpack(frame):
                views.append(frame[y0:y1, x0:x1])
            else:
                if buf is None:
                    if self._pinned[which] is None:
                        self._pinned[which] = PinnedBuffer(self._batch_size * w * h * 3)
                    buf = self._pinned[which].array.reshape(self._batch_size, h, w, 3)
                np.copyto(buf[k], frame[y0:y1, x0:x1])
            tcs.append(window.position)
            k += 1
            if window.done:
                self._done = True
                break
        batch = (views if buf is None else buf[:k]) if k else None
        if batch is None:
            self._done = True
            return None
        self._which ^= 1
        return tcs, batch, True

    def resume(self) -> None:
        """Read on after `next()` returned None, from a stream that reports an end and can then be read past it
        (clips.py's chain of clips pauses at a clip boundary so that the engine can be emptied).  The buffers are
        kept: the caller has synchronised every engine that read them."""
        self._done = False
        self._window.done = False

    def close(self) -> None:
        for p in self._pinned:
            if p is not None:
                p.close()
        self._pinned = [None, None]


class SceneManager:
    def __init__(self, stats_manager: StatsManager | None = None, device: int = 0,
                 batch_size: int = 64):
        self._detector_list: list[EngineDetector] = []
        self._cutting_list: list = []
        self._stats_manager = stats_manager
        self._device = device
        self._batch_size = int(batch_size)
        self._auto_downscale = True
        self._downscale = 1
        self._crop = None
        self._start_pos = None
        self._last_pos = None
        self._base_timecode = None
        self._engine: Engine | None = None
        self._frame_size = None
        self._frame_buffer_size = 0          # max event_buffer_length of the detectors (scene_manager.py:352)
        self._frame_tail: list = []          # last `_frame_buffer_size` (timecode, frame copy) pairs of the previous batch
        self._channel_order = "bgr"          # of the frames the stream returns
        self._scratch: DeviceBuffer | None = None  # one cropped frame: CUDA frames copied out for callbacks

    # -- configuration (scene_manager.py:254-335) --
    @property
    def stats_manager(self):
        return self._stats_manager

    @property
    def auto_downscale(self) -> bool:
        return self._auto_downscale

    @auto_downscale.setter
    def auto_downscale(self, value: bool):
        self._auto_downscale = value

    @property
    def downscale(self) -> int:
        return self._downscale

    @downscale.setter
    def downscale(self, value: int):
        """scene_manager.py:313-325: the factor is IGNORED while auto_downscale is True."""
        if value < 1:
            raise ValueError("Downscale factor must be a positive integer >= 1!")
        if self.auto_downscale:
            logger.warning("Downscale factor will be ignored because auto_downscale=True!")
        if not isinstance(value, int):
            logger.warning("Downscale factor will be truncated to integer!")
            value = int(value)
        self._downscale = value

    @property
    def crop(self):
        """(X0, Y0, X1, Y1), inclusive coordinates (scene_manager.py:279-291)."""
        if self._crop is None:
            return None
        x0, y0, x1, y1 = self._crop
        return (x0, y0, x1 - 1, y1 - 1)

    @crop.setter
    def crop(self, value):
        """scene_manager.py:293-306: any two corners, inclusive; stored one-past-the-end."""
        if value is None:
            self._crop = None
            return
        if not (len(value) == 4 and all(isinstance(v, int) for v in value)):
            raise TypeError("crop region must be tuple of 4 ints")
        if any(v < 0 for v in value):
            raise ValueError("crop coordinates must be >= 0")
        x0, y0, x1, y1 = value
        self._crop = (min(x0, x1), min(y0, y1), max(x0, x1) + 1, max(y0, y1) + 1)

    def add_detector(self, detector: EngineDetector) -> None:
        """scene_manager.py:337-352."""
        if not isinstance(detector, EngineDetector):
            raise TypeError("pyscenedetect_b200.SceneManager drives the GPU detectors of this "
                            "package; use the reference SceneManager for CPU detectors")
        detector.stats_manager = self._stats_manager
        if self._stats_manager is not None:
            self._stats_manager.register_metrics(detector.get_metrics())
        self._detector_list.append(detector)
        self._frame_buffer_size = max(detector.event_buffer_length, self._frame_buffer_size)

    def clear(self) -> None:
        self._cutting_list.clear()
        self._last_pos = None
        self._start_pos = None

    # -- results (scene_manager.py:376-408) --
    def get_cut_list(self) -> list:
        if not self._cutting_list:
            return []
        return sorted(set(self._cutting_list))

    def get_scene_list(self, start_in_scene: bool = False) -> list:
        if self._base_timecode is None or self._last_pos is None:
            return []  # nothing processed yet / empty stream
        cut_list = self.get_cut_list()
        scene_list = get_scenes_from_cuts(cut_list, self._start_pos, self._last_pos + 1)
        if not cut_list and not start_in_scene:
            scene_list = []
        return sorted(scene_list)

    # -- the loop (scene_manager.py:446-623) --
    def _geometry(self, fw: int, fh: int):
        """Crop rectangle, effective size and scored size exactly as scene_manager.py:505-535,657-678:
        the downscale factor comes from the "effective" size (1 + clipped end - start, with the end already
        stored one past: one more than the cropped frame really has), the resize target from the cropped
        frame itself."""
        x0, y0, x1, y1 = (0, 0, fw, fh)
        eff = (fw, fh)
        if self._crop is not None:
            cx0, cy0, cx1, cy1 = self._crop
            if cx0 >= fw or cy0 >= fh:
                raise ValueError("crop starts outside video boundary")
            if cx1 >= fw or cy1 >= fh:
                logger.warning("Warning: crop ends outside of video boundary.")
            eff = (1 + min(cx1, fw) - cx0, 1 + min(cy1, fh) - cy0)
            x0, y0, x1, y1 = cx0, cy0, min(cx1, fw), min(cy1, fh)  # numpy slicing clips the same way
        w, h = x1 - x0, y1 - y0
        factor = compute_downscale_factor(max(eff)) if self._auto_downscale else self._downscale
        if factor > 1.0:
            sw, sh = max(1, round(w / factor)), max(1, round(h / factor))
        else:
            sw, sh = w, h
        return (x0, y0, x1, y1), (w, h), (sw, sh)

    def detect_scenes(self, video, duration=None, end_time=None, frame_skip: int = 0,
                      show_progress: bool = False, callback=None) -> int:
        if not self._detector_list:
            raise ValueError("No detectors added")
        check_window(duration, end_time, frame_skip, self._stats_manager is not None)
        self.clear()
        self._frame_tail = []
        fw, fh = video.frame_size
        (x0, y0, x1, y1), (w, h), (sw, sh) = self._geometry(fw, fh)
        self._engine, holders = shared_engine([pixel_group_of(d) for d in self._detector_list], w, h, sw, sh,
                                              device=self._device, max_batch=self._batch_size)
        for d, holder in zip(self._detector_list, holders):
            d.attach_engine(holder)
        self._base_timecode = base_timecode_of(video)
        if self._stats_manager is not None and hasattr(self._stats_manager, "_base_timecode"):
            self._stats_manager._base_timecode = self._base_timecode
        start_frame_num = video.frame_number
        end_frame = window_end_frame(self._base_timecode, start_frame_num, duration, end_time)
        self._channel_order = getattr(video, "channel_order", "bgr")
        gather = FrameBatches(video, (x0, y0, x1, y1), (w, h), self._batch_size, cropped=self._crop is not None,
                              frame_skip=frame_skip, end_frame=end_frame)
        pending = None  # (timecodes, frames_view, first engine index)
        while True:
            # 1. gather the next batch while the GPU works on the previous one
            tcs, batch, use_pinned = gather.next() or ([], None, False)
            # 2. launch the fused pass on the new batch (its H2D overlaps step 3's host work)
            nxt = None
            if batch is not None:
                first = self._engine.frame_count
                if isinstance(batch, np.ndarray):
                    self._engine.submit(batch, pinned=use_pinned)
                else:  # CUDA frames: a view, or a list of frames from a stream without read_batch
                    for frames in (batch if isinstance(batch, list) else [batch]):
                        self._engine.submit(frames, channel_order=self._channel_order)
                if self._start_pos is None:
                    self._start_pos = tcs[0]
                self._last_pos = tcs[-1]
                nxt = (tcs, batch, first)
            # 3. retire the previous batch (device scans + per-frame state machines)
            if pending is not None:
                self._consume(*pending, callback)
            pending = nxt
            if pending is None:
                break
        if self._last_pos is not None:
            # scene_manager.py:618-621: the stream's position, which is past the last scored frame when
            # frame_skip dropped frames behind it
            self._last_pos = video.position
            for d in self._detector_list:
                self._cutting_list += d.post_process(self._last_pos)
        gather.close()
        if self._scratch is not None:
            self._scratch.close()
            self._scratch = None
        return video.frame_number - start_frame_num

    def _consume(self, timecodes, frames, first, callback) -> None:
        """Per-frame state machines over one scored batch.  A detector may report a cut up to
        `event_buffer_length` frames behind the frame it is looking at (AdaptiveDetector's window,
        FlashFilter's merge), so callbacks search the tail of the previous batch as well - the
        reference's `_frame_buffer` (scene_manager.py:422-434).  Callbacks receive numpy BGR frames: CUDA frames
        are copied out for them (and only for them) through psd_gather_bgr."""
        on_device = isinstance(frames, list) or _dlpack.is_dlpack(frames)

        def host(frame):
            if not on_device:
                return np.array(frame)  # the staging buffer is reused
            if self._scratch is None:  # reused: freeing device memory would wait for the whole device
                self._scratch = DeviceBuffer(self._engine.src_frame_bytes, self._engine.device)
            return download_bgr(frame, self._channel_order, self._engine.device, self._scratch)

        # process_batch only validates the frames of a batch the engine already holds: one stands for a list
        sample = frames[0] if isinstance(frames, list) else frames
        for d in self._detector_list:
            cuts = d.process_batch(timecodes, sample, first=first)
            self._cutting_list += cuts
            if callback:
                for cut in cuts:
                    for tc, frame in self._frame_tail:
                        if cut == tc:
                            callback(frame, tc)
                    for tc, frame in zip(timecodes, frames):
                        if cut == tc:
                            callback(frame if not on_device else host(frame), tc)
        if callback and self._frame_buffer_size > 0:
            k = self._frame_buffer_size
            tail = [(tc, host(f)) for tc, f in list(zip(timecodes, frames))[-k:]]
            self._frame_tail = (self._frame_tail + tail)[-k:]
