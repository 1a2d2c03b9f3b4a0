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

from .compat import FrameTimecode, StatsManager
from .detectors._base import EngineDetector
from ._capi import F_EDGES
from .engine import Engine, PinnedBuffer

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


class FrameBatches:
    """The frame-gathering half of the detection loop (scene_manager.py:650-689): reads `video` in batches of
    up to `batch_size` frames, cropped to `box` = (x0, y0, x1, y1) of size `size` = (w, h).  A stream with
    `read_batch` and no crop / frame skip is read zero-copy; otherwise frames are copied into one of two
    page-locked buffers, so that a batch can be gathered while the GPU scores the previous one.

    `next()` returns (timecodes, frames, pinned) or None at the end.  The frames of a batch stay valid until
    the batch after the next one is gathered: the caller must have synchronised the engines that read a batch
    before asking for the batch two after it.  `close()` frees the buffers, after the last batch is done."""

    def __init__(self, video, box, size, batch_size: int, cropped: bool = False, frame_skip: int = 0,
                 end_frame: int | None = None):
        self._video = video
        self._box, self._size = box, size
        self._batch_size = int(batch_size)
        self._frame_skip = frame_skip
        self._end_frame = end_frame
        self._zero_copy = hasattr(video, "read_batch") and not cropped and frame_skip == 0
        self._pinned = [None, None]
        self._which = 0
        self._done = False
        self._processed = 0

    def next(self):
        if self._done:
            return None
        video, end_frame, zero_copy = self._video, self._end_frame, self._zero_copy
        x0, y0, x1, y1 = self._box
        w, h = self._size
        fps = video.frame_rate
        tcs, batch = [], None
        want = self._batch_size
        if end_frame is not None and zero_copy:
            # the frame at position p is processed, then the loop stops unless p + 1 < end; the first
            # frame is always processed (the check follows the put, scene_manager.py:680-689)
            want = min(want, max(end_frame - video.frame_number, 1 if self._processed == 0 else 0))
        if want > 0:
            if zero_copy:
                pos0 = video.frame_number
                view = video.read_batch(want)
                if view is not None:
                    batch = view
                    tcs = [FrameTimecode(pos0 + i, fps) for i in range(view.shape[0])]
            else:
                which = self._which
                if self._pinned[which] is None:
                    self._pinned[which] = PinnedBuffer(self._batch_size * w * h * 3)
                buf = self._pinned[which].array.reshape(self._batch_size, h, w, 3)
                k = 0
                while k < want:
                    frame = video.read()
                    if frame is False:
                        self._done = True
                        break
                    np.copyto(buf[k], frame[y0:y1, x0:x1])
                    tcs.append(video.position)
                    k += 1
                    for _ in range(self._frame_skip):  # scene_manager.py:682-685
                        if not video.read(decode=False):
                            break
                    if end_frame is not None and not (video.position.frame_num + 1) < end_frame:
                        self._done = True
                        break
                batch = buf[:k] if k else None
        if batch is None:
            self._done = True
            return None
        self._processed += len(tcs)
        self._which ^= 1
        return tcs, batch, (not zero_copy) or bool(getattr(video, "is_pinned", False))

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
        if frame_skip > 0 and self._stats_manager is not None:
            raise ValueError("frame_skip must be 0 when using a StatsManager.")
        if duration is not None and end_time is not None:
            raise ValueError("duration and end_time cannot be set at the same time!")
        if duration is not None and isinstance(duration, (int, float)) and duration < 0:
            raise ValueError("duration must be greater than or equal to 0!")
        if end_time is not None and isinstance(end_time, (int, float)) and end_time < 0:
            raise ValueError("end_time must be greater than or equal to 0!")
        self.clear()
        self._frame_tail = []
        fw, fh = video.frame_size
        (x0, y0, x1, y1), (w, h), (sw, sh) = self._geometry(fw, fh)
        features = 0
        for d in self._detector_list:
            features |= d.required_features()
        # only detectors that use the edge component own a dilation kernel (content_detector.py:126-134)
        ks = {d.edge_kernel_size_arg() for d in self._detector_list if d.required_features() & F_EDGES}
        if len(ks) > 1:
            raise ValueError("detectors sharing a SceneManager's fused pass must agree on kernel_size")
        extra: dict = {}
        for d in self._detector_list:
            for k, v in d.engine_kwargs().items():
                if extra.setdefault(k, v) != v:
                    raise ValueError(f"detectors sharing a SceneManager's fused pass must agree on {k}")
        self._engine = Engine(w, h, features, width=sw, height=sh, device=self._device,
                              max_batch=self._batch_size, edge_kernel_size=ks.pop() if ks else 0, **extra)
        for d in self._detector_list:
            d.attach_engine(self._engine)
        fps = video.frame_rate
        base = getattr(video, "base_timecode", None)
        self._base_timecode = base if base is not None else FrameTimecode(0, fps)
        if self._stats_manager is not None and hasattr(self._stats_manager, "_base_timecode"):
            self._stats_manager._base_timecode = self._base_timecode
        # scene_manager.py:543-547: end_time is absolute, duration is relative to the current position
        start_frame_num = video.frame_number
        end_frame = None  # frames with position + 1 >= end are the last ones processed (scene_manager.py:686-689)
        if end_time is not None:
            end_frame = (self._base_timecode + end_time).frame_num
        elif duration is not None:
            end_frame = ((self._base_timecode + duration) + start_frame_num).frame_num
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
                self._engine.submit(batch, pinned=use_pinned)
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
        return video.frame_number - start_frame_num

    def _consume(self, timecodes, frames, first, callback) -> None:
        """Per-frame state machines over one scored batch.  A detector may report a cut up to
        `event_buffer_length` frames behind the frame it is looking at (AdaptiveDetector's window,
        FlashFilter's merge), so callbacks search the tail of the previous batch as well - the
        reference's `_frame_buffer` (scene_manager.py:422-434)."""
        for d in self._detector_list:
            cuts = d.process_batch(timecodes, frames, first=first)
            self._cutting_list += cuts
            if callback:
                for cut in cuts:
                    for tc, frame in self._frame_tail:
                        if cut == tc:
                            callback(frame, tc)
                    for tc, frame in zip(timecodes, frames):
                        if cut == tc:
                            callback(frame, tc)
        if callback and self._frame_buffer_size > 0:
            k = self._frame_buffer_size
            tail = [(tc, np.array(f)) for tc, f in list(zip(timecodes, frames))[-k:]]  # the staging buffer is reused
            self._frame_tail = (self._frame_tail + tail)[-k:]
