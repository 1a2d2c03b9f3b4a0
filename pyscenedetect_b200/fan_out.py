"""One read of each clip for several settings: the clips of `detect_clips` scored under every (auto_downscale,
downscale, crop, frame_skip) setting of a sweep at once, as the reference harness's FanOutVideoStream
(scenedetect/_fan_out.py) serves one decode to many configurations.

Each clip is read once, over the union of the settings' windows (`StreamWindow.frames_read` of each setting's step; a
setting with frame_skip f reads up to f frames past its last processed frame).  A frame that some setting processes is
decoded; every other frame is read with `decode=False`.  Afterwards the stream stands at the union's end, which is
past some settings' own ends.  Each setting's positions and processed frames follow from its step by the same
arithmetic, not from a second read.

Every (clip group, setting) pair has its own engine, built by `shared_engine` with the setting's `_geometry`:
* CUDA frames: every setting's engine takes its own view of the same frames (`chunk[o::step]`, cropped);
* host frames: each frame a setting processes is copied into page-locked memory once and uploaded once, and every
  setting's engine scores its frames from that device copy (`Engine.submit_layout`: a crop and a frame step are only
  strides).  The copy is overwritten only after every engine has synchronised.
A pass ends for every setting at the same clip boundary, once the pass has read `clips.MAX_PASS_FRAMES` frames.
"""

from __future__ import annotations

import numpy as np

from . import _dlpack, clips
from .clips import ClipResult, _group_key
from .compat import FrameTimecode
from .engine import DeviceBuffer, PinnedBuffer
from .scene_manager import StreamWindow, base_timecode_of, shared_engine, window_end_frame


def _runs(slots: list) -> list:
    """Ascending slot indices -> maximal arithmetic runs [(first, stride, count)]."""
    runs = []
    i = 0
    while i < len(slots):
        if i + 1 == len(slots):
            runs.append((slots[i], 1, 1))
            break
        stride, k = slots[i + 1] - slots[i], 2
        while i + k < len(slots) and slots[i + k] - slots[i + k - 1] == stride:
            k += 1
        runs.append((slots[i], stride, k))
        i += k
    return runs


class _HostFeed:
    """Host frames of one group: copied into a page-locked batch of full frames (or of each frame's `crop` region, the
    part of the current clip's frame that any setting reads), uploaded once per batch, then scored by every setting's
    engine from the device copy, each through its crop and its own frames' slots."""

    def __init__(self, engines, boxes, frame_size, batch_size: int, device: int):
        fw, fh = frame_size
        self.engines, self.boxes = engines, boxes
        self.fw, self.fb = fw, fw * fh * 3
        self.batch_size = batch_size
        self.pinned = PinnedBuffer(batch_size * self.fb)
        self.frames = self.pinned.array.reshape(batch_size, fh, fw, 3)
        self.device_copy = DeviceBuffer(batch_size * self.fb, device)
        self.k = 0
        self.slots = [[] for _ in engines]
        self.uploaded = 0  # bytes copied to the device
        self.crop = None   # (x0, y0, x1, y1) of the current clip's frames that the batch holds; None: the whole frame

    def add(self, frame, users) -> None:
        if self.crop is not None:
            x0, y0, x1, y1 = self.crop
            frame = frame[y0:y1, x0:x1]
        np.copyto(self.frames[self.k], frame)
        for s in users:
            self.slots[s].append(self.k)
        self.k += 1
        if self.k == self.batch_size:
            self.flush()

    def flush(self) -> None:
        if not self.k:
            return
        for e in self.engines:  # the device copy is read by every engine of the previous batch
            e.sync()
        self.device_copy.upload(self.frames[:self.k])
        self.uploaded += self.k * self.fb
        row = self.fw * 3
        for e, (x0, y0, _x1, _y1), slots in zip(self.engines, self.boxes, self.slots):
            for first, stride, count in _runs(slots):
                e.submit_layout(self.device_copy.ptr + first * self.fb + y0 * row + x0 * 3, count,
                                (stride * self.fb, row, 3, 1))
        self.k = 0
        self.slots = [[] for _ in self.engines]

    def close(self) -> None:
        self.pinned.close()
        self.device_copy.close()


class _DeviceFeed:
    """CUDA frames of one group: every setting's engine takes its own cropped view of the frames it processes, its box
    counted from the corner of the current clip's `crop` (None: of the whole frame)."""

    def __init__(self, engines, boxes, order: str, batch_size: int):
        self.engines, self.boxes, self.order = engines, boxes, order
        self.batch_size = batch_size
        self.held = 0
        self.uploaded = 0
        self.crop = None

    def _box(self, s: int) -> tuple:
        x0, y0, x1, y1 = self.boxes[s]
        if self.crop is None:
            return x0, y0, x1, y1
        ox, oy = self.crop[:2]
        return ox + x0, oy + y0, ox + x1, oy + y1

    def add(self, frame, users) -> None:
        for s in users:
            x0, y0, x1, y1 = self._box(s)
            self.engines[s].submit(frame[y0:y1, x0:x1], channel_order=self.order)
        self.held += 1
        if self.held >= self.batch_size:
            self.flush()

    def add_views(self, s: int, view) -> None:
        x0, y0, x1, y1 = self._box(s)
        self.engines[s].submit(view[:, y0:y1, x0:x1], channel_order=self.order)
        self.held += view.shape[0]

    def flush(self) -> None:
        """Retire what the engines read, so that the stream's frames are released."""
        for e in self.engines:
            e.sync()
        self.held = 0

    def close(self) -> None:
        pass


def _read_clip(video, steps, feed, batch_size: int, views: bool, duration, end_time):
    """Read one clip once for every setting -> (frames read, [ClipResult per setting], [frames processed per
    setting])."""
    start, fps = video.frame_number, video.frame_rate
    end_frame = window_end_frame(base_timecode_of(video), start, duration, end_time)
    ext = [StreamWindow.frames_read(st, start, end_frame) for st in steps]
    union = None if any(e is None for e in ext) else max(ext)
    positions = {}  # local frame -> stream position after reading it, where some setting needs one
    needed = {0} | {e - 1 for e in ext if e is not None}
    i = 0
    # a stream that recycles its CUDA batches (`batches_kept`, e.g. a decoder's pool) is read at most that many
    # chunks ahead of the engines' last synchronisation
    kept = getattr(video, "batches_kept", None)
    chunks = 0
    if views:  # read_batch: chunks of the union, each setting's view [o::step] of them
        while union is None or i < union:
            chunk = video.read_batch(batch_size if union is None else min(batch_size, union - i))
            if chunk is None:
                break
            n = int(chunk.shape[0])
            if not n:
                break
            on_cuda = _dlpack.is_dlpack(chunk)
            for s, (st, e) in enumerate(zip(steps, ext)):
                o = (-i) % st
                lim = n if e is None else min(n, e - i)
                if o >= lim:
                    continue
                if on_cuda:
                    feed.add_views(s, chunk[o:lim:st])
            if not on_cuda:
                for r in range(n):
                    users = [s for s, (st, e) in enumerate(zip(steps, ext))
                             if (i + r) % st == 0 and (e is None or i + r < e)]
                    if users:
                        feed.add(chunk[r], users)
            i += n
            chunks += 1
            if on_cuda and (feed.held >= batch_size or (kept is not None and chunks >= kept)):
                feed.flush()
                chunks = 0
        pos_of = lambda j: FrameTimecode(start + j, fps)  # noqa: E731  (as StreamWindow.read_views numbers them)
    else:
        while union is None or i < union:
            users = [s for s, (st, e) in enumerate(zip(steps, ext)) if i % st == 0 and (e is None or i < e)]
            frame = video.read(decode=bool(users))
            if frame is False:
                break
            if i in needed:
                positions[i] = video.position
            if users:
                feed.add(frame, users)
            i += 1
        last = video.position if i else None
        pos_of = lambda j: positions[j] if j < i - 1 else last  # noqa: E731
    results, scored = [], []
    for st, e in zip(steps, ext):
        r = ClipResult(fps=fps)
        r.frames = i if e is None else min(e, i)
        if r.frames:
            r.start, r.end = pos_of(0), pos_of(r.frames - 1)
        results.append(r)
        scored.append(len(range(0, r.frames, st)))
    return i, results, scored


def _clip_plan(windows) -> tuple:
    """One clip's `clips._ClipWindow` under every setting -> (the box of its frames that some setting reads, the group
    key of its geometry: that box's size and every setting's box within it, cropped size and scored size)."""
    boxes = [w.box for w in windows]
    feed = (min(b[0] for b in boxes), min(b[1] for b in boxes), max(b[2] for b in boxes), max(b[3] for b in boxes))
    x0, y0 = feed[:2]
    inner = tuple(((b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0), w.size, w.scored) for b, w in zip(boxes, windows))
    return feed, ((feed[2] - x0, feed[3] - y0), inner)


def settings_passes(videos, groups, geometries, frame_skips, batch_size: int, device: int, duration=None,
                    end_time=None, counters: dict | None = None, windows=None):
    """Score the streams of `videos` once for every setting, pass by pass: clips grouped by `clips._group_key`, one
    engine per (group, setting) built by `shared_engine` with every pixel group of `groups` as a slot and
    `geometries[s]._geometry`, each clip read once (`_read_clip`) with the window of `duration` / `end_time` and
    setting s's `frame_skips[s]`.  With `windows`, clip i's `clips._ClipWindow` under every setting (windows[i][s]: its
    crop box, sizes, frame skip, duration and end_time) replaces those: clips are grouped by the region of their frames
    that the settings read and by every setting's box in it, cropped size and scored size, so clips of any source size
    cropped alike share a group; host frames are cropped to that region as they are copied.  Yields (engines, holders,
    done) at the end of every pass, one engine and one holder list per setting, `done` being [(input index, [ClipResult
    per setting], [frames processed per setting])] of the clips the pass holds, in order; the engines are reset for the
    next pass when the consumer asks for it.  `counters["uploaded"]` accumulates the host frame bytes copied to the
    device.  Close the generator to release the engines of an unfinished group."""
    steps = [int(f) + 1 for f in frame_skips]
    by_key: dict = {}
    for i, v in enumerate(videos):
        key = _group_key(v) if windows is None else _clip_plan(windows[i])[1] + _group_key(v)[1:]
        by_key.setdefault(key, []).append((i, v))
    for key, members in by_key.items():
        size, (on_cuda, views, order) = key[0], key[-3:]
        engines, holders, boxes, feed = [], [], [], None
        try:
            geometry = ([g._geometry(*size) for g in geometries] if windows is None else
                        [(box, w_h, scored) for box, w_h, scored in key[1]])
            for box, (w, h), (sw, sh) in geometry:
                e, hs = shared_engine(groups, w, h, sw, sh, device=device, max_batch=batch_size)
                engines.append(e)
                holders.append(hs)
                boxes.append(box)
            feed = (_DeviceFeed(engines, boxes, order, batch_size) if on_cuda else
                    _HostFeed(engines, boxes, size, batch_size, device))
            done, read = [], 0
            for n, (index, video) in enumerate(members):
                if _dlpack.on_cuda(video) != on_cuda:
                    raise ValueError("a stream's frames are not where its group's are (host or CUDA)")
                clip_steps, clip_duration, clip_end = steps, duration, end_time
                if windows is not None:
                    ws = windows[index]
                    feed.crop = _clip_plan(ws)[0]
                    clip_steps = [int(w.frame_skip) + 1 for w in ws]
                    clip_duration, clip_end = ws[0].duration, ws[0].end_time
                got, results, scored = _read_clip(video, clip_steps, feed, batch_size,
                                                  views or (not on_cuda and hasattr(video, "read_batch")),
                                                  clip_duration, clip_end)
                done.append((index, results, scored))
                read += got
                if read >= clips.MAX_PASS_FRAMES or n + 1 == len(members):
                    feed.flush()
                    for e in engines:
                        e.sync()
                    yield engines, holders, done
                    if n + 1 < len(members):
                        for e in engines:
                            e.reset()
                    done, read = [], 0
        finally:
            if feed is not None:
                if counters is not None:
                    counters["uploaded"] = counters.get("uploaded", 0) + feed.uploaded
                feed.close()
            for e in engines:
                e.close()


__all__ = ["settings_passes"]
