"""Scene detection over many clips in one pass: one engine stream per group of clips, one automaton launch for all
their cuts.

Dataset-curation pipelines split millions of short clips, and the reference's benchmark harness loops `detect()`
once per video (benchmark/__main__.py:44-61).  One `SceneManager.detect_scenes` per clip pays a fixed cost per clip:
a new engine (device allocations, result arrays that grow through synchronising reallocations), per-frame Python
state machines, and a device teardown.  `detect_clips` instead:

* groups the clips by (frame size, host or CUDA, channel order) and builds one engine per group through
  `shared_engine`, with every detector's edge and hash slots, exactly as SceneManager does for one video (with
  `windows`, by cropped and scored size instead of frame size: clips of any source size cropped to one size share an
  engine);
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

Results are those of a fresh `SceneManager(batch_size=...)` with the same `auto_downscale` / `downscale` / `crop`
and fresh detectors, running `detect_scenes(video, duration=, end_time=, frame_skip=)` on each clip: cut list, scene
lists and frame count.  Frame numbers are clip-local, frame-number timecodes at the clip's constant frame rate (as
`DeviceCuts` gives them).  Each clip is read through its own `StreamWindow`, the one detect_scenes reads a stream
through; with a frame skip, element i of a clip's metric slice is frame first + i * (frame_skip + 1), which
psd_clip_cuts_step's automata walk.  With `windows` every clip has its own crop, duration / end_time and frame_skip;
a pass whose clips step differently runs psd_clip_cuts_steps, which takes one step per clip, in the same one launch.

With `stats=True` each clip also gets the text a `StatsManager` attached to that SceneManager saves
(`save_to_csv`): the metric arrays the cuts are made from are already on the device, so psd_clip_stats_csv prints
every clip's rows there (three launches a pass) and one download per pass brings them back, instead of a
`set_metrics` per frame and a `str()` per value on the host.
"""

from __future__ import annotations

import csv
import ctypes as C
import io
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from . import _capi, _dlpack
from ._capi import check
from .compat import FrameTimecode
from .detectors import ContentDetector, ThresholdDetector
from .detectors._base import EngineDetector, pixel_group_of
from .device_cuts import scan_metric
from .engine import DeviceBuffer
from .scene_manager import (FrameBatches, SceneManager, StreamWindow, base_timecode_of, check_window,
                            get_scenes_from_cuts, shared_engine, window_end_frame)
from .sweep import _KIND, plan_cell

MAX_PASS_FRAMES = 1 << 16     # frames an engine holds before its pass is finished at the next clip boundary
FIRST_CUTS_PER_FRAME = 0.25   # first cut buffer of a pass, in cuts per frame held; grown once if the cuts need more
FIRST_STATS_BYTES = (32, 24)  # first CSV text buffer, in bytes per frame held: a + b * columns; grown once if short
WINDOW_KEYS = ("crop", "duration", "end_time", "frame_skip")  # what an entry of detect_clips(windows=) may set


@dataclass(frozen=True)
class _ClipWindow:
    """How one clip is read: its crop `box` (x0, y0, x1, y1) of cropped `size` (w, h), scored at `scored` (sw, sh), as
    `SceneManager._geometry` gives them under the clip's crop; and its detect_scenes window."""

    box: tuple
    size: tuple
    scored: tuple
    frame_skip: int = 0
    duration: object = None
    end_time: object = None


@dataclass
class ClipResult:
    """One clip's detection: what `SceneManager.get_cut_list` / `get_scene_list` / `detect_scenes` give."""

    fps: Fraction
    frames: int = 0                           # what detect_scenes returns: frames read from the stream
    cut_frames: list = field(default_factory=list)  # sorted unique cut frame numbers
    start: FrameTimecode | None = None       # position of the first frame scored (None: the clip had no frames)
    end: FrameTimecode | None = None         # the stream's position after the last frame
    stats_csv: bytes | None = None           # detect_clips(stats=True): what StatsManager.save_to_csv writes

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
    """A group's streams read one after the other as one stream, for `FrameBatches`: `read()` gives the next frame to
    process of the current clip's `StreamWindow` (with the clip's `frame_skip` and its own end frame of `duration` /
    `end_time`, as detect_scenes reads one stream) and moves on to the next clip when that window ends, recording each
    clip's positions and frame count; `box()` is the crop box of the clip the last frame came from.  At a clip
    boundary, once the pass holds `bound` frames, it reports an end (`paused`) until `resume()`."""

    def __init__(self, clips, bound: int, on_cuda: bool):
        self._clips = clips       # [(input index, stream, _ClipWindow)]
        self._k = -1
        self._on_cuda = on_cuda
        self.bound = bound
        self.paused = False
        self.held = 0             # frames processed in this pass
        self.done = []            # (input index, ClipResult, frames scored) of every clip finished in this pass
        self._result = self._window = self._pos = None
        self._start_num = self._scored = 0
        self._next()

    frame_number = property(lambda self: self.held)   # FrameBatches only reads positions relative to its start
    frame_rate = property(lambda self: self._result.fps if self._result else Fraction(30))
    position = property(lambda self: self._pos)       # of the last frame processed

    def _next(self):
        self._k += 1
        if self._k < len(self._clips):
            _, video, w = self._clips[self._k]
            self._start_num = video.frame_number
            self._result = ClipResult(fps=video.frame_rate)
            self._scored = 0
            end = window_end_frame(base_timecode_of(video), self._start_num, w.duration, w.end_time)
            self._window = StreamWindow(video, w.frame_skip, end)

    def box(self) -> tuple:
        return self._clips[min(self._k, len(self._clips) - 1)][2].box

    def _end_clip(self) -> None:
        """Close the current clip; pause if the pass holds enough frames and another clip follows."""
        index, video, _ = self._clips[self._k]
        r = self._result
        r.frames = video.frame_number - self._start_num
        if r.start is not None:
            r.end = video.position  # past the last frame processed when frame_skip read frames behind it
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
            frame = self._window.read()
            if frame is not False:
                if _dlpack.is_dlpack(frame) != self._on_cuda:
                    raise ValueError("a stream's frames are not where its group's are (host or CUDA)")
                self._pos = self._window.position
                self._took(1, self._pos)
                return frame
            self._end_clip()
        return False

    def resume(self) -> None:
        self.paused = False
        self.held = 0
        self.done = []


class _DeviceClipChain(_ClipChain):
    """The chain over CUDA streams with `read_batch`: views `chunk[skip::step]` of one clip at a time, as SceneManager
    reads them (FrameBatches crops them)."""

    def __dlpack_device__(self):
        return self._clips[min(self._k, len(self._clips) - 1)][1].__dlpack_device__()

    def read_batch(self, max_frames: int):
        while not self.paused and self._k < len(self._clips):
            got = self._window.read_views(max_frames)
            if got is not None:
                first, k, view = got
                self._took(k, FrameTimecode(first, self._result.fps))
                return view
            self._end_clip()
        return None


@dataclass
class PassCuts:
    """One pass's (cell, clip) cut lists in device memory, which this object owns: cell k's cuts in clip j are
    cuts[offsets[k * n_clips + j] .. offsets[k * n_clips + j + 1]), in emission order.  `table` holds the clip table
    psd_clip_cuts read: offsets[n_clips + 1], first frames[n_clips], end frames[n_clips] (what
    `SceneManager.get_scene_list` ends at: the last position + 1), then min_frames[n_cells * n_clips]."""

    clips: list                 # ClipResult of every clip scored, in pass order
    n_cells: int
    table: DeviceBuffer
    offsets: DeviceBuffer       # int64[n_cells * n_clips + 1]: exclusive offsets, then the total
    cuts: DeviceBuffer
    total: int
    tables: object = None       # cuts_tables: every setting's psd_clip_table (HOST), for psd_clip_eval_tables
    cell_table: object = None   # cuts_tables: the setting of every cell (HOST int32)

    @property
    def n_clips(self) -> int:
        return len(self.clips)

    @property
    def end_frames(self) -> int:
        """Device pointer to the int64 end frame of every clip."""
        return self.table.ptr + (2 * self.n_clips + 1) * 8

    def close(self) -> None:
        for b in (self.table, self.offsets, self.cuts):
            b.close()


class _Pass:
    """The device half of a many-clip pass: the cells' metric keys and metric arrays (reused pass after pass and
    group after group; they only grow), and the step that turns an engine's pass into every (cell, clip) cut list.
    `cells` are CellPlans over `groups`, the pixel groups whose results each engine holds as slots."""

    def __init__(self, cells, groups, device: int):
        self._lib = _capi.load()
        self.device = device
        self.cells, self.groups = list(cells), list(groups)
        self.keys = []  # metric keys in order of first use: content_val before the adaptive ratio that reads it
        for c in self.cells:
            for key in (c.metric2, c.metric):
                if key is not None and key not in self.keys:
                    self.keys.append(key)
        self._bufs = {}
        self.frame_step = 1         # frame_skip + 1 of the clips' windows (`cuts` without per-clip steps)
        self.columns = None         # stats: [(CSV key, metric key, component or None, head, tail)] in CSV order
        self.components_key = None  # stats: the content_val key whose scan also writes the four components
        self.header = b""

    @classmethod
    def of_detectors(cls, detectors, device: int, stats: bool = False) -> _Pass:
        groups, gi, cells = [], {}, []
        for d in detectors:
            g = pixel_group_of(d, stats)
            if g not in gi:
                gi[g] = len(groups)
                groups.append(g)
            cells.append(plan_cell(d, gi[g]))
        p = cls(cells, groups, device)
        if stats:
            p.plan_stats(detectors)
        return p

    def plan_stats(self, detectors) -> None:
        """One CSV column per metric key of the detectors, read from the metric array of the last detector that
        writes the key (SceneManager runs the detectors in order on every batch, so at every frame the last writer's
        value stands), with the frames of a clip that have no value: head / tail as the detectors skip them."""
        writers = {}
        for d, cell in zip(detectors, self.cells):
            if cell.kind in ("content", "adaptive"):  # content_detector.py:161-164,183-186: frames 1 .. n-1
                val = cell.metric if cell.kind == "content" else cell.metric2
                writers[ContentDetector.FRAME_SCORE_KEY] = (val, None, 1, 0)
                for i, name in enumerate(ContentDetector.Components._fields):
                    writers[name] = (val, i, 1, 0)
                if cell.kind == "adaptive":       # adaptive_detector.py:116-128: frames W .. n-1-W
                    writers[d.get_metrics()[-1]] = (cell.metric, None, cell.window, cell.window)
            elif cell.kind == "threshold":        # threshold_detector.py:127-129: every frame
                writers[ThresholdDetector.THRESHOLD_VALUE_KEY] = (cell.metric, None, 0, 0)
            else:                                 # histogram, hash: every frame with a predecessor
                writers[d.get_metrics()[0]] = (cell.metric, None, 1, 0)
        keys = sorted(set().union(*(d.get_metrics() for d in detectors)))
        assert set(keys) == set(writers), (keys, sorted(writers))
        if len(keys) > _capi.STATS_MAX_COLUMNS:
            raise ValueError(f"{len(keys)} metric columns: psd_clip_stats_csv prints at most {_capi.STATS_MAX_COLUMNS}")
        self.columns = [(k, *writers[k]) for k in keys]
        self.components_key = next((c[1] for c in self.columns if c[2] is not None), None)
        text = io.StringIO()
        csv.writer(text, lineterminator="\n").writerow(["Frame Number", "Timecode", *keys])
        self.header = text.getvalue().encode()

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

    def _scan(self, holders, offsets: int, c: int, n: int, tag=None) -> dict:
        """Every metric array of the cells over the n frames `holders` hold, clips at the device table `offsets` of c
        clips: one psd_scan_* (and its psd_clip_fill) per key.  `tag` keeps one setting's arrays apart from
        another's."""
        arrays = {key: self._buf(key if tag is None else (tag, key), n * 8) for key in self.keys}
        comps = self._buf("components", n * 32).ptr if self.components_key is not None else None
        for key in self.keys:
            val = arrays[("content_val",) + key[1:3]].ptr if key[0] == "adaptive_ratio" else None
            scan_metric(self._lib, holders[key[1]], (key[0],) + key[2:], arrays[key].ptr, val, clips=(offsets, c),
                        components=comps if key == self.components_key else None)
        return arrays

    def _cells(self, arrays_of) -> C.Array:
        """The psd_sweep_cell of every cell for each metric-array set of `arrays_of`, set-major."""
        k = len(self.cells)
        cells = (_capi.PsdSweepCell * (k * len(arrays_of)))()
        for s, arrays in enumerate(arrays_of):
            for i, cell in enumerate(self.cells):
                cells[s * k + i] = _capi.PsdSweepCell(
                    kind=_KIND[cell.kind], mode=cell.mode, metric=arrays[cell.metric].ptr,
                    metric2=arrays[cell.metric2].ptr if cell.metric2 is not None else None, threshold=cell.threshold,
                    min_content_val=cell.min_content_val, fade_bias=cell.fade_bias, min_frames=0, window=cell.window,
                    add_final_scene=cell.add_final_scene)
        return cells

    def _cut_lists(self, engine, m: int, n: int, launch, name: str):
        """The compact cut lists of m (cell, clip) automata over a pass of n frames: `launch(cuts, cap, offsets)`
        queues the cut entry on the engine's stream; the buffer is grown once if the total needs more.
        -> (offsets buffer, cuts buffer, total)."""
        obuf = DeviceBuffer((m + 1) * 8, self.device)
        cap = max(1, int(n * FIRST_CUTS_PER_FRAME)) if FIRST_CUTS_PER_FRAME > 0 else 0
        cuts = DeviceBuffer(max(8, cap * 8), self.device)
        cap = cuts.nbytes // 8
        for attempt in range(2):
            launch(cuts.ptr, cap, obuf.ptr)
            engine.sync()
            total = int(obuf.download(8, offset=m * 8).view(np.int64)[0])
            if total <= cap:
                break
            if attempt:
                raise RuntimeError(f"{name} needs {total} cuts after growing its buffer to {cap}")
            cuts.close()
            cuts = DeviceBuffer(total * 8, self.device)
            cap = cuts.nbytes // 8
        return obuf, cuts, total

    def cuts(self, engine, holders, clips: list, steps: list | None = None) -> PassCuts | None:
        """Every (cell, clip) cut list of `clips` ((ClipResult, frames scored) of the frames `engine` holds, in
        order), left in device memory; None when no clip has a frame.  Element i of clip j is frame start + i *
        steps[j] (`frame_step` for every clip when `steps` is None).  Only the cut total comes back to the host."""
        lib = self._lib
        scored = [r for r, m in clips if m]
        steps = [self.frame_step] * len(clips) if steps is None else list(steps)
        steps = [s for s, (_, m) in zip(steps, clips) if m]
        n = engine.frame_count
        if not scored:
            return None
        c, k = len(scored), len(self.cells)
        sizes = np.array([m for _, m in clips if m], dtype=np.int64)
        if int(sizes.sum()) != n:
            raise RuntimeError(f"the engine holds {n} frames, the clips {int(sizes.sum())}")
        table = np.concatenate([
            np.concatenate([[0], np.cumsum(sizes)]),
            [r.start.frame_num for r in scored],
            [r.end.frame_num + 1 for r in scored],
            [cell.min_frames(r.fps) for cell in self.cells for r in scored]]).astype(np.int64)
        tbuf = DeviceBuffer(table.nbytes, self.device)
        tbuf.upload(table)
        offsets, first, min_frames = tbuf.ptr, tbuf.ptr + (c + 1) * 8, tbuf.ptr + (3 * c + 1) * 8
        cells = self._cells([self._scan(holders, offsets, c, n)])
        st = engine.compute_stream

        step = steps[0] if len(set(steps)) == 1 else None
        per_clip = (C.c_int64 * c)(*steps) if step is None else None

        def launch(cuts, cap, obuf):
            if step == 1:
                check(lib.psd_clip_cuts(cells, k, offsets, first, c, min_frames, cuts, cap, obuf, st), "psd_clip_cuts")
            elif step is not None:  # post_process sees each clip's end position, past its last processed frame
                check(lib.psd_clip_cuts_step(cells, k, offsets, first, c, min_frames, cuts, cap, obuf, step,
                                             first + c * 8, st), "psd_clip_cuts_step")
            else:                   # clips read with different frame skips: each clip's own step
                check(lib.psd_clip_cuts_steps(cells, k, offsets, first, c, min_frames, cuts, cap, obuf, per_clip,
                                              first + c * 8, st), "psd_clip_cuts_steps")

        obuf, cuts, total = self._cut_lists(engine, k * c, n, launch, "psd_clip_cuts")
        return PassCuts(scored, k, tbuf, obuf, cuts, total)

    def cuts_tables(self, engines, holders, clips: list, steps: list, clip_steps: list | None = None) -> PassCuts:
        """`cuts` for the same clips scored under several settings: setting s's engine `engines[s]` holds clip j's
        clips[s][j] = (ClipResult, frames scored), element i of which is frame start + i * steps[s], or start + i *
        clip_steps[j] under every setting when `clip_steps` is given.  Each setting's scans run on its engine with its
        own clip table; then ONE psd_clip_cuts_tables (psd_clip_cuts_tables_steps for clips that step differently)
        runs every (setting, cell, clip) automaton, cell index s * len(cells) + k.  Every clip must have frames.  The
        result's `tables` hold each setting's table, its `clips` are setting 0's."""
        lib = self._lib
        n_set, k, c = len(engines), len(self.cells), len(clips[0])
        if clip_steps is not None and len(set(clip_steps)) == 1:  # clips that step alike: the table's frame_step
            steps, clip_steps = [int(clip_steps[0])] * n_set, None
        parts, lens = [], []
        for s, e in enumerate(engines):
            sizes = np.array([m for _, m in clips[s]], dtype=np.int64)
            if not sizes.all() or int(sizes.sum()) != e.frame_count:
                raise RuntimeError(f"setting {s}: the engine holds {e.frame_count} frames, the clips "
                                   f"{sizes.tolist()}")
            parts += [np.concatenate([[0], np.cumsum(sizes)]), [r.start.frame_num for r, _ in clips[s]],
                      [r.end.frame_num + 1 for r, _ in clips[s]]]
            lens.append(e.frame_count)
        parts.append(np.tile([cell.min_frames(r.fps) for cell in self.cells for r, _ in clips[0]], n_set))
        if clip_steps is not None:
            parts.append(clip_steps)
        table = np.concatenate(parts).astype(np.int64)
        tbuf = DeviceBuffer(table.nbytes, self.device)
        tbuf.upload(table)
        per = (3 * c + 1) * 8  # bytes of one setting's offsets, first frames and end frames
        min_frames = tbuf.ptr + n_set * per
        # psd_clip_eval_tables reads a table's end frames only: with per-clip steps its frame_step is a placeholder
        tables = (_capi.PsdClipTable * n_set)()
        for s in range(n_set):
            base = tbuf.ptr + s * per
            tables[s] = _capi.PsdClipTable(offsets=base, first_frame=base + (c + 1) * 8,
                                           end_frame=base + (2 * c + 1) * 8,
                                           frame_step=steps[s] if clip_steps is None else 1)
        if clip_steps is not None:
            step_ptr = min_frames + n_set * k * c * 8
            steps_tables = (_capi.PsdClipStepsTable * n_set)(*[
                _capi.PsdClipStepsTable(offsets=t.offsets, first_frame=t.first_frame, end_frame=t.end_frame,
                                        frame_step=step_ptr) for t in tables])
        arrays = [self._scan(holders[s], tables[s].offsets, c, lens[s], tag=s if s else None) for s in range(n_set)]
        for e in engines[1:]:  # the automata read every setting's arrays: order them after every engine's scans
            e.sync()
        cells = self._cells(arrays)
        cell_table = (C.c_int32 * (n_set * k))(*[s for s in range(n_set) for _ in range(k)])
        st = engines[0].compute_stream

        def launch(cuts, cap, obuf):
            if clip_steps is None:
                check(lib.psd_clip_cuts_tables(cells, n_set * k, tables, n_set, cell_table, c, min_frames, cuts, cap,
                                               obuf, st), "psd_clip_cuts_tables")
            else:
                check(lib.psd_clip_cuts_tables_steps(cells, n_set * k, steps_tables, n_set, cell_table, c, min_frames,
                                                     cuts, cap, obuf, st), "psd_clip_cuts_tables_steps")

        obuf, cuts, total = self._cut_lists(engines[0], n_set * k * c, sum(lens), launch, "psd_clip_cuts_tables")
        pc = PassCuts([r for r, _ in clips[0]], n_set * k, tbuf, obuf, cuts, total)
        pc.tables, pc.cell_table = tables, cell_table
        return pc

    def union(self, engine, pc: PassCuts, cell_offsets, cell_lists, max_cuts: int):
        """Cells that are sets of `pc`'s cells: cell k's list on clip j is the sorted union of the lists (i, j) for i in
        cell_lists[cell_offsets[k] .. cell_offsets[k + 1]) (host int32 arrays), as SceneManager.get_cut_list merges its
        detectors' cuts.  psd_clip_union's counting call gives the exact size, its writing call fills a buffer of that
        size.  `pc`'s lists are sorted in place and stay `pc`'s.  -> (PassCuts of the unions, sharing `pc`'s clip
        table, -1), or (None, the lowest list * n_clips + clip of `pc` with more than max_cuts cuts)."""
        c, n_cells = pc.n_clips, len(cell_offsets) - 1
        m = n_cells * c
        # offsets, their total, the overflow index, then every member list's unique length (int32)
        obuf = DeviceBuffer((m + 2) * 8 + -(-pc.n_cells * c // 2) * 8, self.device)
        cuts = None
        try:
            def call(out, cap):
                check(self._lib.psd_clip_union(pc.cuts.ptr, pc.offsets.ptr, pc.n_cells, c, pc.total, max_cuts,
                                               cell_offsets, cell_lists, n_cells, obuf.ptr + (m + 2) * 8, out, cap,
                                               obuf.ptr, obuf.ptr + (m + 1) * 8, engine.compute_stream),
                      "psd_clip_union")

            call(None, 0)
            engine.sync()
            total, over = (int(x) for x in obuf.download(16, offset=m * 8).view(np.int64))
            if over >= 0:
                obuf.close()
                return None, over
            cuts = DeviceBuffer(max(8, total * 8), self.device)
            call(cuts.ptr, total)
        except BaseException:
            obuf.close()
            if cuts is not None:
                cuts.close()
            raise
        return PassCuts(pc.clips, n_cells, pc.table, obuf, cuts, total, tables=pc.tables), -1

    def stats_csv(self, engine, pc: PassCuts) -> list:
        """The CSV of every clip of `pc` (header and rows), printed on the device by one psd_clip_stats_csv from the
        metric arrays `cuts` left, and brought back with one download."""
        n, c = engine.frame_count, pc.n_clips
        cols = (_capi.PsdStatsColumn * len(self.columns))()
        for i, (_, key, comp, head, tail) in enumerate(self.columns):
            ptr, stride = (self._bufs[key].ptr, 1) if comp is None else (self._bufs["components"].ptr + 8 * comp, 4)
            cols[i] = _capi.PsdStatsColumn(values=ptr, stride=stride, head=head, tail=tail)
        rates = np.array([float(r.start.frame_rate) for r in pc.clips], dtype=np.float64)
        rbuf = DeviceBuffer(rates.nbytes, self.device)
        cbuf = DeviceBuffer((c + 1) * 8, self.device)
        try:
            rbuf.upload(rates)
            rows = self._buf("stats_rows", (n + 1) * 8)
            a, b = FIRST_STATS_BYTES
            text = self._buf("stats_text", n * (a + b * len(cols)))
            for attempt in range(2):
                cap = text.nbytes
                check(self._lib.psd_clip_stats_csv(cols, len(cols), pc.table.ptr, pc.table.ptr + (c + 1) * 8, rbuf.ptr,
                                                   c, n, rows.ptr, text.ptr, cap, cbuf.ptr, engine.compute_stream),
                      "psd_clip_stats_csv")
                engine.sync()
                offs = cbuf.download((c + 1) * 8).view(np.int64).tolist()
                if offs[-1] <= cap:
                    break
                if attempt:
                    raise RuntimeError(f"psd_clip_stats_csv needs {offs[-1]} bytes after growing its buffer to {cap}")
                text = self._buf("stats_text", offs[-1])
            data = text.download(offs[-1]).tobytes() if offs[-1] else b""
        finally:
            rbuf.close()
            cbuf.close()
        return [self.header + data[offs[j]:offs[j + 1]] for j in range(c)]

    def finish(self, engine, holders, clips: list, steps: list | None = None) -> None:
        """Every clip of `clips` ((ClipResult, frames scored) of the frames `engine` holds, in order, each read with
        its step of `steps`, as `cuts` takes them) gets its cut frames: the union of every cell's cuts, as
        SceneManager.get_cut_list gives them; and with a stats plan its CSV (the header alone for a clip without
        frames)."""
        for r, _ in clips:
            if self.columns is not None:
                r.stats_csv = self.header
        pc = self.cuts(engine, holders, clips, steps)
        if pc is None:
            return
        try:
            k, c = pc.n_cells, pc.n_clips
            offs = pc.offsets.download((k * c + 1) * 8).view(np.int64).tolist()
            got = pc.cuts.download(pc.total * 8).view(np.int64).tolist() if pc.total else []
            texts = self.stats_csv(engine, pc) if self.columns is not None else None
        finally:
            pc.close()
        for j, r in enumerate(pc.clips):  # (cell i, clip j) is list i * c + j: SceneManager.get_cut_list per clip
            r.cut_frames = sorted({f for i in range(k) for f in got[offs[i * c + j]:offs[i * c + j + 1]]})
            if texts is not None:
                r.stats_csv = texts[j]


def _group_key(video) -> tuple:
    """(frame size, CUDA frames, read as views of `read_batch`, channel order of the CUDA frames)"""
    on_cuda = _dlpack.on_cuda(video)
    return (tuple(video.frame_size), on_cuda, on_cuda and hasattr(video, "read_batch"),
            getattr(video, "channel_order", "bgr") if on_cuda else "bgr")


def detect_clips(videos, detectors, auto_downscale: bool = True, downscale: int = 1, device: int = 0,
                 batch_size: int = 64, stats: bool = False, crop=None, duration=None, end_time=None,
                 frame_skip: int = 0, *, windows=None) -> list[ClipResult]:
    """Detect scenes in every stream of `videos` with every detector of `detectors`: for each clip, in input order,
    what a fresh `SceneManager(device=device, batch_size=batch_size)` with these `auto_downscale` / `downscale` /
    `crop` and fresh copies of the detectors give from `detect_scenes(video, duration=duration, end_time=end_time,
    frame_skip=frame_skip)`.  Streams are anything `detect_scenes` reads (`ArrayVideoStream` over numpy or CUDA
    arrays of any layout and channel order, a reference `VideoStream`) and may differ in length, frame rate and frame
    size; a stream is read from its current position.

    Every clip gets the same window, applied to it as detect_scenes applies it to one stream: `duration` counts from
    the clip's own position, `end_time` from its base timecode, both at its own frame rate; the first frame is always
    processed; `frame_skip` frames are read and not processed after each processed one, and `ClipResult.frames`
    counts them.  `crop` is SceneManager.crop's (X0, Y0, X1, Y1), inclusive, in every clip.

    `windows` (keyword only) gives each clip its own window instead: one entry per video, None or a dict with keys
    among `crop`, `duration`, `end_time` and `frame_skip`, meaning what the arguments of those names mean.  Clip i's
    result is then that SceneManager's with `crop = windows[i].get("crop")`, from `detect_scenes(video,
    duration=, end_time=, frame_skip=)` with the entry's values.  Clips cropped to one size share an engine and a pass
    whatever their source sizes, and clips with different frame skips share the pass's one automaton launch.

    `stats=True`: every result also has `stats_csv`, the bytes `StatsManager.save_to_csv` writes (line terminator
    "\\n") after that SceneManager, built with a fresh `StatsManager()`, ran `detect_scenes(video)`: the header
    `Frame Number,Timecode,` and the sorted metric keys of the detectors, then one row per frame that has a metric.
    As an attached StatsManager does, it turns on ContentDetector's edge component; the cut lists are those of
    `stats=False`.

    The detectors are configuration only: they are not attached to an engine or otherwise changed.  ValueError for
    an empty detector list or a detector with a `stats_manager` (the detectors take no StatsManager here: ask for
    `stats` instead), for the window arguments detect_scenes refuses (with its messages; `frame_skip` with `stats`
    included), and, before any frame is read, for a crop that starts outside some clip's frame; TypeError for a
    malformed crop.  With `windows`, every entry is checked the same way before any frame is read; TypeError for
    `windows` together with a window argument (`crop`, `duration` or `end_time` not None, `frame_skip` not 0), for
    an entry that is not None or a dict and for an unknown key; ValueError for a number of entries other than the
    number of videos."""
    detectors = list(detectors)
    if not detectors:
        raise ValueError("No detectors added")
    for d in detectors:
        if not isinstance(d, EngineDetector):
            raise TypeError("detect_clips drives the GPU detectors of this package")
        if d.stats_manager is not None:
            raise ValueError("detect_clips produces no per-frame metrics: detectors must not have a stats_manager")
    if windows is not None and (crop is not None or duration is not None or end_time is not None or frame_skip != 0):
        raise TypeError("detect_clips takes windows or crop / duration / end_time / frame_skip, not both")
    check_window(duration, end_time, frame_skip, stats)
    if downscale < 1:
        raise ValueError("Downscale factor must be a positive integer >= 1!")
    geometry = SceneManager(device=device, batch_size=batch_size)
    geometry._auto_downscale, geometry._downscale = bool(auto_downscale), int(downscale)
    geometry.crop = crop
    videos = list(videos)
    clip_windows = None
    if windows is not None:
        clip_windows = _clip_windows(videos, windows, geometry, stats)
    elif crop is not None:
        for i, v in enumerate(videos):
            fw, fh = v.frame_size
            x0, y0 = geometry._crop[:2]
            if x0 >= fw or y0 >= fh:
                raise ValueError(f"crop starts outside video boundary of clip {i} ({fw}x{fh})")
    results: list = [None] * len(videos)
    device_pass = _Pass.of_detectors(detectors, device, stats=stats)
    device_pass.frame_step = int(frame_skip) + 1
    passes = clip_passes(videos, device_pass.groups, geometry, batch_size, device, frame_skip=frame_skip,
                         duration=duration, end_time=end_time, windows=clip_windows)
    try:
        for engine, holders, done in passes:
            steps = () if clip_windows is None else ([int(clip_windows[i].frame_skip) + 1 for i, _, _ in done],)
            device_pass.finish(engine, holders, [(r, m) for _, r, m in done], *steps)
            for index, r, _ in done:
                results[index] = r
    finally:
        passes.close()
        device_pass.close()
    return results


def _clip_windows(videos, windows, geometry, stats: bool) -> list:
    """The `_ClipWindow` of every clip from detect_clips' `windows`, each entry checked as SceneManager.crop and
    detect_scenes check their arguments, and its crop against the clip's frame, before any geometry is computed.  An
    entry without a `crop` key keeps `geometry`'s crop; `geometry` is left as it was given."""
    windows = list(windows)
    if len(windows) != len(videos):
        raise ValueError(f"windows has {len(windows)} entries for {len(videos)} videos")
    base = geometry._crop
    try:
        checked = []
        for i, (v, w) in enumerate(zip(videos, windows)):
            w = {} if w is None else w
            if not isinstance(w, dict):
                raise TypeError(f"window {i} must be None or a dict, not {type(w).__name__}")
            for key in w:
                if key not in WINDOW_KEYS:
                    raise TypeError(f"window {i} has an unknown key {key!r}: the keys are {', '.join(WINDOW_KEYS)}")
            skip = w.get("frame_skip", 0)
            check_window(w.get("duration"), w.get("end_time"), skip, stats)
            geometry._crop = base
            if "crop" in w:
                geometry.crop = w["crop"]
            if geometry._crop is not None:
                fw, fh = v.frame_size
                if geometry._crop[0] >= fw or geometry._crop[1] >= fh:
                    raise ValueError(f"crop starts outside video boundary of clip {i} ({fw}x{fh})")
            checked.append((geometry._crop, skip, w.get("duration"), w.get("end_time")))
        out = []
        for v, (box, skip, duration, end_time) in zip(videos, checked):
            geometry._crop = box
            out.append(_ClipWindow(*geometry._geometry(*v.frame_size), skip, duration, end_time))  # its warning per clip
    finally:
        geometry._crop = base
    return out


def clip_passes(videos, groups, geometry, batch_size: int, device: int, frame_skip: int = 0, duration=None,
                end_time=None, windows=None):
    """Score the streams of `videos` pass by pass: one engine per group of clips built by `shared_engine` with every
    pixel group of `groups` as a slot, the clips of a group scored back to back, each through its own window
    (`_ClipChain`).  Without `windows`, clips are grouped by `_group_key` and read through `geometry._geometry` (a
    SceneManager's: its crop and scored size) and the window of `frame_skip` / `duration` / `end_time`; with
    `windows`, the `_ClipWindow` of every clip, they are grouped by cropped and scored size instead of frame size and
    each is read through its own.  Frames scored are frames processed.  Yields (engine, holders, done) at the end of
    every pass, `done` being [(input index, ClipResult, frames scored)] of the clips the engine holds, in order; the
    engine is reset for the next pass when the consumer asks for it.  Close the generator to release the engine of an
    unfinished group."""
    by_key: dict = {}
    for i, v in enumerate(videos):
        key = _group_key(v) if windows is None else (windows[i].size, windows[i].scored) + _group_key(v)[1:]
        by_key.setdefault(key, []).append((i, v))
    for key, members in by_key.items():
        on_cuda, views, order = key[-3:]
        if windows is None:
            group_window = _ClipWindow(*geometry._geometry(*key[0]), frame_skip, duration, end_time)
            clips = [(i, v, group_window) for i, v in members]
        else:
            clips = [(i, v, windows[i]) for i, v in members]
        (w, h), (sw, sh) = clips[0][2].size, clips[0][2].scored
        engine, holders = shared_engine(groups, w, h, sw, sh, device=device, max_batch=batch_size)
        chain = (_DeviceClipChain if views else _ClipChain)(clips, MAX_PASS_FRAMES, on_cuda)
        gather = FrameBatches(chain, chain.box, (w, h), batch_size)
        try:
            while True:
                item = gather.next()  # overlaps the GPU's work on the previous batch
                engine.sync()         # retire the previous batch before its buffer is reused
                if item is None:
                    yield engine, holders, chain.done
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


from .images import save_clip_images, save_images  # noqa: E402  (images of the scenes detect_clips finds)

__all__ = ["detect_clips", "ClipResult", "MAX_PASS_FRAMES", "save_images", "save_clip_images"]
