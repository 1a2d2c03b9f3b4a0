"""Detector parameter sweeps on the device: score a video once, then run every grid cell's cut automaton and
its precision / recall counts on the GPU.

The reference's benchmark harness (benchmark/sweep.py:142-187) decodes a video once per chunk of cells
and runs a complete SceneManager + detector per cell, so the per-frame cv2 arithmetic runs once per cell.
Almost no grid parameter changes that arithmetic, only the cut automaton after it.  Here:

* cells whose pixel-pass parameters agree (`required_features`, `edge_kernel_size_arg`, `engine_kwargs`)
  form one pixel group; `run` decodes the video once into ONE `Engine` that holds every group's dilation
  kernel size and hash geometry as a slot (as SceneManager.detect_scenes does for its detectors), so each
  batch is uploaded, resized, scored and Canny-classified once;
* each distinct metric array (content_val per weight vector, adaptive ratio per (weights, window_width,
  min_content_val), average_rgb, hist correlation per `bins`, hash distance) is computed once by the
  existing psd_scan_* kernels;
* psd_sweep_cuts runs every cell's automaton (one thread per cell) and psd_sweep_eval scores every
  (cell, tolerance) as benchmark/evaluator.py:307-331 does.  Only the counts come back to the host; a
  cell's cut list is read back when `SweepResult.cuts` asks for it.

Usage::

    sw = ParameterSweep(ContentDetector, grid=[{"threshold": t, "min_scene_len": s} for t in ts for s in ss],
                        tolerances=(0, 1))
    r = sw.run(video, ground_truth=GroundTruth(hard_cuts=[...], fades=[(start, end), ...]))
    r.cuts(k); r.hard(k, 1); r.hard_offset(k, 1); r.fades(k)
    sw.totals()   # counts summed over every video run so far, with precision / recall / F1
"""

from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass, field

import numpy as np

from . import _capi
from ._capi import check
from .detectors._base import EngineDetector, PixelGroup, pixel_group_of
from .device_cuts import automaton_args, flash_filter_frames, histogram_threshold, min_len_frames, scan_metric
from .engine import DeviceBuffer
from .scene_manager import FrameBatches, SceneManager, shared_engine

_KIND = {"content": _capi.SWEEP_CONTENT, "adaptive": _capi.SWEEP_ADAPTIVE, "threshold": _capi.SWEEP_THRESHOLD,
         "histogram": _capi.SWEEP_HISTOGRAM, "hash": _capi.SWEEP_HASH}


@dataclass
class GroundTruth:
    """One video's ground truth (benchmark/evaluator.py:58-64): strictly increasing hard-cut frames and
    inclusive (start, end) fade intervals, kept in the order given."""

    hard_cuts: list[int]
    fades: list[tuple[int, int]] = field(default_factory=list)

    def __post_init__(self):
        self.hard_cuts = [int(g) for g in self.hard_cuts]
        if any(b <= a for a, b in zip(self.hard_cuts, self.hard_cuts[1:])):
            raise ValueError("GroundTruth.hard_cuts must be strictly increasing")
        fades = []
        for f in self.fades:
            start, end = f
            fades.append((int(start), int(end)))
        self.fades = fades


@dataclass
class EventCounts:
    """Counts of one event type; precision / recall / F1 as evaluator.py:94-114 computes them."""

    matched: int = 0
    false_positives: int = 0
    missed: int = 0

    @property
    def precision(self) -> float:
        denom = self.matched + self.false_positives
        return self.matched / denom if denom else 0.0

    @property
    def recall(self) -> float:
        denom = self.matched + self.missed
        return self.matched / denom if denom else 0.0

    @property
    def f1(self) -> float:
        p, r = self.precision, self.recall
        return 2 * p * r / (p + r) if (p + r) else 0.0

    def __add__(self, other: EventCounts) -> EventCounts:
        return EventCounts(self.matched + other.matched, self.false_positives + other.false_positives,
                           self.missed + other.missed)


@dataclass
class CellTotals:
    """One cell's counts summed over videos (evaluator.py:167-186)."""

    params: dict
    hard: dict          # tolerance -> EventCounts
    hard_offset: dict   # tolerance -> (sum of |prediction - ground truth|, match count)
    fades: EventCounts

    def mean_abs_offset(self, tolerance: int) -> float:
        s, n = self.hard_offset[tolerance]
        return s / n if n else float("nan")


@dataclass(frozen=True)
class CellPlan:
    """One cell's automaton: kind, the metric key(s) it reads and the psd_sweep_cell fields; `min_scene_len`
    is converted to frames per video (`min_frames`)."""

    kind: str
    metric: tuple
    metric2: tuple | None
    threshold: float
    mode: int = 0
    window: int = 0
    min_content_val: float = 0.0
    fade_bias: float = 0.0
    add_final_scene: int = 0
    min_scene_len: object = 0

    def min_frames(self, fps) -> int:
        if self.kind == "content":  # FlashFilter's own conversion (detector.py:130-137)
            return flash_filter_frames(self.min_scene_len, fps)
        return min_len_frames(self.min_scene_len, fps)


def plan_cell(detector, group: int) -> CellPlan:
    """Detector object -> automaton arguments, through the same mapping `cuts_for_detector` uses and with
    the per-kind conversions the `DeviceCuts` methods apply before calling psd_cuts_*."""
    method, a = automaton_args(detector)
    if method == "content":
        w = tuple(a["weights"])
        return CellPlan("content", ("content_val", group, w), None, float(a["threshold"]),
                        mode=1 if a["suppress"] else 0, min_scene_len=a["min_scene_len"])
    if method == "adaptive":
        w, win, mcv = tuple(a["weights"]), int(a["window_width"]), float(a["min_content_val"])
        return CellPlan("adaptive", ("adaptive_ratio", group, w, win, mcv), ("content_val", group, w),
                        float(a["adaptive_threshold"]), window=win, min_content_val=mcv,
                        min_scene_len=a["min_scene_len"])
    if method == "histogram":
        return CellPlan("histogram", ("hist_correl", group, int(a["bins"])), None,
                        histogram_threshold(a["threshold"]), min_scene_len=a["min_scene_len"])
    if method == "hash":
        return CellPlan("hash", ("hash_dist", group), None, float(a["threshold"]), min_scene_len=a["min_scene_len"])
    return CellPlan("threshold", ("average_rgb", group), None, float(int(a["threshold"])),
                    mode=1 if a["ceiling"] else 0, fade_bias=float(a["fade_bias"]),
                    add_final_scene=1 if a["add_final_scene"] else 0, min_scene_len=a["min_scene_len"])


class SweepResult:
    """One video's sweep: per-cell counts on the host, cut lists on the device until `cuts` reads them."""

    def __init__(self, tolerances, slot_of, count, n_pred, hard, fades, cuts_buf, cap, end_frame, grid_ms):
        self.tolerances = tuple(tolerances)
        self._slot = slot_of
        self._count, self._n_pred = count, n_pred
        self._hard, self._fades = hard, fades
        self._cuts_buf, self._cap = cuts_buf, cap
        self.end_frame = end_frame
        self.grid_ms = grid_ms  # scans + psd_sweep_cuts + psd_sweep_eval, host clock ending in a sync

    def __len__(self) -> int:
        return len(self._slot)

    def _q(self, tol) -> int:
        try:
            return self.tolerances.index(tol)
        except ValueError:
            raise KeyError(f"tolerance {tol} was not evaluated (tolerances {self.tolerances})") from None

    def cuts(self, k: int) -> list[int]:
        """Cell k's predicted list as benchmark/sweep.py:169 records it: sorted unique cuts, then the end
        position; empty when the cell found no cut."""
        s = self._slot[k]
        m = int(self._n_pred[s])
        if m <= 0:
            return []
        got = self._cuts_buf.download((m - 1) * 8, offset=s * self._cap * 8).view(np.int64).tolist()
        return got + [self.end_frame]

    def raw_count(self, k: int) -> int:
        """How many cuts cell k's automaton emitted (before de-duplication)."""
        return int(self._count[self._slot[k]])

    def hard(self, k: int, tol: int) -> tuple[int, int, int]:
        """(matched, false_positives, missed) of hard cuts at tolerance `tol`."""
        h = self._hard[self._slot[k], self._q(tol)]
        return int(h[0]), int(h[1]), int(h[2])

    def hard_offset(self, k: int, tol: int) -> tuple[float, int]:
        """(sum of |prediction - ground truth|, match count) over the hard-cut matches (evaluator.py:136-139)."""
        h = self._hard[self._slot[k], self._q(tol)]
        return float(h[3]), int(h[4])

    def fades(self, k: int) -> tuple[int, int, int]:
        f = self._fades[self._slot[k]]
        return int(f[0]), int(f[1]), int(f[2])


def _cell_totals(grid, tolerances, th, tf) -> list[CellTotals]:
    """CellTotals per cell from summed counts th[cell][tolerance][5] and tf[cell][3], in grid order."""
    out = []
    for k, params in enumerate(grid):
        h, f = th[k], tf[k]
        out.append(CellTotals(
            params=params,
            hard={t: EventCounts(int(h[q, 0]), int(h[q, 1]), int(h[q, 2])) for q, t in enumerate(tolerances)},
            hard_offset={t: (float(h[q, 3]), int(h[q, 4])) for q, t in enumerate(tolerances)},
            fades=EventCounts(int(f[0]), int(f[1]), int(f[2]))))
    return out


def clip_eval_workspace_bytes(n_cells: int, n_clips: int, n_tol: int, cuts_total: int, n_gt: int,
                              n_fades: int) -> int:
    """The matching bitmaps psd_clip_eval needs (include/psd_b200.h), from sizes the host already has."""
    words = lambda bits: -(-bits // 32)  # noqa: E731
    return 4 * (n_tol * (n_cells * n_clips + words(cuts_total))
                + n_cells * n_tol * (2 * n_clips + words(n_gt) + words(n_fades)))


class _ClipPass:
    """One pass of `run_clips`: psd_clip_cuts' and psd_clip_eval's per-(cell, clip) arrays in device memory, owned
    here; each array is downloaded once, by the first accessor that reads it."""

    def __init__(self, pc, n_tol, n_pred, hard, fades):
        self.c, self.n_tol = pc.n_clips, n_tol
        self._bufs = {"offsets": (pc.offsets, np.int64, (-1,)), "n_pred": (n_pred, np.int32, (-1,)),
                      "hard": (hard, np.int64, (-1, n_tol, 5)), "fades": (fades, np.int64, (-1, 3))}
        self.cuts_buf = pc.cuts
        self._host = {}

    def host(self, name) -> np.ndarray:
        if name not in self._host:
            buf, dtype, shape = self._bufs[name]
            self._host[name] = buf.download(buf.nbytes).view(dtype).reshape(shape)
        return self._host[name]


class ClipSweepResult:
    """Every (cell, clip) of one `ParameterSweep.run_clips` call.  Per-(cell, clip) counts and cut lists stay in
    device memory until an accessor reads them; `totals` holds this call's counts summed over its clips."""

    def __init__(self, grid, tolerances, passes, where, end_frames, totals_hard, totals_fades, grid_ms):
        self.grid = grid
        self.tolerances = tuple(tolerances)
        self._passes = passes        # [_ClipPass]
        self._where = where          # clip -> (pass index, index within the pass)
        self._end = end_frames
        self._th, self._tf = totals_hard, totals_fades
        self.grid_ms = grid_ms       # scans + psd_clip_cuts + psd_clip_eval of every pass, host clock ending in syncs

    def __len__(self) -> int:
        return len(self.grid)

    @property
    def n_clips(self) -> int:
        return len(self._where)

    def _at(self, k: int, j: int):
        if not 0 <= k < len(self.grid):
            raise IndexError(f"cell {k} out of range")
        p, jj = self._where[j]
        ps = self._passes[p]
        return ps, k * ps.c + jj

    def _q(self, tol) -> int:
        try:
            return self.tolerances.index(tol)
        except ValueError:
            raise KeyError(f"tolerance {tol} was not evaluated (tolerances {self.tolerances})") from None

    def end_frame(self, j: int) -> int:
        """Clip j's end as SceneManager.get_scene_list ends it: its last position + 1 (clip-local frames)."""
        return self._end[j]

    def cuts(self, k: int, j: int) -> list[int]:
        """Cell k's predicted list on clip j, as `SweepResult.cuts` gives it: sorted unique cuts, then the clip's
        end frame; empty when the cell found no cut."""
        ps, t = self._at(k, j)
        m = int(ps.host("n_pred")[t])
        if m <= 0:
            return []
        o = int(ps.host("offsets")[t])
        got = ps.cuts_buf.download((m - 1) * 8, offset=o * 8).view(np.int64).tolist()
        return got + [self._end[j]]

    def raw_count(self, k: int, j: int) -> int:
        """How many cuts cell k's automaton emitted on clip j (before de-duplication)."""
        ps, t = self._at(k, j)
        o = ps.host("offsets")
        return int(o[t + 1] - o[t])

    def hard(self, k: int, j: int, tol: int) -> tuple[int, int, int]:
        """(matched, false_positives, missed) of clip j's hard cuts at tolerance `tol`."""
        ps, t = self._at(k, j)
        h = ps.host("hard")[t, self._q(tol)]
        return int(h[0]), int(h[1]), int(h[2])

    def hard_offset(self, k: int, j: int, tol: int) -> tuple[float, int]:
        """(sum of |prediction - ground truth|, match count) over clip j's hard-cut matches."""
        ps, t = self._at(k, j)
        h = ps.host("hard")[t, self._q(tol)]
        return float(h[3]), int(h[4])

    def fades(self, k: int, j: int) -> tuple[int, int, int]:
        ps, t = self._at(k, j)
        f = ps.host("fades")[t]
        return int(f[0]), int(f[1]), int(f[2])

    def totals(self) -> list[CellTotals]:
        """Every cell's counts summed over this call's clips, in grid order."""
        return _cell_totals(self.grid, self.tolerances, self._th, self._tf)


class ParameterSweep:
    """Every cell of `grid` (a list of `detector_cls(**params)` keyword dicts, as the reference harness takes
    them) over each video `run` is given.  `detector_cls` is one of this package's detectors; each cell is
    built by its constructor, so defaults, validation, `luma_only` and the histogram's threshold map are the
    constructor's own."""

    def __init__(self, detector_cls, grid, tolerances=(0, 1), device: int = 0, batch_size: int = 64,
                 max_cuts_per_cell: int = 4096):
        if not (isinstance(detector_cls, type) and issubclass(detector_cls, EngineDetector)):
            raise TypeError("ParameterSweep sweeps the detectors of this package")
        self.grid = [dict(p) for p in grid]
        if not self.grid:
            raise ValueError("the grid has no cells")
        tols = tuple(int(t) for t in tolerances)
        if not 1 <= len(tols) <= _capi.SWEEP_MAX_TOLERANCES or any(t < 0 for t in tols) or len(set(tols)) != len(tols):
            raise ValueError(f"tolerances must be 1 to {_capi.SWEEP_MAX_TOLERANCES} distinct non-negative frame counts")
        if int(batch_size) < 1 or int(max_cuts_per_cell) < 1:
            raise ValueError("batch_size and max_cuts_per_cell must be >= 1")
        self.tolerances = tols
        self.device = int(device)
        self.batch_size = int(batch_size)
        self.cap = int(max_cuts_per_cell)
        detectors = [detector_cls(**p) for p in self.grid]
        self.groups: list[PixelGroup] = []
        group_index: dict = {}
        self.cells: list[CellPlan] = []
        for d in detectors:
            g = pixel_group_of(d)
            gi = group_index.setdefault(g, len(self.groups))
            if gi == len(self.groups):
                self.groups.append(g)
            self.cells.append(plan_cell(d, gi))
        # metric keys in order of first use; cells sorted by the key they read (stable), so that the 32
        # cells of a warp share one metric array except where one key's run of cells ends inside the warp
        self.metric_keys: list[tuple] = []
        key_index: dict = {}
        for c in self.cells:
            for key in (c.metric2, c.metric):
                if key is not None and key not in key_index:
                    key_index[key] = len(self.metric_keys)
                    self.metric_keys.append(key)
        self.order = sorted(range(len(self.cells)), key=lambda k: (key_index[self.cells[k].metric], k))
        self.slot_of = [0] * len(self.cells)
        for s, k in enumerate(self.order):
            self.slot_of[k] = s
        self._lib = None
        self._totals_hard = np.zeros((len(self.cells), len(tols), 5), dtype=np.int64)
        self._totals_fades = np.zeros((len(self.cells), 3), dtype=np.int64)
        self.videos = 0

    # -- the whole pass --
    def run(self, video, ground_truth: GroundTruth | None = None) -> SweepResult:
        """Decode `video` once, score it with one Engine (SceneManager's default geometry: auto-downscale, no
        crop) that holds every pixel group's kernel size and hash geometry as a slot, then evaluate every cell.
        Without ground truth nothing is scored (every count is against an empty truth) and `totals` is not
        updated."""
        fw, fh = video.frame_size
        box, (w, h), (sw, sh) = SceneManager()._geometry(fw, fh)
        engine, holders = shared_engine(self.groups, w, h, sw, sh, device=self.device, max_batch=self.batch_size)
        gather = FrameBatches(video, box, (w, h), self.batch_size)
        first_frame = None
        try:
            try:
                while True:
                    item = gather.next()  # overlaps the GPU's work on the previous batch
                    engine.sync()  # retire the previous batch before its buffer is reused
                    if item is None:
                        break
                    tcs, frames, pinned = item
                    if first_frame is None:
                        first_frame = tcs[0].frame_num
                    engine.submit(frames, pinned=pinned)
            finally:
                gather.close()
            if first_frame is None:
                raise ValueError("the video has no frames")
            end_frame = video.position.frame_num + 1  # SceneManager.get_scene_list's end (last position + 1)
            return self.run_scored(holders, video.frame_rate, ground_truth, first_frame=first_frame,
                                   end_frame=end_frame)
        finally:
            engine.close()

    # -- the grid stage over results already held on the device --
    def run_scored(self, engines, fps, ground_truth: GroundTruth | None = None, first_frame: int = 0,
                   end_frame: int | None = None) -> SweepResult:
        """Evaluate every cell over frames the engines already scored: `engines[i]` holds pixel group
        `self.groups[i]`'s results for the same frames, the first of which is frame `first_frame` - an Engine
        per group, or the group's view (`Engine.view`) of one engine that holds every group's slots.
        `end_frame` defaults to first_frame + frame count."""
        if len(engines) != len(self.groups):
            raise ValueError(f"{len(self.groups)} pixel groups need as many engines, got {len(engines)}")
        lib = self._lib = self._lib or _capi.load()
        n = engines[0].frame_count
        if n <= 0 or any(e.frame_count != n for e in engines):
            raise ValueError("every engine must hold the same, non-zero number of frames")
        end_frame = first_frame + n if end_frame is None else int(end_frame)
        gt = ground_truth if ground_truth is not None else GroundTruth([])
        n_cells, n_tol, cap, dev = len(self.cells), len(self.tolerances), self.cap, self.device
        # allocations first, so the timed stage below is launches only
        arrays = {key: DeviceBuffer(n * 8, dev) for key in self.metric_keys}
        cuts =DeviceBuffer(n_cells * cap * 8, dev)
        count = DeviceBuffer(n_cells * 4, dev)
        n_pred = DeviceBuffer(n_cells * 4, dev)
        hard = DeviceBuffer(n_cells * n_tol * 5 * 8, dev)
        fades = DeviceBuffer(max(8, n_cells * 3 * 8), dev)
        gt_buf = DeviceBuffer(max(8, len(gt.hard_cuts) * 8), dev)
        fade_buf = DeviceBuffer(max(16, len(gt.fades) * 16), dev)
        if gt.hard_cuts:
            gt_buf.upload(np.asarray(gt.hard_cuts, dtype=np.int64))
        if gt.fades:
            fade_buf.upload(np.asarray(gt.fades, dtype=np.int64).reshape(-1, 2))
        words = -(-(cap + 1) // 32) + -(-len(gt.hard_cuts) // 32) + -(-len(gt.fades) // 32)
        ws_bytes = n_cells * n_tol * 4 * words
        ws = DeviceBuffer(max(8, ws_bytes), dev)
        cells = (_capi.PsdSweepCell * n_cells)()
        for s, k in enumerate(self.order):
            c = self.cells[k]
            cells[s] = _capi.PsdSweepCell(
                kind=_KIND[c.kind], mode=c.mode, metric=arrays[c.metric].ptr,
                metric2=arrays[c.metric2].ptr if c.metric2 is not None else None, threshold=c.threshold,
                min_content_val=c.min_content_val, fade_bias=c.fade_bias, min_frames=c.min_frames(fps),
                window=c.window, add_final_scene=c.add_final_scene)
        tols = (C.c_int32 * n_tol)(*self.tolerances)

        t0 = time.perf_counter()
        for key in self.metric_keys:  # one scan launch per distinct metric array
            val = arrays[("content_val",) + key[1:3]].ptr if key[0] == "adaptive_ratio" else None
            scan_metric(lib, engines[key[1]], (key[0],) + key[2:], arrays[key].ptr, val)
        if len(engines) > 1:  # the cells read every group's arrays: order them after every group's scans
            for e in engines[1:]:
                e.sync()
        st = engines[0].compute_stream
        check(lib.psd_sweep_cuts(cells, n_cells, n, first_frame, cuts.ptr, count.ptr, cap, st), "psd_sweep_cuts")
        check(lib.psd_sweep_eval(cuts.ptr, count.ptr, n_cells, cap, end_frame, gt_buf.ptr, len(gt.hard_cuts),
                                 fade_buf.ptr, len(gt.fades), tols, n_tol, ws.ptr, ws.nbytes, n_pred.ptr, hard.ptr,
                                 fades.ptr, st), "psd_sweep_eval")
        engines[0].sync()
        grid_ms = (time.perf_counter() - t0) * 1e3

        count_h = count.download(n_cells * 4).view(np.int32)
        over = np.nonzero(count_h[self.slot_of] > cap)[0]  # grid order
        if over.size:
            k = int(over[0])
            raise RuntimeError(f"cell {k} ({self.grid[k]}) found {int(count_h[self.slot_of[k]])} cuts, more than "
                               f"max_cuts_per_cell={cap}")
        n_pred_h = n_pred.download(n_cells * 4).view(np.int32)
        hard_h = hard.download(n_cells * n_tol * 40).view(np.int64).reshape(n_cells, n_tol, 5)
        fades_h = fades.download(n_cells * 24).view(np.int64).reshape(n_cells, 3)
        if ground_truth is not None:
            self._totals_hard += hard_h[self.slot_of]
            self._totals_fades += fades_h[self.slot_of]
            self.videos += 1
        return SweepResult(self.tolerances, self.slot_of, count_h, n_pred_h, hard_h, fades_h, cuts, cap, end_frame,
                           grid_ms)

    # -- many clips per pass --
    def run_clips(self, videos, ground_truths=None) -> ClipSweepResult:
        """Every cell over every stream of `videos`: for each (cell, clip), what `run(videos[j], ground_truths[j])`
        gives on a fresh ParameterSweep with this grid, tolerances and batch size; `totals` and `videos` afterwards
        are what a loop of `run` leaves.  Streams are anything `detect_clips` reads (host or CUDA `ArrayVideoStream`s
        of any layout and channel order, reference `VideoStream`s) and may differ in length, frame rate and frame
        size; each is read from its current position, with SceneManager's default geometry, and its frame numbers
        are clip-local.

        The clips are scored as `detect_clips` scores them, pass by pass.  Each pass ends with the scans, ONE
        psd_clip_cuts for every (cell, clip) automaton and ONE psd_clip_eval that scores every (cell, clip,
        tolerance) against clip j's ground truth and sums the counts over the pass's clips on the device; only
        those sums and the cut total come back to the host.

        `ground_truths`: None (every count is against an empty truth and `totals` is not updated), or one
        GroundTruth per video.  ValueError for a length mismatch or a clip without frames, RuntimeError for a
        (cell, clip) with more than max_cuts_per_cell cuts; `totals` only changes when the call returns."""
        from .clips import _Pass, clip_passes
        videos = list(videos)
        if ground_truths is None:
            gts = [GroundTruth([])] * len(videos)
        else:
            gts = list(ground_truths)
            if len(gts) != len(videos):
                raise ValueError(f"{len(videos)} videos need as many ground truths, got {len(gts)}")
            if not all(isinstance(g, GroundTruth) for g in gts):
                raise ValueError("every ground truth must be a GroundTruth (GroundTruth([]) for a clip without cuts)")
        lib = self._lib = self._lib or _capi.load()
        n_cells, n_tol, dev = len(self.cells), len(self.tolerances), self.device
        tols = (C.c_int32 * n_tol)(*self.tolerances)
        th = np.zeros((n_cells, n_tol, 5), dtype=np.int64)
        tf = np.zeros((n_cells, 3), dtype=np.int64)
        passes, where, ends = [], [None] * len(videos), [0] * len(videos)
        grid_ms = 0.0
        device_pass = _Pass(self.cells, self.groups, dev)
        scoring = clip_passes(videos, self.groups, SceneManager(device=dev, batch_size=self.batch_size),
                              self.batch_size, dev)
        try:
            for engine, holders, done in scoring:
                for index, _r, m in done:
                    if not m:
                        raise ValueError(f"clip {index} has no frames")
                t0 = time.perf_counter()
                pc = device_pass.cuts(engine, holders, [(r, m) for _, r, m in done])
                indices = [index for index, _r, _m in done]
                c = pc.n_clips
                ggt = [gts[i] for i in indices]
                gt_off = np.concatenate([[0], np.cumsum([len(g.hard_cuts) for g in ggt])]).astype(np.int64)
                fade_off = np.concatenate([[0], np.cumsum([len(g.fades) for g in ggt])]).astype(np.int64)
                n_gt, n_fades = int(gt_off[-1]), int(fade_off[-1])
                gt_table = np.concatenate([gt_off, fade_off, [x for g in ggt for x in g.hard_cuts],
                                           [x for g in ggt for f in g.fades for x in f]]).astype(np.int64)
                gbuf = DeviceBuffer(gt_table.nbytes, dev)
                gbuf.upload(gt_table)
                m = n_cells * c
                ws = DeviceBuffer(max(8, clip_eval_workspace_bytes(n_cells, c, n_tol, pc.total, n_gt, n_fades)), dev)
                n_pred = DeviceBuffer(max(8, m * 4), dev)
                hard = DeviceBuffer(m * n_tol * 40, dev)
                fades = DeviceBuffer(m * 24, dev)
                sums = DeviceBuffer(n_cells * (n_tol * 5 + 3) * 8 + 8, dev)  # totals_hard, totals_fades, over
                try:
                    gt_cuts = gbuf.ptr + 2 * (c + 1) * 8
                    check(lib.psd_clip_eval(
                        pc.cuts.ptr, pc.offsets.ptr, n_cells, c, pc.total, self.cap, pc.end_frames, gbuf.ptr, gt_cuts,
                        n_gt, gbuf.ptr + (c + 1) * 8, gt_cuts + n_gt * 8, n_fades, tols, n_tol, ws.ptr, ws.nbytes,
                        n_pred.ptr, hard.ptr, fades.ptr, sums.ptr, sums.ptr + n_cells * n_tol * 40,
                        sums.ptr + n_cells * (n_tol * 5 + 3) * 8, engine.compute_stream), "psd_clip_eval")
                    engine.sync()
                    grid_ms += (time.perf_counter() - t0) * 1e3
                    got = sums.download(sums.nbytes).view(np.int64)
                finally:
                    for b in (gbuf, ws, sums, pc.table):
                        b.close()
                over = int(got[-1])
                if over >= 0:
                    k, jj = divmod(over, c)
                    o = pc.offsets.download(16, offset=over * 8).view(np.int64)
                    raise RuntimeError(f"cell {k} ({self.grid[k]}) found {int(o[1] - o[0])} cuts in clip "
                                       f"{indices[jj]}, more than max_cuts_per_cell={self.cap}")
                th += got[:n_cells * n_tol * 5].reshape(n_cells, n_tol, 5)
                tf += got[n_cells * n_tol * 5:-1].reshape(n_cells, 3)
                for jj, (index, r) in enumerate(zip(indices, pc.clips)):
                    where[index] = (len(passes), jj)
                    ends[index] = r.end.frame_num + 1
                passes.append(_ClipPass(pc, n_tol, n_pred, hard, fades))
        finally:
            scoring.close()
            device_pass.close()
        if ground_truths is not None:
            self._totals_hard += th
            self._totals_fades += tf
            self.videos += len(videos)
        return ClipSweepResult(self.grid, self.tolerances, passes, where, ends, th, tf, grid_ms)

    def totals(self) -> list[CellTotals]:
        """Every cell's counts summed over the videos and clips run with ground truth so far, in grid order."""
        return _cell_totals(self.grid, self.tolerances, self._totals_hard, self._totals_fades)


__all__ = ["ParameterSweep", "SweepResult", "ClipSweepResult", "GroundTruth", "EventCounts", "CellTotals",
           "PixelGroup", "CellPlan", "plan_cell", "pixel_group_of"]
