"""Detector parameter sweeps on the device: score a video once, then run every grid cell's cut automaton and
its precision / recall counts on the GPU.

The reference's benchmark harness (benchmark/sweep.py:142-187) decodes a video once per chunk of cells
and runs a complete SceneManager + detector per cell, so the per-frame cv2 arithmetic runs once per cell.
Almost no grid parameter changes that arithmetic, only the cut automaton after it.  Here:

* cells whose pixel-pass parameters agree (`required_features`, `edge_kernel_size_arg`, `engine_kwargs`:
  the rules SceneManager.detect_scenes applies) form one pixel group with one `Engine`; the video is
  decoded once and every batch goes to every group's engine;
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
from ._capi import F_EDGES, check
from .detectors._base import EngineDetector
from .device_cuts import automaton_args, flash_filter_frames, histogram_threshold, min_len_frames
from .engine import DeviceBuffer, Engine
from .scene_manager import FrameBatches, SceneManager

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
class PixelGroup:
    """Cells that share one fused score pass: the Engine arguments they need."""

    features: int
    edge_kernel_size: int
    engine_kwargs: tuple  # sorted (name, value) pairs

    def make_engine(self, src_width: int, src_height: int, width: int, height: int, device: int = 0,
                    max_batch: int = 64) -> Engine:
        return Engine(src_width, src_height, self.features, width=width, height=height, device=device,
                      max_batch=max_batch, edge_kernel_size=self.edge_kernel_size, **dict(self.engine_kwargs))


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


def pixel_group_of(detector) -> PixelGroup:
    """SceneManager.detect_scenes' rules: the features a detector needs, its dilation kernel when it uses the
    edge component, and its extra Engine arguments."""
    feats = detector.required_features()
    return PixelGroup(feats, detector.edge_kernel_size_arg() if feats & F_EDGES else 0,
                      tuple(sorted(detector.engine_kwargs().items())))


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
        """Decode `video` once, score it with one Engine per pixel group (SceneManager's default geometry:
        auto-downscale, no crop), then evaluate every cell.  Without ground truth nothing is scored (every
        count is against an empty truth) and `totals` is not updated."""
        fw, fh = video.frame_size
        box, (w, h), (sw, sh) = SceneManager()._geometry(fw, fh)
        engines = [g.make_engine(w, h, sw, sh, self.device, self.batch_size) for g in self.groups]
        gather = FrameBatches(video, box, (w, h), self.batch_size)
        first_frame = None
        try:
            while True:
                item = gather.next()  # overlaps the GPU's work on the previous batch
                for e in engines:
                    e.sync()  # retire the previous batch before its buffer is reused
                if item is None:
                    break
                tcs, frames, pinned = item
                if first_frame is None:
                    first_frame = tcs[0].frame_num
                for e in engines:
                    e.submit(frames, pinned=pinned)
        finally:
            gather.close()
        if first_frame is None:
            raise ValueError("the video has no frames")
        end_frame = video.position.frame_num + 1  # SceneManager.get_scene_list's end (last position + 1)
        try:
            return self.run_scored(engines, video.frame_rate, ground_truth, first_frame=first_frame,
                                   end_frame=end_frame)
        finally:
            for e in engines:
                e.close()

    # -- the grid stage over results already held on the device --
    def run_scored(self, engines, fps, ground_truth: GroundTruth | None = None, first_frame: int = 0,
                   end_frame: int | None = None) -> SweepResult:
        """Evaluate every cell over frames the engines already scored: `engines[i]` holds pixel group
        `self.groups[i]`'s results for the same frames, the first of which is frame `first_frame`.
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
        comps = DeviceBuffer(4 * n * 8, dev)  # psd_scan_content's components (not read)
        cuts = DeviceBuffer(n_cells * cap * 8, dev)
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
            e = engines[key[1]]
            st = e.compute_stream
            if key[0] == "content_val":
                sums, _ = e.device_results()
                wts = key[2]
                w = (C.c_double * 4)(*[float(x) for x in wts])
                check(lib.psd_scan_content(sums, n, e.n_pixels, w, float(sum(abs(x) for x in wts)), comps.ptr,
                                           arrays[key].ptr, st), "psd_scan_content")
            elif key[0] == "adaptive_ratio":
                check(lib.psd_scan_adaptive(arrays[("content_val",) + key[1:3]].ptr, n, key[3], key[4],
                                            arrays[key].ptr, st), "psd_scan_adaptive")
            elif key[0] == "average_rgb":
                sums, _ = e.device_results()
                check(lib.psd_scan_average(sums, n, e.n_pixels * 3, arrays[key].ptr, st), "psd_scan_average")
            elif key[0] == "hist_correl":
                _, yhist = e.device_results()
                check(lib.psd_scan_hist_correl(yhist, n, key[2], None, arrays[key].ptr, st), "psd_scan_hist_correl")
            else:
                check(lib.psd_scan_hash_dist(e.device_hash(), n, int(e.hash_size), None, arrays[key].ptr, st),
                      "psd_scan_hash_dist")
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

    def totals(self) -> list[CellTotals]:
        """Every cell's counts summed over the videos run with ground truth so far, in grid order."""
        out = []
        for k, params in enumerate(self.grid):
            h, f = self._totals_hard[k], self._totals_fades[k]
            out.append(CellTotals(
                params=params,
                hard={t: EventCounts(int(h[q, 0]), int(h[q, 1]), int(h[q, 2])) for q, t in enumerate(self.tolerances)},
                hard_offset={t: (float(h[q, 3]), int(h[q, 4])) for q, t in enumerate(self.tolerances)},
                fades=EventCounts(int(f[0]), int(f[1]), int(f[2]))))
        return out


__all__ = ["ParameterSweep", "SweepResult", "GroundTruth", "EventCounts", "CellTotals", "PixelGroup", "CellPlan",
           "plan_cell", "pixel_group_of"]
