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

`settings` adds how frames are read and scored (auto_downscale, downscale, crop, frame_skip) as a second axis:
`ParameterSweep(..., settings=[{}, {"frame_skip": 1}, {"crop": (0, 60, 1279, 659)}]).run_clips(videos, gts,
duration="30s")` reads each clip once for every setting (fan_out.py) and evaluates every (setting, cell, clip) with
one psd_clip_cuts_tables and one psd_clip_eval_tables per pass.

`detector_sets` sweeps detectors of any classes, and SceneManagers with several detectors, instead of one class's grid:
`ParameterSweep(detector_sets=[AdaptiveDetector(), [ContentDetector(), ThresholdDetector()], ...]).run_clips(videos,
gts)`.  Each distinct detector configuration runs its automaton once per setting and clip, and psd_clip_union merges
the members' cut lists into every set's list on the device before the evaluator scores it.
"""

from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass, field, replace

import numpy as np

from . import _capi
from ._capi import check
from .detectors._base import EngineDetector, PixelGroup, pixel_group_of
from .device_cuts import automaton_args, flash_filter_frames, histogram_threshold, min_len_frames, scan_metric
from .engine import DeviceBuffer
from .scene_manager import FrameBatches, SceneManager, check_window, shared_engine

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
    detectors: tuple | None = None  # the cell's detectors in a sweep over detector sets; None in a grid sweep

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
        self.end_frames = [end_frame]  # one per setting; `end_frame` is setting 0's
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


class _OneClipResult(SweepResult):
    """`run`'s result when the video went through the clip path (settings or a window): clip 0 of a
    ClipSweepResult, with the accessors of SweepResult."""

    def __init__(self, r: ClipSweepResult):
        self._r = r
        self.tolerances = r.tolerances
        self.end_frames = [r.end_frame(0, setting=s) for s in range(r.n_settings)]
        self.end_frame = self.end_frames[0]
        self.grid_ms = r.grid_ms

    def __len__(self) -> int:
        return len(self._r)

    def cuts(self, k: int) -> list[int]:
        return self._r.cuts(k, 0)

    def raw_count(self, k: int) -> int:
        return self._r.raw_count(k, 0)

    def hard(self, k: int, tol: int) -> tuple[int, int, int]:
        return self._r.hard(k, 0, tol)

    def hard_offset(self, k: int, tol: int) -> tuple[float, int]:
        return self._r.hard_offset(k, 0, tol)

    def fades(self, k: int) -> tuple[int, int, int]:
        return self._r.fades(k, 0)


def _cell_totals(grid, tolerances, th, tf, sets=None) -> list[CellTotals]:
    """CellTotals per cell from summed counts th[cell][tolerance][5] and tf[cell][3], in grid order; `sets` gives
    every cell's detectors in a sweep over detector sets."""
    out = []
    for k, params in enumerate(grid):
        h, f = th[k], tf[k]
        out.append(CellTotals(
            params=params,
            hard={t: EventCounts(int(h[q, 0]), int(h[q, 1]), int(h[q, 2])) for q, t in enumerate(tolerances)},
            hard_offset={t: (float(h[q, 3]), int(h[q, 4])) for q, t in enumerate(tolerances)},
            fades=EventCounts(int(f[0]), int(f[1]), int(f[2])),
            detectors=None if sets is None else sets[k]))
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
    device memory until an accessor reads them; `totals` holds this call's counts summed over its clips.  Cells are
    settings x grid, settings-major: cell k is setting k // n_grid's run of grid cell k % n_grid; `grid` holds every
    cell's params ({**setting, **grid cell}).  In a sweep over detector sets the grid cells are the sets: `grid` holds
    every cell's setting and `sets` its detectors (None in a grid sweep)."""

    def __init__(self, grid, tolerances, passes, where, end_frames, totals_hard, totals_fades, grid_ms,
                 n_grid: int | None = None, upload_bytes: int | None = None, sets=None):
        self.grid = grid
        self.sets = sets
        self.tolerances = tuple(tolerances)
        self._passes = passes        # [_ClipPass]
        self._where = where          # clip -> (pass index, index within the pass)
        self._end = end_frames       # [setting][clip]
        self._n_grid = n_grid or len(grid)
        self._th, self._tf = totals_hard, totals_fades
        self.grid_ms = grid_ms       # scans + cut and eval entries of every pass, host clock ending in syncs
        self.upload_bytes = upload_bytes  # host frame bytes copied to the device (settings path; None otherwise)

    def __len__(self) -> int:
        return len(self.grid)

    @property
    def n_clips(self) -> int:
        return len(self._where)

    @property
    def n_settings(self) -> int:
        return len(self._end)

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

    def end_frame(self, j: int, setting: int = 0) -> int:
        """Clip j's end under setting `setting` as SceneManager.get_scene_list ends it: its last position + 1
        (clip-local frames).  Settings differ when their frame skips read past the window differently."""
        return self._end[setting][j]

    def cuts(self, k: int, j: int) -> list[int]:
        """Cell k's predicted list on clip j, as `SweepResult.cuts` gives it: sorted unique cuts, then the clip's
        end frame; empty when the cell found no cut."""
        ps, t = self._at(k, j)
        m = int(ps.host("n_pred")[t])
        if m <= 0:
            return []
        o = int(ps.host("offsets")[t])
        got = ps.cuts_buf.download((m - 1) * 8, offset=o * 8).view(np.int64).tolist()
        return got + [self._end[k // self._n_grid][j]]

    def raw_count(self, k: int, j: int) -> int:
        """How many cuts cell k's automaton emitted on clip j (before de-duplication); for a set of detectors, the
        length of the union of their cuts."""
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
        return _cell_totals(self.grid, self.tolerances, self._th, self._tf, self.sets)


SETTING_KEYS = ("auto_downscale", "downscale", "crop", "frame_skip")


def _setting_geometry(setting: dict, device: int, batch_size: int) -> SceneManager:
    """A SceneManager configured with one setting's `auto_downscale`, `downscale` and `crop` through its own setters
    (their checks, messages and warnings: `downscale` is ignored while `auto_downscale` is on), whose `_geometry`
    the setting's engines are built with."""
    unknown = sorted(set(setting) - set(SETTING_KEYS))
    if unknown:
        raise TypeError(f"unknown setting key(s) {unknown}: a setting takes {', '.join(SETTING_KEYS)}")
    sm = SceneManager(device=device, batch_size=batch_size)
    if "auto_downscale" in setting:
        sm.auto_downscale = setting["auto_downscale"]
    if "downscale" in setting:
        sm.downscale = setting["downscale"]
    if "crop" in setting:
        sm.crop = setting["crop"]
    skip = setting.get("frame_skip", 0)
    if isinstance(skip, bool) or not isinstance(skip, (int, np.integer)):
        raise TypeError("frame_skip must be an integer")
    if skip < 0:
        raise ValueError("frame_skip must be >= 0")
    return sm


def _detector_set(x) -> tuple:
    """One element of `detector_sets` -> its detectors: one of this package's detectors, or a non-empty list of them,
    configuration only (no stats_manager), as detect_clips takes them."""
    dets = (x,) if isinstance(x, EngineDetector) else tuple(x) if isinstance(x, (list, tuple)) else None
    if dets is None:
        raise TypeError(f"a detector set is a detector or a list of detectors, not {type(x).__name__}")
    if not dets:
        raise ValueError("a detector set is empty")
    for d in dets:
        if not isinstance(d, EngineDetector):
            raise TypeError("ParameterSweep sweeps the detectors of this package")
        if d.stats_manager is not None:
            raise ValueError("a sweep produces no per-frame metrics: detectors must not have a stats_manager")
    return dets


def _length_key(length) -> tuple:
    """A min_scene_len as a key that keeps its meaning: the type decides the unit (an int counts frames, a float is
    seconds, a string either), so 2 and 2.0 are different lengths although they compare equal; a timecode is its frame
    number at its own rate."""
    if hasattr(length, "frame_num") and hasattr(length, "framerate"):
        return ("timecode", int(length.frame_num), float(length.framerate))
    return (type(length).__qualname__, length)


def _describe(detector) -> str:
    """A detector by class and the parameters its automaton runs with."""
    _, a = automaton_args(detector)
    return f"{type(detector).__name__}({', '.join(f'{k}={v!r}' for k, v in a.items())})"


class ParameterSweep:
    """Every cell of `grid` (a list of `detector_cls(**params)` keyword dicts, as the reference harness takes
    them) over each video `run` is given.  `detector_cls` is one of this package's detectors; each cell is
    built by its constructor, so defaults, validation, `luma_only` and the histogram's threshold map are the
    constructor's own.

    `settings` sweeps how the frames are read and scored as well: a list of dicts with the keys `auto_downscale`,
    `downscale`, `crop` (SceneManager's properties) and `frame_skip` (detect_scenes'), each checked as those check
    it.  The cells are settings x grid, settings-major (cell s * len(grid) + g, params {**settings[s], **grid[g]}).
    None means [{}]: one setting, SceneManager's defaults, and the cells of the grid alone.

    `detector_sets` (keyword-only, instead of `detector_cls` and `grid`) sweeps detectors of any classes and their
    combinations: each element is one detector or a non-empty list of detectors, configuration only as `detect_clips`
    takes them, and stands for a SceneManager with those detectors, whose cut list is the sorted union of theirs.  The
    cells are settings x sets, settings-major (cell s * len(detector_sets) + k): `params[cell]` is the setting and
    `sets[cell]` the detectors.  Every distinct detector configuration (a member) runs its automaton once per setting
    and clip, however many sets hold it, and one psd_clip_union per pass merges the members' cuts into every set's
    list.  A set holds at most `_capi.SWEEP_MAX_MEMBERS` distinct configurations."""

    def __init__(self, detector_cls=None, grid=None, tolerances=(0, 1), device: int = 0, batch_size: int = 64,
                 max_cuts_per_cell: int = 4096, settings=None, *, detector_sets=None):
        if detector_sets is not None:
            if detector_cls is not None or grid is not None:
                raise TypeError("ParameterSweep takes detector_cls and grid, or detector_sets, not both")
            self.detector_sets = [_detector_set(x) for x in detector_sets]
            if not self.detector_sets:
                raise ValueError("detector_sets is empty")
            self.grid = None
        elif detector_cls is None and grid is None:
            raise TypeError("ParameterSweep needs detector_cls and grid, or detector_sets")
        else:
            if not (isinstance(detector_cls, type) and issubclass(detector_cls, EngineDetector)):
                raise TypeError("ParameterSweep sweeps the detectors of this package")
            self.grid = [dict(p) for p in grid]
            if not self.grid:
                raise ValueError("the grid has no cells")
            self.detector_sets = None
        self.settings = [{}] if settings is None else [dict(x) for x in settings]
        if not self.settings:
            raise ValueError("settings is empty (None means one setting with SceneManager's defaults)")
        self._geometries = [_setting_geometry(x, int(device), int(batch_size)) for x in self.settings]
        self._frame_skips = [int(x.get("frame_skip", 0)) for x in self.settings]
        self._default_settings = self.settings == [{}]
        if self.grid is not None:
            self.params = [{**x, **g} for x in self.settings for g in self.grid]
            self.sets = None
        else:
            self.params = [dict(x) for x in self.settings for _ in self.detector_sets]
            self.sets = [d for _ in self.settings for d in self.detector_sets]
        tols = tuple(int(t) for t in tolerances)
        if not 1 <= len(tols) <= _capi.SWEEP_MAX_TOLERANCES or any(t < 0 for t in tols) or len(set(tols)) != len(tols):
            raise ValueError(f"tolerances must be 1 to {_capi.SWEEP_MAX_TOLERANCES} distinct non-negative frame counts")
        if int(batch_size) < 1 or int(max_cuts_per_cell) < 1:
            raise ValueError("batch_size and max_cuts_per_cell must be >= 1")
        self.tolerances = tols
        self.device = int(device)
        self.batch_size = int(batch_size)
        self.cap = int(max_cuts_per_cell)
        self.groups: list[PixelGroup] = []
        group_index: dict = {}
        self.cells: list[CellPlan] = []

        def plan(d) -> CellPlan:
            g = pixel_group_of(d)
            gi = group_index.setdefault(g, len(self.groups))
            if gi == len(self.groups):
                self.groups.append(g)
            return plan_cell(d, gi)

        if self.grid is not None:
            self.cells = [plan(detector_cls(**p)) for p in self.grid]
        else:
            # the cells are the members: one automaton per distinct (CellPlan, pixel group); a set names its members
            member_index: dict = {}
            self._member_detectors = []
            self._set_members = []
            for dets in self.detector_sets:
                own = []
                for d in dets:
                    c = plan(d)
                    key = replace(c, min_scene_len=_length_key(c.min_scene_len))
                    if key not in member_index:
                        member_index[key] = len(self.cells)
                        self.cells.append(c)
                        self._member_detectors.append(d)
                    if member_index[key] not in own:
                        own.append(member_index[key])
                if len(own) > _capi.SWEEP_MAX_MEMBERS:
                    raise ValueError(f"a detector set holds {len(own)} distinct detectors, more than "
                                     f"{_capi.SWEEP_MAX_MEMBERS}")
                self._set_members.append(own)
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
        self._totals_hard = np.zeros((len(self.params), len(tols), 5), dtype=np.int64)
        self._totals_fades = np.zeros((len(self.params), 3), dtype=np.int64)
        self.videos = 0

    # -- the whole pass --
    def run(self, video, ground_truth: GroundTruth | None = None, duration=None, end_time=None) -> SweepResult:
        """Decode `video` once, score it with one Engine (SceneManager's default geometry: auto-downscale, no
        crop) that holds every pixel group's kernel size and hash geometry as a slot, then evaluate every cell.
        Without ground truth nothing is scored (every count is against an empty truth) and `totals` is not
        updated.

        With settings other than the default, or a window (`duration` / `end_time`, as detect_scenes takes them),
        the video goes through `run_clips` as its one clip: cell k's results are run_clips' (k, 0), `end_frames`
        holds every setting's end frame and `end_frame` setting 0's.  So does a sweep over detector sets."""
        if self.sets is not None or not self._default_settings or duration is not None or end_time is not None:
            gts = None if ground_truth is None else [ground_truth]
            return _OneClipResult(self._run_clips([video], gts, duration, end_time, "the video"))
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
        if self.sets is not None:
            raise TypeError("run_scored evaluates a grid; a sweep over detector sets runs through run or run_clips")
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
    def run_clips(self, videos, ground_truths=None, duration=None, end_time=None, *, windows=None) -> ClipSweepResult:
        """Every cell over every stream of `videos`: for each (cell, clip), what `run(videos[j], ground_truths[j])`
        gives on a fresh ParameterSweep with this grid, tolerances and batch size; `totals` and `videos` afterwards
        are what a loop of `run` leaves.  Streams are anything `detect_clips` reads (host or CUDA `ArrayVideoStream`s
        of any layout and channel order, reference `VideoStream`s) and may differ in length, frame rate and frame
        size; each is read from its current position and its frame numbers are clip-local.

        With settings, cell (s, g) on clip j is what a fresh SceneManager with setting s's `auto_downscale`,
        `downscale` and `crop` finds with `detector_cls(**grid[g])` in `detect_scenes(videos[j], duration=,
        end_time=, frame_skip=)`: its sorted unique cuts followed by its end position + 1, scored against
        ground_truths[j].  `duration` / `end_time` give every setting and clip the same window, as in
        `detect_clips`.  Each stream is read once for every setting (fan_out.py): afterwards it stands at the end of
        the union of the settings' windows, which a frame skip can put past some settings' own ends.

        The clips are scored as `detect_clips` scores them, pass by pass.  Each pass ends with every setting's
        scans, ONE cut entry (psd_clip_cuts; psd_clip_cuts_tables for settings) for every (cell, clip) automaton and
        ONE eval entry (psd_clip_eval / psd_clip_eval_tables) that scores every (cell, clip, tolerance) against clip
        j's ground truth and sums the counts over the pass's clips on the device; only those sums and the cut total
        come back to the host.

        `ground_truths`: None (every count is against an empty truth and `totals` is not updated), or one
        GroundTruth per video.  ValueError for a length mismatch, a clip without frames, a window detect_scenes
        refuses (its messages) or, before any frame is read, a crop that starts outside some clip's frame (naming
        the clip and the setting); RuntimeError for a (cell, clip) with more than max_cuts_per_cell cuts; `totals`
        only changes when the call returns.

        `windows` (keyword only) gives each clip its own window, as `detect_clips(windows=)` takes it: one entry per
        video, None or a dict with keys among `crop`, `duration`, `end_time` and `frame_skip`, checked as detect_clips
        checks them.  Cell (s, g) on clip j is then what a one-clip ParameterSweep with this grid (or these
        detector_sets) and `settings=[{**settings[s], **w}]` gives on it from `run_clips([videos[j]], [ground_truths[j]],
        duration=, end_time=)`, w being the entry's `crop` and `frame_skip` and the other two its window: counts, cut
        lists, end frames and totals.  A window does not change a clip's ground truth: cuts and fades past the window's
        end are scored against the frames it reads, so those cuts count as missed; give the truth of the window alone to
        score the window alone.  Per setting, clips whose crops and downscale give one scored size share an engine and a
        pass whatever their source sizes, every clip is still read once for every setting, ending at its own window's
        end, and a pass whose clips step differently runs psd_clip_cuts_tables_steps in place of psd_clip_cuts_tables,
        with the same launches.  TypeError, before any frame is read, for `windows` together with `duration` or
        `end_time`, and for a key (`crop`, `frame_skip`) that both some setting and some window set."""
        return self._run_clips(videos, ground_truths, duration, end_time, "clip {}", windows)

    def _window_plan(self, videos, windows) -> tuple:
        """detect_clips' checks of `windows`, then every clip's `clips._ClipWindow` under every setting (windows[j][s]:
        the setting's geometry under the window's crop, the window's frame skip or else the setting's) and the clips'
        own steps, or None when the windows set no frame_skip."""
        from .clips import _clip_windows
        windows = list(windows)
        set_keys = {k for x in self.settings for k in x}
        both = sorted(set_keys & {k for w in windows if isinstance(w, dict) for k in w})
        if both:
            raise TypeError(f"{', '.join(both)} set both by a setting and by a window: a clip takes each from one or "
                            f"the other")
        per_setting = [_clip_windows(videos, windows, g, False) for g in self._geometries]
        skips = any(isinstance(w, dict) and "frame_skip" in w for w in windows)
        plan = [[w if skips else replace(w, frame_skip=f) for w, f in zip(ws, self._frame_skips)]
                for ws in zip(*per_setting)]
        return plan, [int(ws[0].frame_skip) + 1 for ws in plan] if skips else None

    def _run_clips(self, videos, ground_truths, duration, end_time, clip_name: str, windows=None) -> ClipSweepResult:
        from .clips import _Pass, clip_passes
        from .fan_out import settings_passes
        videos = list(videos)
        if ground_truths is None:
            gts = [GroundTruth([])] * len(videos)
        else:
            gts = list(ground_truths)
            if len(gts) != len(videos):
                raise ValueError(f"{len(videos)} videos need as many ground truths, got {len(gts)}")
            if not all(isinstance(g, GroundTruth) for g in gts):
                raise ValueError("every ground truth must be a GroundTruth (GroundTruth([]) for a clip without cuts)")
        if windows is not None and (duration is not None or end_time is not None):
            raise TypeError("run_clips takes windows or duration / end_time, not both")
        check_window(duration, end_time)
        for s, g in enumerate(self._geometries):
            if g._crop is not None:
                x0, y0 = g._crop[:2]
                for i, v in enumerate(videos):
                    fw, fh = v.frame_size
                    if x0 >= fw or y0 >= fh:
                        raise ValueError(f"crop starts outside video boundary of clip {i} ({fw}x{fh}) in setting {s} "
                                         f"({self.settings[s]})")
        plan = clip_steps = None
        if windows is not None:
            plan, clip_steps = self._window_plan(videos, windows)
        fanned = plan is not None or not self._default_settings  # through fan_out.settings_passes
        lib = self._lib = self._lib or _capi.load()
        n_set, n_tol, dev = len(self.settings), len(self.tolerances), self.device
        n_cells = len(self.params)
        n_grid = n_cells // n_set
        max_cuts = self.cap
        if self.sets is not None:
            # the set-cells over the member lists of psd_clip_cuts(_tables): list s * members + i is member i under
            # setting s; a union of members that each keep within the cap keeps within cap x its member count
            n_mem = len(self.cells)
            lists = [[s * n_mem + i for i in own] for s in range(n_set) for own in self._set_members]
            set_table = ((C.c_int32 * (n_cells + 1))(*np.concatenate([[0], np.cumsum([len(x) for x in lists])])),
                         (C.c_int32 * sum(len(x) for x in lists))(*[i for x in lists for i in x]))
            set_of_cell = (C.c_int32 * n_cells)(*[k // n_grid for k in range(n_cells)])
            max_cuts = min(self.cap * max(len(x) for x in self._set_members), 2 ** 31 - 1)
        tols = (C.c_int32 * n_tol)(*self.tolerances)
        th = np.zeros((n_cells, n_tol, 5), dtype=np.int64)
        tf = np.zeros((n_cells, 3), dtype=np.int64)
        passes, where, ends = [], [None] * len(videos), [[0] * len(videos) for _ in range(n_set)]
        grid_ms = 0.0
        counters = {}
        device_pass = _Pass(self.cells, self.groups, dev)
        if not fanned:
            scoring = clip_passes(videos, self.groups, SceneManager(device=dev, batch_size=self.batch_size),
                                  self.batch_size, dev, duration=duration, end_time=end_time)
        else:
            scoring = settings_passes(videos, self.groups, self._geometries, self._frame_skips, self.batch_size, dev,
                                      duration=duration, end_time=end_time, counters=counters, windows=plan)
        steps = [f + 1 for f in self._frame_skips]
        try:
            for engine, holders, done in scoring:
                if not fanned:
                    done = [(index, [r], [m]) for index, r, m in done]
                for index, _rs, ms in done:
                    if not ms[0]:
                        raise ValueError(f"{clip_name.format(index)} has no frames")
                t0 = time.perf_counter()
                if not fanned:
                    pc = device_pass.cuts(engine, holders, [(rs[0], ms[0]) for _, rs, ms in done])
                else:
                    own = () if clip_steps is None else ([clip_steps[i] for i, _, _ in done],)
                    pc = device_pass.cuts_tables(engine, holders, [[(rs[s], ms[s]) for _, rs, ms in done]
                                                                   for s in range(n_set)], steps, *own)
                    engine = engine[0]
                indices = [index for index, _rs, _ms in done]
                members = None
                if self.sets is not None:
                    members = pc
                    try:
                        pc, over = device_pass.union(engine, members, *set_table, self.cap)
                    except BaseException:
                        members.close()
                        raise
                    if over >= 0:
                        self._member_overflow(members, over, indices)
                    if pc.tables is not None:
                        pc.cell_table = set_of_cell
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
                    truth = (gbuf.ptr, gt_cuts, n_gt, gbuf.ptr + (c + 1) * 8, gt_cuts + n_gt * 8, n_fades, tols, n_tol,
                             ws.ptr, ws.nbytes, n_pred.ptr, hard.ptr, fades.ptr, sums.ptr,
                             sums.ptr + n_cells * n_tol * 40, sums.ptr + n_cells * (n_tol * 5 + 3) * 8,
                             engine.compute_stream)
                    if pc.tables is None:
                        check(lib.psd_clip_eval(pc.cuts.ptr, pc.offsets.ptr, n_cells, c, pc.total, max_cuts,
                                                pc.end_frames, *truth), "psd_clip_eval")
                    else:
                        check(lib.psd_clip_eval_tables(pc.cuts.ptr, pc.offsets.ptr, n_cells, c, pc.total, max_cuts,
                                                       pc.tables, n_set, pc.cell_table, *truth), "psd_clip_eval_tables")
                    engine.sync()
                    grid_ms += (time.perf_counter() - t0) * 1e3
                    got = sums.download(sums.nbytes).view(np.int64)
                finally:
                    done_with = (gbuf, ws, sums, pc.table)
                    if members is not None:  # the member lists the unions were merged from
                        done_with += (members.offsets, members.cuts)
                    for b in done_with:
                        b.close()
                over = int(got[-1])
                if over >= 0:
                    k, jj = divmod(over, c)
                    o = pc.offsets.download(16, offset=over * 8).view(np.int64)
                    what = self.grid[k % n_grid] if self.sets is None else list(self.sets[k])
                    where_k = f"({what})" if self._default_settings else \
                        f"({what}) of setting {k // n_grid} ({self.settings[k // n_grid]})"
                    raise RuntimeError(f"cell {k} {where_k} found {int(o[1] - o[0])} cuts in clip "
                                       f"{indices[jj]}, more than max_cuts_per_cell={self.cap}")
                th += got[:n_cells * n_tol * 5].reshape(n_cells, n_tol, 5)
                tf += got[n_cells * n_tol * 5:-1].reshape(n_cells, 3)
                for jj, (index, rs, _ms) in enumerate(done):
                    where[index] = (len(passes), jj)
                    for s in range(n_set):
                        ends[s][index] = rs[s].end.frame_num + 1
                passes.append(_ClipPass(pc, n_tol, n_pred, hard, fades))
        finally:
            scoring.close()
            device_pass.close()
        if ground_truths is not None:
            self._totals_hard += th
            self._totals_fades += tf
            self.videos += len(videos)
        return ClipSweepResult(self.params, self.tolerances, passes, where, ends, th, tf, grid_ms, n_grid=n_grid,
                               upload_bytes=counters.get("uploaded", 0) if fanned else None,
                               sets=self.sets)

    def _member_overflow(self, members, over: int, indices) -> None:
        """Raise for member list `over` of a pass (list * n_clips + clip of psd_clip_cuts' output), which has more than
        max_cuts_per_cell cuts; releases the pass's member lists and clip table."""
        try:
            o = members.offsets.download(16, offset=over * 8).view(np.int64)
        finally:
            members.close()
        i, jj = divmod(over, members.n_clips)
        s, m = divmod(i, len(self.cells))
        raise RuntimeError(f"detector {_describe(self._member_detectors[m])} of setting {s} ({self.settings[s]}) found "
                           f"{int(o[1] - o[0])} cuts in clip {indices[jj]}, more than max_cuts_per_cell={self.cap}")

    def totals(self) -> list[CellTotals]:
        """Every cell's counts summed over the videos and clips run with ground truth so far, in grid order."""
        return _cell_totals(self.params, self.tolerances, self._totals_hard, self._totals_fades, self.sets)


__all__ = ["ParameterSweep", "SweepResult", "ClipSweepResult", "GroundTruth", "EventCounts", "CellTotals",
           "PixelGroup", "CellPlan", "plan_cell", "pixel_group_of"]
