"""`ParameterSweep(detector_sets=...)` without a GPU: the oracle-backed engine scores the frames, and the twins of the
clip kernels and of psd_clip_union (tests/sweep_sets_twin.py) stand in for the library.  Every (setting, set, clip)
must be what `detect_clips` with that setting and the set's detectors gives, scored by tests/sweep_model.py; every
distinct detector runs its automaton once per setting and clip, and every clip is read once per setting."""

from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import pytest

from tests import clip_twin, sweep_model, sweep_sets_twin, sweep_settings_twin
from tests.test_sweep_clips_host import _grids, _truth
from tests.test_sweep_settings_host import CLIPS, _check, _frames, _streams

BATCH = 16
TOLS = (0, 1, 3)
SETTINGS = [{}, {"frame_skip": 2}, {"crop": (4, 2, 50, 30)}, {"auto_downscale": False, "downscale": 2}]
WINDOWS = {"none": {}, "duration": {"duration": 1.1}, "end_time": {"end_time": "00:00:02.2"}}


class CountingLib(sweep_sets_twin.Lib):
    """The twin, recording the number of (cell) automata of every cut entry."""

    def __init__(self):
        super().__init__()
        self.automata = []

    def psd_clip_cuts(self, cells, n_cells, *args):
        self.automata.append(n_cells)
        return super().psd_clip_cuts(cells, n_cells, *args)

    def psd_clip_cuts_tables(self, cells, n_cells, *args):
        self.automata.append(n_cells)
        return super().psd_clip_cuts_tables(cells, n_cells, *args)


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, fan_out, scene_manager, sweep
    lib = CountingLib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", sweep_settings_twin.SettingsEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(fan_out, "PinnedBuffer", clip_twin.PinnedHost)
    for mod in (clips, sweep, fan_out):
        monkeypatch.setattr(mod, "DeviceBuffer", clip_twin.Buffer)
    monkeypatch.setattr(clip_twin, "_ids", itertools.count(1 << 32, 1 << 28))
    sweep_settings_twin.SettingsEngine.layouts = []
    clip_twin.ClipEngine.submissions = []
    sweep_sets_twin.Lib.unsorted_inputs = 0
    return lib


@pytest.fixture(scope="module")
def clip_set():
    out = []
    for i, (n, w, h, fps) in enumerate(CLIPS):
        frames, cuts = _frames(n, 7 * i + 3, w, h)
        out.append((frames, fps, _truth(n, cuts, i)))
    return out


def _one_detector_sets():
    """Every detector of the five classes' grids, each its own set."""
    return [cls(**p) for cls, grid in _grids().values() for p in grid]


def _mixes():
    """Sets of several detectors: content + threshold, adaptive + threshold, hash + histogram with other thresholds
    and bins (the twin engine holds one hash geometry; tests/test_gpu_sweep_sets.py mixes hash sizes), members shared
    by several sets, one configuration twice in a set, and a ThresholdDetector whose |fade_bias| > 1 places its cuts
    out of order."""
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    content = ContentDetector(threshold=12.0, min_scene_len=3)
    adaptive = AdaptiveDetector(adaptive_threshold=1.5, min_scene_len=4, window_width=1)
    dark = ThresholdDetector(threshold=125, min_scene_len=2, add_final_scene=True)
    wide = ThresholdDetector(threshold=122, min_scene_len=1, fade_bias=3.0)
    return [
        [content, dark],
        [adaptive, ThresholdDetector(threshold=125, min_scene_len=2, add_final_scene=True)],  # dark's twin: shared
        [HashDetector(threshold=0.25, min_scene_len=2), HistogramDetector(threshold=0.05, bins=64)],
        [HashDetector(threshold=0.3), HistogramDetector(threshold=0.1, bins=128), content],
        [content, ContentDetector(threshold=12.0, min_scene_len=3)],  # the same configuration twice
        [wide, adaptive],
        [wide],
        dark,
    ]


def _expect(sets, settings, clip_set, window, advance=0):
    """(setting, set, clip) -> (predicted list, end frame, hard counts per tolerance, fade counts), from one detect_clips
    per (setting, set)."""
    from pyscenedetect_b200.clips import detect_clips
    out = {}
    for s, st in enumerate(settings):
        for k, dets in enumerate(sets):
            dets = list(dets) if isinstance(dets, list) else [dets]
            res = detect_clips(_streams(clip_set, advance), dets, batch_size=BATCH, **st, **window)
            for j, r in enumerate(res):
                end = r.end.frame_num + 1
                preds = sweep_model.predicted_list(r.cut_frames, end)
                gt = clip_set[j][2]
                scores = [sweep_model.score(preds, gt.hard_cuts, gt.fades, t) for t in TOLS]
                out[s, k, j] = (preds, end, [x[0] for x in scores], scores[0][1])
    return out


def test_one_detector_sets_of_every_class_equal_per_class_sweeps(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    gts = [gt for _, _, gt in clip_set]
    sets = _one_detector_sets()
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH)
    r = sw.run_clips(_streams(clip_set), gts)
    assert len(r) == len(sets) and r.sets == [(d,) for d in sets] and r.grid == [{}] * len(sets)
    _check(r, _expect(sets, [{}], clip_set, {}), len(sets), len(clip_set))
    k = 0
    for cls, grid in _grids().values():
        one = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH).run_clips(_streams(clip_set), gts)
        for g in range(len(grid)):
            for j in range(len(clip_set)):
                assert r.cuts(k + g, j) == one.cuts(g, j)
                assert [r.hard_offset(k + g, j, t) for t in TOLS] == [one.hard_offset(g, j, t) for t in TOLS]
                assert r.fades(k + g, j) == one.fades(g, j)
            a, b = r.totals()[k + g], one.totals()[g]
            assert (a.hard, a.hard_offset, a.fades) == (b.hard, b.hard_offset, b.fades)
            assert a.detectors == (sets[k + g],) and b.detectors is None
        k += len(grid)
    assert [t.detectors for t in sw.totals()] == [(d,) for d in sets] and sw.videos == len(clip_set)


@pytest.mark.parametrize("window", list(WINDOWS))
def test_mixed_sets_equal_detect_clips_per_setting(twin, clip_set, window):
    from pyscenedetect_b200.sweep import ParameterSweep
    gts = [gt for _, _, gt in clip_set]
    sets = _mixes()
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS)
    r = sw.run_clips(_streams(clip_set), gts, **WINDOWS[window])
    automata, launches = list(twin.automata), dict(twin.launches)
    assert len(r) == len(SETTINGS) * len(sets) and r.n_settings == len(SETTINGS)
    assert r.grid == [s for s in SETTINGS for _ in sets]
    assert r.sets == [tuple(x) if isinstance(x, list) else (x,) for _ in SETTINGS for x in sets]
    want = _expect(sets, SETTINGS, clip_set, WINDOWS[window])
    _check(r, want, len(sets), len(clip_set))
    # the threshold members do cut these clips
    k_dark, k_wide = len(sets) - 1, len(sets) - 2
    assert any(want[0, k_dark, j][0] for j in range(len(clip_set)))
    assert any(want[0, k_wide, j][0] for j in range(len(clip_set)))
    # 8 distinct detectors (the shared and repeated ones once), under every setting: one cut entry per pass
    assert set(automata) == {len(SETTINGS) * 8}
    # per pass (one per frame size): one union count and one union write, one evaluator sequence
    assert launches["psd_clip_union"] == 2 * (3 + 1)
    # over whole clips the |fade_bias| > 1 member emits a list out of order, which the counting call sorts
    assert window != "none" or sweep_sets_twin.Lib.unsorted_inputs > 0
    assert launches["psd_clip_eval_tables"] == 2 * 3


def test_members_run_once_and_launches_do_not_grow(twin, clip_set):
    """An Adaptive grid of 4 crossed with a Threshold grid of 2: 8 cells, 6 automata per (setting, clip).  Launches of
    the union and the evaluator per pass do not depend on the numbers of sets, members or clips, and every clip's
    frames are submitted as a one-set sweep submits them."""
    from pyscenedetect_b200.detectors import AdaptiveDetector, ThresholdDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    gts = [gt for _, _, gt in clip_set]
    ad = [AdaptiveDetector(adaptive_threshold=t, min_scene_len=m) for t in (1.5, 2.5) for m in (2, 6)]
    th = [ThresholdDetector(threshold=t, min_scene_len=2) for t in (120, 135)]
    cross = [[a, t] for a in ad for t in th]
    counts = {}
    for name, sets, settings in (("one", [ad[0]], None), ("cross", cross, None), ("cross2", cross + ad + th, None),
                                 ("one_s", [ad[0]], SETTINGS[:2]), ("cross_s", cross, SETTINGS[:2])):
        twin.launches.clear()
        twin.automata.clear()
        clip_twin.ClipEngine.submissions = []
        r = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH, settings=settings).run_clips(
            _streams(clip_set), gts)
        counts[name] = (dict(twin.launches), list(twin.automata), sum(clip_twin.ClipEngine.submissions),
                        r.upload_bytes)
        if name.startswith("cross"):
            _check(r, _expect(sets, settings or [{}], clip_set, {}), len(sets), len(clip_set))
    # automata per cut entry (an entry runs twice when its first cut buffer was short)
    assert [set(counts[n][1]) for n in ("one", "cross", "cross2", "one_s", "cross_s")] == [{1}, {6}, {6}, {2}, {12}]
    for a, b in (("one", "cross"), ("one", "cross2"), ("one_s", "cross_s")):
        for entry in ("psd_clip_union", "psd_clip_eval", "psd_clip_eval_tables"):
            assert counts[a][0].get(entry) == counts[b][0].get(entry), (a, b, entry)
        assert counts[a][2] == counts[b][2]  # frames submitted to the engines
        assert counts[a][3] == counts[b][3]  # host bytes uploaded (settings path)
    assert counts["one_s"][3] == sum(f.nbytes for f, _, _ in clip_set)
    # fewer clips: the same launches per pass
    twin.launches.clear()
    ParameterSweep(detector_sets=cross, tolerances=TOLS, batch_size=BATCH).run_clips(_streams(clip_set[:2]), gts[:2])
    assert twin.launches["psd_clip_union"] == 3 + 1 and twin.launches["psd_clip_eval"] == 3


def test_run_is_run_clips_of_one_clip(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    sets = _mixes()[:3]
    want = _expect(sets, [{}], clip_set, {})
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH)
    for j, (frames, fps, gt) in enumerate(clip_set):
        r = sw.run(ArrayVideoStream(frames, fps), gt)
        for k in range(len(sets)):
            preds, end, hard, fades = want[0, k, j]
            assert r.end_frame == end and r.cuts(k) == preds and r.fades(k) == fades
            assert [r.hard(k, t) for t in TOLS] == [h[:3] for h in hard]
    assert sw.videos == len(clip_set)
    with pytest.raises(TypeError, match="run_scored evaluates a grid"):
        sw.run_scored([], 30)


def test_split_passes_retry_and_overflow(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    from pyscenedetect_b200.sweep import ParameterSweep
    gts = [gt for _, _, gt in clip_set]
    sets = _mixes()
    window = {"duration": 2.0}
    want = _expect(sets, SETTINGS[:2], clip_set, window, advance=3)
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 20)
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 0)
    twin.launches.clear()
    r = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS[:2]).run_clips(
        _streams(clip_set, advance=3), gts, **window)
    _check(r, want, len(sets), len(clip_set))
    passes = twin.launches["psd_clip_eval_tables"] // 3
    assert passes > 2 and twin.launches["psd_clip_cuts_tables"] > 3 * passes  # retries of the member cut buffer
    assert twin.launches["psd_clip_union"] == 4 * passes
    # one member over the cap: named with its setting and clip; the totals do not change
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH, max_cuts_per_cell=1,
                        settings=[{"frame_skip": 1}, {}])
    with pytest.raises(RuntimeError, match=r"detector (Content|Adaptive|Hash|Histogram|Threshold)Detector\(.*\) of "
                                           r"setting \d \(\{.*\}\) found \d+ cuts in clip \d+, more than "
                                           r"max_cuts_per_cell=1"):
        sw.run_clips(_streams(clip_set), gts)
    assert sw.videos == 0 and all(t.hard[0].matched == 0 for t in sw.totals())
    # a union longer than the cap is fine when each member keeps within it
    pair = _mixes()[0]  # content + threshold: cuts at different frames
    full = ParameterSweep(detector_sets=[pair], tolerances=TOLS, batch_size=BATCH).run_clips(_streams(clip_set), gts)
    one = [ParameterSweep(detector_sets=[d], batch_size=BATCH).run_clips(_streams(clip_set)) for d in pair]
    cap = max(r.raw_count(0, j) for r in one for j in range(len(clip_set)))  # the longest member list in any clip
    assert cap >= 1 and max(full.raw_count(0, j) for j in range(len(clip_set))) > cap
    capped = ParameterSweep(detector_sets=[pair], tolerances=TOLS, batch_size=BATCH,
                            max_cuts_per_cell=cap).run_clips(_streams(clip_set), gts)
    assert [capped.cuts(0, j) for j in range(len(clip_set))] == [full.cuts(0, j) for j in range(len(clip_set))]
    assert [(t.hard, t.fades) for t in capped.totals()] == [(t.hard, t.fades) for t in full.totals()]


def test_grid_sweeps_make_todays_calls(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    sw.run_clips(_streams(clip_set), gts)
    assert set(twin.launches) == {"scan", "psd_clip_fill", "psd_clip_cuts", "psd_clip_eval"}
    assert sw.sets is None and sw.detector_sets is None and all(t.detectors is None for t in sw.totals())
    twin.launches.clear()
    ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS[:2]).run_clips(_streams(clip_set))
    assert set(twin.launches) == {"scan", "psd_clip_fill", "psd_clip_cuts_tables", "psd_clip_eval_tables"}


def test_refusals(twin, clip_set):
    from pyscenedetect_b200 import StatsManager, _capi
    from pyscenedetect_b200.detectors import ContentDetector, HistogramDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    d = ContentDetector()
    with pytest.raises(TypeError, match="not both"):
        ParameterSweep(ContentDetector, [{}], detector_sets=[d])
    with pytest.raises(TypeError, match="not both"):
        ParameterSweep(grid=[{}], detector_sets=[d])
    with pytest.raises(TypeError, match="needs detector_cls and grid, or detector_sets"):
        ParameterSweep()
    with pytest.raises(TypeError):
        ParameterSweep(ContentDetector, None, 0, 0, 64, 4096, None, [d])  # detector_sets is keyword-only
    with pytest.raises(ValueError, match="detector_sets is empty"):
        ParameterSweep(detector_sets=[])
    with pytest.raises(ValueError, match="a detector set is empty"):
        ParameterSweep(detector_sets=[d, []])
    with pytest.raises(TypeError, match="sweeps the detectors of this package"):
        ParameterSweep(detector_sets=[[d, object()]])
    with pytest.raises(TypeError, match="a detector set is a detector or a list of detectors"):
        ParameterSweep(detector_sets=[ContentDetector])
    with pytest.raises(TypeError, match="a detector set is a detector or a list of detectors"):
        ParameterSweep(detector_sets=["content"])
    stats = ContentDetector()
    stats.stats_manager = StatsManager()
    with pytest.raises(ValueError, match="must not have a stats_manager"):
        ParameterSweep(detector_sets=[[d, stats]])
    many = [HistogramDetector(threshold=0.01 * (i + 1)) for i in range(_capi.SWEEP_MAX_MEMBERS + 1)]
    with pytest.raises(ValueError, match=f"holds {_capi.SWEEP_MAX_MEMBERS + 1} distinct detectors, more than "
                                         f"{_capi.SWEEP_MAX_MEMBERS}"):
        ParameterSweep(detector_sets=[d, many])
    ParameterSweep(detector_sets=[many[:-1] + many[:3]])  # repeats are one member each
    with pytest.raises(ValueError, match="settings is empty"):
        ParameterSweep(detector_sets=[d], settings=[])
    with pytest.raises(TypeError, match="unknown setting key"):
        ParameterSweep(detector_sets=[d], settings=[{"threshold": 1}])
    streams = _streams(clip_set)
    with pytest.raises(ValueError, match=r"crop starts outside video boundary of clip 2 \(48x40\) in setting 0"):
        ParameterSweep(detector_sets=[d], settings=[{"crop": (50, 0, 60, 30)}]).run_clips(streams)


def test_union_twin_matches_a_direct_merge():
    rng = np.random.default_rng(5)
    n_lists, n_clips = 5, 3
    lists = [sorted(rng.choice(50, size=int(rng.integers(0, 6)), replace=False).tolist()) for _ in range(15)]
    lists[4] = [9, 3, 9, 1]  # unsorted, with a repeat
    cell_offsets, cell_lists = [0, 1, 3, 6], [2, 0, 4, 1, 1, 3]
    got = sweep_sets_twin.union_lists([sorted(set(x)) for x in lists], n_clips, cell_offsets, cell_lists, 3)
    assert got[0 * 3 + 1] == sorted(set(lists[2 * 3 + 1]))
    assert got[1 * 3 + 1] == sorted(set(lists[0 * 3 + 1]) | set(lists[4 * 3 + 1]))
    assert got[2 * 3 + 2] == sorted(set(lists[1 * 3 + 2]) | set(lists[3 * 3 + 2]))


def test_c_abi_rejects_bad_cell_tables_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    p = 4096
    i32 = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731

    def union(offsets, lists, n_cells, n_lists=3, out_cap=0, out=None, unique=p):
        return lib.psd_clip_union(p, p, n_lists, 2, 10, 16, offsets, lists, n_cells, unique, out, out_cap, p, p, None)

    assert union(i32(0, 1, 3), i32(0, 3, 1), 2) == _capi.PSD_ERR_INVALID
    assert b"psd_clip_union: cell 1 names list 3 of 3" in lib.psd_last_error()
    assert union(i32(0, 1, 3), i32(0, -1, 1), 2) == _capi.PSD_ERR_INVALID
    assert b"cell 1 names list -1 of 3" in lib.psd_last_error()
    assert union(i32(0, 1, 1), i32(0), 2) == _capi.PSD_ERR_INVALID
    assert b"psd_clip_union: cell 1 has 0 lists, not 1 to 16" in lib.psd_last_error()
    n = _capi.SWEEP_MAX_MEMBERS + 1
    assert union(i32(0, n), i32(*([0] * n)), 1) == _capi.PSD_ERR_INVALID
    assert b"cell 0 has 17 lists, not 1 to 16" in lib.psd_last_error()
    assert union(i32(1, 2), i32(0, 0), 1) == _capi.PSD_ERR_INVALID
    assert b"cell_offsets[0] is 1, not 0" in lib.psd_last_error()
    assert union(None, None, 1) == _capi.PSD_ERR_INVALID
    assert b"no cell table" in lib.psd_last_error()
    assert union(i32(0, 1), i32(0), 1, out_cap=8) == _capi.PSD_ERR_INVALID
    assert b"no out_cuts array" in lib.psd_last_error()
    assert union(i32(0, 1), i32(0), 1, unique=None) == _capi.PSD_ERR_INVALID
    assert b"no unique workspace" in lib.psd_last_error()
    assert lib.psd_clip_union(p, p, 3, 2, 10, -1, i32(0, 1), i32(0), 1, p, None, 0, p, p, None) == \
        _capi.PSD_ERR_INVALID
    assert b"max_cuts must be 0 to" in lib.psd_last_error()


def test_union_kernels_do_not_spill():
    import os
    import re
    import shutil
    import subprocess
    from pyscenedetect_b200 import _capi
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([tool, "-res-usage", _capi.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    pat = r"Function (\S*clip_union\S*):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)"
    found = {fn: (stack, local) for fn, stack, local in re.findall(pat, out)}
    assert len(found) == 3, out[:2000]  # the sort, the count and the writing pass
    assert all(v == ("0", "0") for v in found.values()), found


def test_min_scene_len_in_frames_and_in_seconds_are_different_members(twin, clip_set):
    """2 (frames) and 2.0 (seconds) compare equal but are different lengths: each is its own member, and each set gives
    what detect_clips gives with its own detector."""
    from pyscenedetect_b200.detectors import ContentDetector, HashDetector, ThresholdDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    gts = [gt for _, _, gt in clip_set]
    sets = [[HashDetector(threshold=0.2, min_scene_len=2)], [HashDetector(threshold=0.2, min_scene_len=2.0)],
            [ContentDetector(threshold=12.0, min_scene_len=1)], [ContentDetector(threshold=12.0, min_scene_len=1.0)],
            [ThresholdDetector(threshold=125, min_scene_len=1)], [ThresholdDetector(threshold=125, min_scene_len=1.0)],
            [HashDetector(threshold=0.2, min_scene_len=2), HashDetector(threshold=0.2, min_scene_len=2.0)]]
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH)
    assert len(sw.cells) == 6
    r = sw.run_clips(_streams(clip_set), gts)
    want = _expect(sets, [{}], clip_set, {})
    _check(r, want, len(sets), len(clip_set))
    # the lengths do change the cuts here, so a shared member would have given one set the other's
    for a in (0, 2, 4):
        assert any(want[0, a, j][0] != want[0, a + 1, j][0] for j in range(len(clip_set))), a
