"""`ParameterSweep.run_clips(windows=...)` without a GPU: the oracle-backed engine scores the frames and the twins of
the clip kernels (tests/sweep_windows_twin.py adds psd_clip_cuts_tables_steps) stand in for the library.  Every
(setting, cell, clip) must be what a one-clip sweep with the setting and the clip's window gives: its crop and
frame_skip added to the setting, its duration / end_time as run_clips' window."""

from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import pytest

from tests import clip_steps_twin, clip_twin, clip_window_cases, sweep_settings_twin, sweep_windows_twin
from tests.test_sweep_clips_host import _grids, _truth
from tests.test_sweep_sets_host import _mixes
from tests.test_sweep_settings_host import CLIPS, _frames, _streams

BATCH = 16
TOLS = (0, 1, 3)
# CLIPS: (1, 64x36), (40, 64x36), (3, 48x40), (90, 64x36), (17, 48x40), (2, 64x36), (61, 48x40).  The windows crop
# clips 1, 2 and 4 to 40x30 from both source sizes, clip 6 to a size of its own; durations and end times as int
# (frames), float (seconds) and str; frame skips 0 to 3.
CROPS_AND_SKIPS = [None, {"crop": (4, 2, 43, 31)}, {"crop": (0, 0, 39, 29), "frame_skip": 2, "duration": 1.1},
                   {"frame_skip": 1, "end_time": "00:00:02.200"}, {"crop": (4, 2, 43, 31), "frame_skip": 3,
                                                                   "duration": 20},
                   {"end_time": 1}, {"crop": (8, 4, 40, 39), "frame_skip": 0, "duration": "00:00:01.500"}]
ENDS_ONLY = [None, {"duration": 1.1}, {"end_time": "00:00:02.200"}, {"duration": 30}, None, {"end_time": 2},
             {"duration": "00:00:01.500"}]
CASES = {
    # the windows set crop and frame_skip: the settings may only scale
    "crops_and_skips": ([{}, {"auto_downscale": False, "downscale": 2}], CROPS_AND_SKIPS),
    # the windows set duration / end_time only: the settings crop and skip
    "ends_only": ([{}, {"frame_skip": 2}, {"crop": (4, 2, 50, 30)}, {"auto_downscale": False, "downscale": 2}],
                  ENDS_ONLY),
}


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, fan_out, scene_manager, sweep
    lib = sweep_windows_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", sweep_settings_twin.SettingsEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(fan_out, "PinnedBuffer", clip_twin.PinnedHost)
    for mod in (clips, sweep, fan_out):
        monkeypatch.setattr(mod, "DeviceBuffer", clip_twin.Buffer)
    monkeypatch.setattr(clip_twin, "_ids", itertools.count(1 << 32, 1 << 28))
    sweep_settings_twin.SettingsEngine.layouts = []
    return lib


@pytest.fixture(scope="module")
def clip_set():
    out = []
    for i, (n, w, h, fps) in enumerate(CLIPS):
        frames, cuts = _frames(n, 7 * i + 3, w, h)
        # the truth keeps the cuts and fades past every window's end
        out.append((frames, fps, _truth(n, cuts, i)))
    return out


def _make(kind, settings, sets=None):
    from pyscenedetect_b200.sweep import ParameterSweep
    if sets is not None:
        return ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=BATCH, settings=settings)
    cls, grid = _grids()[kind]
    return ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=settings)


def _one_clip(kind, settings, sets, clip_set, windows, s, j, read_only=False):
    """The contract's oracle: a one-clip sweep of clip j with settings[s] and the window's crop and frame_skip."""
    w = windows[j] or {}
    sw = _make(kind, [{**settings[s], **{k: v for k, v in w.items() if k in ("crop", "frame_skip")}}], sets)
    r = sw.run_clips(_streams([clip_set[j]], read_only=read_only), [clip_set[j][2]],
                     **{k: v for k, v in w.items() if k in ("duration", "end_time")})
    return sw, r


def _check(kind, settings, sets, clip_set, windows, r, sw):
    n_cells = len(r) // len(settings)
    th = np.zeros((len(r), len(TOLS), 5), np.int64)
    tf = np.zeros((len(r), 3), np.int64)
    for s in range(len(settings)):
        for j in range(len(clip_set)):
            one_sw, one = _one_clip(kind, settings, sets, clip_set, windows, s, j)
            assert r.end_frame(j, setting=s) == one.end_frame(0), (s, j)
            for g in range(n_cells):
                k = s * n_cells + g
                assert r.cuts(k, j) == one.cuts(g, 0), (s, g, j)
                assert r.raw_count(k, j) == one.raw_count(g, 0), (s, g, j)
                assert r.fades(k, j) == one.fades(g, 0), (s, g, j)
                for t in TOLS:
                    assert r.hard(k, j, t) == one.hard(g, 0, t), (s, g, j, t)
                    assert r.hard_offset(k, j, t) == one.hard_offset(g, 0, t), (s, g, j, t)
            for g, tot in enumerate(one_sw.totals()):
                k = s * n_cells + g
                for q, t in enumerate(TOLS):
                    e = tot.hard[t]
                    th[k, q] += (e.matched, e.false_positives, e.missed, int(tot.hard_offset[t][0]), tot.hard_offset[t][1])
                tf[k] += (tot.fades.matched, tot.fades.false_positives, tot.fades.missed)
    for k, tot in enumerate(r.totals()):
        for q, t in enumerate(TOLS):
            e = tot.hard[t]
            assert (e.matched, e.false_positives, e.missed) == tuple(th[k, q, :3])
            assert tot.hard_offset[t] == (float(th[k, q, 3]), int(th[k, q, 4]))
        assert (tot.fades.matched, tot.fades.false_positives, tot.fades.missed) == tuple(tf[k])
    assert [(t.hard, t.fades) for t in sw.totals()] == [(t.hard, t.fades) for t in r.totals()]
    assert sw.videos == len(clip_set)


@pytest.mark.parametrize("kind", ["content", "adaptive", "threshold", "histogram", "hash", "sets"])
@pytest.mark.parametrize("case", list(CASES))
def test_windows_equal_one_clip_sweeps(twin, clip_set, kind, case):
    settings, windows = CASES[case]
    sets = _mixes() if kind == "sets" else None
    sw = _make(kind, settings, sets)
    r = sw.run_clips(_streams(clip_set), [gt for _, _, gt in clip_set], windows=windows)
    assert r.n_clips == len(clip_set) and r.n_settings == len(settings)
    assert [t.params for t in r.totals()] == sw.params
    # one evaluator per pass, whatever the windows: the crops give three groups, the source sizes two
    passes = 3 if case == "crops_and_skips" else 2
    assert twin.launches["psd_clip_eval_tables"] == 3 * passes
    cut_calls = twin.launches.get("psd_clip_cuts_tables", 0) + twin.launches.get("psd_clip_cuts_tables_steps", 0)
    assert 3 * passes <= cut_calls <= 2 * 3 * passes
    assert ("psd_clip_cuts_tables_steps" in twin.launches) == (case == "crops_and_skips")
    assert "psd_clip_cuts" not in twin.launches and "psd_clip_eval" not in twin.launches
    if kind == "sets":
        assert twin.launches["psd_clip_union"] == 4 * passes
    # the synthetic clips have no fades, so ThresholdDetector finds nothing in them
    assert kind == "threshold" or any(r.cuts(k, j) for k in range(len(r)) for j in range(len(clip_set)))
    _check(kind, settings, sets, clip_set, windows, r, sw)


def test_read_only_streams_split_passes_and_tiny_cut_buffer(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    settings, windows = CASES["crops_and_skips"]
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 20)
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 0)
    sw = _make("content", settings)
    streams = _streams(clip_set, read_only=True)
    r = sw.run_clips(streams, [gt for _, _, gt in clip_set], windows=windows)
    assert twin.launches["psd_clip_eval_tables"] > 3 * 3
    _check("content", settings, None, clip_set, windows, r, sw)
    # each stream was read once, to the end of its own window: where a one-clip sweep leaves it
    for j, v in enumerate(streams):
        own = _streams([clip_set[j]], read_only=True)[0]
        w = windows[j] or {}
        _make("content", [{k: x for k, x in w.items() if k in ("crop", "frame_skip")}]).run_clips(
            [own], **{k: x for k, x in w.items() if k in ("duration", "end_time")})
        assert v.reads == own.reads and v.decodes == own.decodes and v.frame_number == own.frame_number, j


def test_crops_share_engines_across_source_sizes(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import scene_manager
    made = []

    class Recording(sweep_settings_twin.SettingsEngine):
        def __init__(self, w, h, *args, **kw):
            made.append((w, h))
            super().__init__(w, h, *args, **kw)

    monkeypatch.setattr(scene_manager, "Engine", Recording)
    settings, windows = CASES["crops_and_skips"]
    r = _make("hash", settings).run_clips(_streams(clip_set), windows=windows)
    # per setting: 64x36 (clips 0, 3, 5), 40x30 (clips 1, 2, 4 from both source sizes), 33x36 (clip 6)
    assert sorted(made) == sorted([(64, 36), (40, 30), (33, 36)] * 2)
    # host frames are cropped as they are copied: every uploaded frame is a cropped one
    rows = {layout[1] for _n, layout in sweep_settings_twin.SettingsEngine.layouts}
    assert rows == {64 * 3, 40 * 3, 33 * 3} and r.upload_bytes > 0


def test_no_windows_and_empty_windows(twin, clip_set):
    gts = [gt for _, _, gt in clip_set]
    for settings in ([{}], CASES["ends_only"][0]):
        plain = _make("adaptive", settings).run_clips(_streams(clip_set), gts)
        twin.launches.clear()
        empty = _make("adaptive", settings).run_clips(_streams(clip_set), gts, windows=[None, {}] * 3 + [None])
        assert "psd_clip_cuts_tables_steps" not in twin.launches
        for k in range(len(plain)):
            for j in range(len(clip_set)):
                assert empty.cuts(k, j) == plain.cuts(k, j) and empty.hard(k, j, 1) == plain.hard(k, j, 1)
        assert [(t.hard, t.fades) for t in empty.totals()] == [(t.hard, t.fades) for t in plain.totals()]


def test_refusals_before_any_frame_is_read(twin, clip_set):
    gts = [gt for _, _, gt in clip_set]
    n = len(clip_set)

    def refused(exc, match, settings, windows, **kw):
        sw = _make("content", settings)
        streams = _streams(clip_set, read_only=True)
        with pytest.raises(exc, match=match):
            sw.run_clips(streams, gts, windows=windows, **kw)
        assert all(v.reads == [] for v in streams) and sw.videos == 0

    refused(TypeError, "crop set both by a setting and by a window", [{}, {"crop": (0, 0, 9, 9)}],
            [None] * (n - 1) + [{"crop": (1, 1, 5, 5)}])
    refused(TypeError, "frame_skip set both by a setting and by a window", [{"frame_skip": 1}],
            [{"frame_skip": 0}] + [None] * (n - 1))
    refused(TypeError, "run_clips takes windows or duration / end_time, not both", [{}], [None] * n, duration=2)
    refused(TypeError, "run_clips takes windows or duration / end_time, not both", [{}], [None] * n, end_time=2)
    refused(ValueError, f"windows has {n - 1} entries for {n} videos", [{}], [None] * (n - 1))
    refused(TypeError, "window 2 must be None or a dict, not tuple", [{}], [None, None, (1, 2)] + [None] * (n - 3))
    refused(TypeError, "window 0 has an unknown key 'start_time'", [{}], [{"start_time": 1}] + [None] * (n - 1))
    refused(ValueError, "duration and end_time cannot be set at the same time!", [{}],
            [{"duration": 1, "end_time": 2}] + [None] * (n - 1))
    refused(ValueError, "duration must be greater than or equal to 0!", [{}], [{"duration": -1}] + [None] * (n - 1))
    refused(TypeError, "crop region must be tuple of 4 ints", [{}], [{"crop": (1, 2, 3)}] + [None] * (n - 1))
    refused(ValueError, r"crop starts outside video boundary of clip 2 \(48x40\)", [{}],
            [None, None, {"crop": (50, 0, 60, 30)}] + [None] * (n - 3))
    refused(ValueError, r"crop starts outside video boundary of clip 2 \(48x40\) in setting 1",
            [{}, {"crop": (50, 0, 60, 30)}], [{"duration": 1}] * n)


# -- the twin of psd_clip_cuts_tables_steps --------------------------------------------------------------------------
CAP = 1 << 17


def _array_of(buf, n):
    return buf.data[:8 * n].view(np.int64).copy()


def test_tables_steps_twin_is_the_steps_twin_per_table_and_the_tables_twin_for_equal_steps():
    """psd_clip_cuts_tables_steps with one table is psd_clip_cuts_steps (twins); with every step of a table equal to s
    it is psd_clip_cuts_tables with that table's frame_step = s; with two tables, each cell over its own."""
    from pyscenedetect_b200 import _capi
    lib = sweep_windows_twin.Lib()
    Buf = clip_twin.Buffer
    for gi, (kind, _w, sizes, metric, metric2, params) in enumerate(clip_window_cases.groups()):
        c = len(sizes)
        mbuf = Buf(metric.nbytes)
        mbuf.upload(metric)
        m2 = None
        if metric2 is not None:
            m2 = Buf(metric2.nbytes)
            m2.upload(metric2)
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, mbuf.ptr, m2.ptr if m2 else None, c, gi)
        mfb = Buf(mf.nbytes)
        mfb.upload(mf)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        rng = np.random.default_rng(gi)
        steps = rng.integers(1, 5, c).astype(np.int64)
        first, end = clip_window_cases.first_and_end(sizes, int(steps.max()), gi)
        tabs = []
        for st in (steps, np.full(c, 3, np.int64)):
            t = Buf(8 * (4 * c + 1))
            t.upload(np.concatenate([off, first, end, st]).astype(np.int64))
            tabs.append((t, st))

        def steps_table(t):
            return _capi.PsdClipStepsTable(t.ptr, t.ptr + 8 * (c + 1), t.ptr + 8 * (2 * c + 1), t.ptr + 8 * (3 * c + 1))

        def lists(o, cuts, m):
            return [cuts.data[8 * o[i]:8 * o[i + 1]].view(np.int64).tolist() for i in range(m)]

        for t, st in tabs:
            # one table: psd_clip_cuts_steps's twin over the same steps (a HOST array there)
            o1, c1 = Buf(8 * (k * c + 1)), Buf(8 * CAP)
            lib.psd_clip_cuts_tables_steps(cells, k, (_capi.PsdClipStepsTable * 1)(steps_table(t)), 1, None, c,
                                           mfb.ptr, c1.ptr, CAP, o1.ptr, None)
            o2, c2 = Buf(8 * (k * c + 1)), Buf(8 * CAP)
            lib.psd_clip_cuts_steps(cells, k, t.ptr, t.ptr + 8 * (c + 1), c, mfb.ptr, c2.ptr, CAP, o2.ptr,
                                    (C.c_int64 * c)(*st.tolist()), t.ptr + 8 * (2 * c + 1), None)
            a, b = _array_of(o1, k * c + 1), _array_of(o2, k * c + 1)
            assert (a == b).all() and a[-1] > 0
            assert lists(a, c1, k * c) == lists(b, c2, k * c)
        # equal steps: psd_clip_cuts_tables with frame_step 3
        t, _ = tabs[1]
        o1, c1 = Buf(8 * (k * c + 1)), Buf(8 * CAP)
        lib.psd_clip_cuts_tables_steps(cells, k, (_capi.PsdClipStepsTable * 1)(steps_table(t)), 1, None, c, mfb.ptr,
                                       c1.ptr, CAP, o1.ptr, None)
        o2, c2 = Buf(8 * (k * c + 1)), Buf(8 * CAP)
        plain = _capi.PsdClipTable(t.ptr, t.ptr + 8 * (c + 1), t.ptr + 8 * (2 * c + 1), 3)
        lib.psd_clip_cuts_tables(cells, k, (_capi.PsdClipTable * 1)(plain), 1, None, c, mfb.ptr, c2.ptr, CAP, o2.ptr,
                                 None)
        a, b = _array_of(o1, k * c + 1), _array_of(o2, k * c + 1)
        assert (a == b).all() and lists(a, c1, k * c) == lists(b, c2, k * c)
        # two tables: cells 0 .. k-1 over table 1, then the same cells over table 0
        both = (_capi.PsdSweepCell * (2 * k))(*(list(cells) + list(cells)))
        mf2 = Buf(2 * mf.nbytes)
        mf2.upload(np.concatenate([mf, mf]))
        o, cuts = Buf(8 * (2 * k * c + 1)), Buf(16 * CAP)
        lib.psd_clip_cuts_tables_steps(both, 2 * k, (_capi.PsdClipStepsTable * 2)(*[steps_table(t) for t, _ in tabs]),
                                       2, (C.c_int32 * (2 * k))(*([1] * k + [0] * k)), c, mf2.ptr, cuts.ptr, 2 * CAP,
                                       o.ptr, None)
        got = lists(_array_of(o, 2 * k * c + 1), cuts, 2 * k * c)
        for half, (t, st) in ((0, tabs[1]), (1, tabs[0])):
            want = clip_steps_twin.clip_cut_lists_steps(cells, k, off, first, c, mf, st, end)
            assert got[half * k * c:(half + 1) * k * c] == want


def test_c_abi_rejects_bad_steps_tables_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    p = 4096
    cells = (_capi.PsdSweepCell * 2)(*[_capi.PsdSweepCell(kind=_capi.SWEEP_HASH, metric=p, threshold=0.5)] * 2)
    good = (_capi.PsdClipStepsTable * 2)(_capi.PsdClipStepsTable(p, p, p, p), _capi.PsdClipStepsTable(p, p, p, p))

    def cuts(tables=good, n_tables=2, cell_table=(C.c_int32 * 2)(0, 1)):
        return lib.psd_clip_cuts_tables_steps(cells, 2, tables, n_tables, cell_table, 3, p, p, 16, p, None)

    assert cuts(tables=None) == _capi.PSD_ERR_INVALID
    assert b"psd_clip_cuts_tables_steps: no clip table" in lib.psd_last_error()
    assert cuts(n_tables=0) == _capi.PSD_ERR_INVALID
    assert cuts(cell_table=(C.c_int32 * 2)(0, 2)) == _capi.PSD_ERR_INVALID
    assert b"cell 1 names table 2 of 2" in lib.psd_last_error()
    no_steps = (_capi.PsdClipStepsTable * 2)(_capi.PsdClipStepsTable(p, p, p, p), _capi.PsdClipStepsTable(p, p, p, None))
    assert cuts(tables=no_steps) == _capi.PSD_ERR_INVALID
    assert b"table 1 has no frame_step array" in lib.psd_last_error()
    no_first = (_capi.PsdClipStepsTable * 2)(_capi.PsdClipStepsTable(p, None, p, p), _capi.PsdClipStepsTable(p, p, p, p))
    assert cuts(tables=no_first) == _capi.PSD_ERR_INVALID
    assert b"no clip first frames" in lib.psd_last_error()
