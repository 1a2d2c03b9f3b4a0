"""`ParameterSweep` with `settings` (auto_downscale, downscale, crop, frame_skip) and a window, without a GPU: the
oracle-backed engine scores the frames (tests/sweep_settings_twin.py adds `submit_layout` from twin device memory),
and the twins of psd_clip_cuts_tables / psd_clip_eval_tables stand in for the library.  Every (setting, cell, clip)
must be what `detect_clips` with that setting and the cell's detector gives, scored by tests/sweep_model.py; each
clip must be read once for all settings."""

from __future__ import annotations

import ctypes as C
import itertools
import logging
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_twin, clip_window_cases, sweep_clip_twin, sweep_model, sweep_settings_twin
from tests.test_sweep_clips_host import _grids, _truth

BATCH = 16
TOLS = (0, 1, 3)
SETTINGS = [{}, {"frame_skip": 1}, {"frame_skip": 2}, {"frame_skip": 5}, {"auto_downscale": False, "downscale": 2},
            {"crop": (4, 2, 50, 30)}, {"crop": (60, 33, 1, 3), "frame_skip": 2}]
# (frames, width, height, rate): sizes, rates and lengths differ; one-frame clips and clips shorter than a step
CLIPS = [(1, 64, 36, 25), (40, 64, 36, Fraction(30000, 1001)), (3, 48, 40, 24), (90, 64, 36, 25), (17, 48, 40, 30),
         (2, 64, 36, 25), (61, 48, 40, Fraction(24000, 1001))]


def _frames(n, seed, w, h):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    plan = ScenePlan(n, seed=seed, min_len=2 if n < 100 else 36, max_len=9 if n < 100 else 60)
    return render_frames(plan.params, w, h), [int(c) for c in plan.cut_frames]


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, fan_out, scene_manager, sweep
    lib = sweep_settings_twin.Lib()
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
        out.append((frames, fps, _truth(n, cuts, i)))
    return out


class ReadOnly:
    """An ArrayVideoStream without read_batch, counting every read and decode by frame number."""

    def __init__(self, frames, fps):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._v = ArrayVideoStream(frames, fps)
        self.reads, self.decodes = [], []

    def __getattr__(self, name):
        if name == "read_batch":
            raise AttributeError(name)
        return getattr(self._v, name)

    def __dlpack_device__(self):
        return self._v.__dlpack_device__()

    def read(self, decode: bool = True):
        n = self._v.frame_number
        got = self._v.read(decode)
        if got is not False:
            self.reads.append(n)
            if decode:
                self.decodes.append(n)
        return got


def _streams(clip_set, advance=0, read_only=False):
    from pyscenedetect_b200.video import ArrayVideoStream
    out = []
    for frames, fps, _ in clip_set:
        v = ReadOnly(frames, fps) if read_only else ArrayVideoStream(frames, fps)
        for _ in range(min(advance, len(frames) - 1)):
            v.read()
        out.append(v)
    return out


def _expect(cls, grid, settings, clip_set, window, advance=0, read_only=False):
    """(setting, cell, clip) -> (predicted list, end frame, hard counts per tolerance, fade counts), from one
    detect_clips per (setting, cell)."""
    from pyscenedetect_b200.clips import detect_clips
    out = {}
    for s, st in enumerate(settings):
        for g, params in enumerate(grid):
            res = detect_clips(_streams(clip_set, advance, read_only), [cls(**params)], batch_size=BATCH, **st,
                               **window)
            for j, r in enumerate(res):
                end = r.end.frame_num + 1
                preds = sweep_model.predicted_list(r.cut_frames, end)
                gt = clip_set[j][2]
                scores = [sweep_model.score(preds, gt.hard_cuts, gt.fades, t) for t in TOLS]
                out[s, g, j] = (preds, end, [x[0] for x in scores], scores[0][1])
    return out


def _check(r, want, n_grid, n_clips):
    th = np.zeros((len(r), len(TOLS), 5), np.int64)
    tf = np.zeros((len(r), 3), np.int64)
    for (s, g, j), (preds, end, hard, fades) in want.items():
        k = s * n_grid + g
        assert r.end_frame(j, setting=s) == end, (s, j)
        assert r.cuts(k, j) == preds, (s, g, j)
        for q, t in enumerate(TOLS):
            assert r.hard(k, j, t) == hard[q][:3], (s, g, j, t)
            assert r.hard_offset(k, j, t) == (float(hard[q][3]), hard[q][4])
            th[k, q] += hard[q]
        assert r.fades(k, j) == fades
        tf[k] += fades
    for k, tot in enumerate(r.totals()):
        for q, t in enumerate(TOLS):
            e = tot.hard[t]
            assert (e.matched, e.false_positives, e.missed) == tuple(th[k, q, :3])
            assert tot.hard_offset[t] == (float(th[k, q, 3]), int(th[k, q, 4]))
        assert (tot.fades.matched, tot.fades.false_positives, tot.fades.missed) == tuple(tf[k])


WINDOWS = {"none": {}, "duration": {"duration": 1.1}, "end_time": {"end_time": "00:00:02.2"}}


@pytest.mark.parametrize("kind", ["content", "adaptive", "threshold", "histogram", "hash"])
@pytest.mark.parametrize("window", list(WINDOWS))
def test_run_clips_equals_detect_clips_per_setting(twin, clip_set, kind, window):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()[kind]
    gts = [gt for _, _, gt in clip_set]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS)
    r = sw.run_clips(_streams(clip_set), gts, **WINDOWS[window])
    assert len(r) == len(SETTINGS) * len(grid) and r.n_clips == len(clip_set) and r.n_settings == len(SETTINGS)
    # one pass per frame size (two here): one evaluator sequence for every setting, cell and clip, and one automaton
    # sequence (two when the first cut buffer was short)
    assert twin.launches["psd_clip_eval_tables"] == 2 * 3
    assert twin.launches["psd_clip_eval_tables"] <= twin.launches["psd_clip_cuts_tables"] <= 2 * 2 * 3
    assert "psd_clip_cuts" not in twin.launches and "psd_clip_eval" not in twin.launches
    want = _expect(cls, grid, SETTINGS, clip_set, WINDOWS[window])
    # the synthetic clips have no fades, so ThresholdDetector finds nothing in them
    assert kind == "threshold" or any(w[0] for w in want.values()), "the clips must have cuts to compare"
    _check(r, want, len(grid), len(clip_set))
    assert [t.params for t in r.totals()] == [{**s, **g} for s in SETTINGS for g in grid]
    assert sw.videos == len(clip_set)
    assert [(t.hard, t.fades) for t in sw.totals()] == [(t.hard, t.fades) for t in r.totals()]


def test_advanced_read_only_streams_split_passes_and_tiny_cut_buffer(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]
    window = {"duration": 2.0}
    want = _expect(cls, grid, SETTINGS, clip_set, window, advance=3, read_only=True)
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 20)
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 0)
    twin.launches.clear()
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS)
    r = sw.run_clips(_streams(clip_set, advance=3, read_only=True), gts, **window)
    _check(r, want, len(grid), len(clip_set))
    assert twin.launches["psd_clip_eval_tables"] > 3  # several passes
    assert twin.launches["psd_clip_cuts_tables"] > twin.launches["psd_clip_eval_tables"]  # and retries


def test_run_with_settings_is_run_clips_of_one_clip(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    cls, grid = _grids()["adaptive"]
    gts = [gt for _, _, gt in clip_set]
    window = {"end_time": 2.5}
    want = _expect(cls, grid, SETTINGS, clip_set, window)
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=SETTINGS)
    for j, (frames, fps, gt) in enumerate(clip_set):
        r = sw.run(ArrayVideoStream(frames, fps), gt, **window)
        assert r.end_frames == [want[s, 0, j][1] for s in range(len(SETTINGS))] and r.end_frame == r.end_frames[0]
        for s in range(len(SETTINGS)):
            for g in range(len(grid)):
                k = s * len(grid) + g
                preds, _end, hard, fades = want[s, g, j]
                assert r.cuts(k) == preds and r.fades(k) == fades
                assert [r.hard(k, t) for t in TOLS] == [h[:3] for h in hard]
    assert sw.videos == len(clip_set)
    # a window alone also goes through the clip path
    plain = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    twin.launches.clear()
    r = plain.run(ArrayVideoStream(clip_set[3][0], clip_set[3][1]), gts[3], **window)
    assert twin.launches["psd_clip_eval"] == 3 and "psd_sweep_eval" not in twin.launches
    assert [r.cuts(g) for g in range(len(grid))] == [want[0, g, 3][0] for g in range(len(grid))]


def test_each_frame_is_read_once_and_decoded_when_processed(twin, clip_set):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["histogram"]
    for settings, window in (([{"frame_skip": 2}, {"frame_skip": 3}], {}),
                             ([{"frame_skip": 5}, {"crop": (0, 0, 30, 30), "frame_skip": 1}], {"duration": 1.0}),
                             (SETTINGS, {"end_time": 1.5})):
        streams = _streams(clip_set, advance=1, read_only=True)
        starts = [v.frame_number for v in streams]
        ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=settings).run_clips(streams, **window)
        for j, v in enumerate(streams):
            # what each setting's own SceneManager reads and processes
            reads, decodes = set(), set()
            for st in settings:
                own = _streams([clip_set[j]], advance=1, read_only=True)[0]
                detect_clips([own], [cls(**grid[0])], batch_size=BATCH, **st, **window)
                reads |= set(own.reads[1:] if len(clip_set[j][0]) > 1 else own.reads)
                decodes |= set(own.decodes[1:] if len(clip_set[j][0]) > 1 else own.decodes)
            got_reads = [n for n in v.reads if n >= starts[j]]
            assert got_reads == sorted(reads), (j, settings)   # every frame once, in order: the union
            assert [n for n in v.decodes if n >= starts[j]] == sorted(decodes), (j, settings)
            assert v.frame_number == max(reads) + 1   # the stream stands at the union's end


def test_host_frames_cross_once_and_read_batch_streams(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["hash"]
    settings = [{}, {"frame_skip": 2}, {"crop": (4, 2, 40, 30)}]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=settings)
    r = sw.run_clips(_streams(clip_set))
    # host streams with read_batch are read in chunks, and give what streams read frame by frame give
    r_read = sw.run_clips(_streams(clip_set, read_only=True))
    assert all(r.cuts(k, j) == r_read.cuts(k, j) and r.end_frame(j, s) == r_read.end_frame(j, s)
               for k in range(len(r)) for j in range(len(clip_set)) for s in range(3))
    sweep_settings_twin.SettingsEngine.layouts = []
    r = sw.run_clips(_streams(clip_set))
    # every frame is processed by setting 0, so every frame read is uploaded once, whatever the number of settings
    assert r.upload_bytes == sum(f.nbytes for f, _, _ in clip_set)
    # each step-1 setting takes every full batch as one run, across the clip boundaries inside it (the 64x36 clips
    # hold 133 frames: 8 full batches)
    fb = 64 * 36 * 3
    assert sum(1 for n, lay in sweep_settings_twin.SettingsEngine.layouts if lay[0] == fb and n == BATCH) == 2 * 8
    one = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=settings[2:])
    assert one.run_clips(_streams(clip_set)).upload_bytes == r.upload_bytes


def test_defaults_keep_todays_results_and_calls(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]
    base = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    r0 = base.run_clips(_streams(clip_set), gts)
    assert set(twin.launches) == {"scan", "psd_clip_fill", "psd_clip_cuts", "psd_clip_eval"}
    assert base.params == base.grid and [t.params for t in base.totals()] == grid
    twin.launches.clear()
    same = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=[{}])
    r1 = same.run_clips(_streams(clip_set), gts)
    assert set(twin.launches) == {"scan", "psd_clip_fill", "psd_clip_cuts", "psd_clip_eval"}
    assert r1.upload_bytes is None and r1.n_settings == 1
    for k in range(len(grid)):
        for j in range(len(clip_set)):
            assert r1.cuts(k, j) == r0.cuts(k, j) and r1.end_frame(j) == r0.end_frame(j)
    assert [(t.hard, t.fades) for t in same.totals()] == [(t.hard, t.fades) for t in base.totals()]


def test_refusals(twin, clip_set, caplog):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]

    def make(settings):
        return ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, settings=settings)

    with pytest.raises(TypeError, match="unknown setting key"):
        make([{"frame_skip": 1}, {"interpolation": 1}])
    with pytest.raises(ValueError, match="settings is empty"):
        make([])
    with pytest.raises(ValueError, match="Downscale factor must be a positive integer >= 1!"):
        make([{"auto_downscale": False, "downscale": 0}])
    with pytest.raises(TypeError, match="crop region must be tuple of 4 ints"):
        make([{"crop": (1, 2, 3)}])
    with pytest.raises(ValueError, match="crop coordinates must be >= 0"):
        make([{"crop": (1, -2, 3, 4)}])
    with pytest.raises(ValueError, match="frame_skip must be >= 0"):
        make([{"frame_skip": -1}])
    with pytest.raises(TypeError, match="frame_skip must be an integer"):
        make([{"frame_skip": 1.5}])
    with caplog.at_level(logging.WARNING, logger="pyscenedetect_b200"):
        ignored = make([{"downscale": 2}])  # ignored while auto_downscale is on, as SceneManager's setter says
    assert "Downscale factor will be ignored because auto_downscale=True!" in caplog.text
    a = ignored.run_clips(_streams(clip_set[:3]), gts[:3])
    b = make(None).run_clips(_streams(clip_set[:3]), gts[:3])
    assert [a.cuts(k, j) for k in range(len(grid)) for j in range(3)] == \
        [b.cuts(k, j) for k in range(len(grid)) for j in range(3)]

    sw = make(SETTINGS)
    sw.run_clips(_streams(clip_set[:2]), gts[:2])
    before = ([(t.hard, t.fades) for t in sw.totals()], sw.videos)
    streams = _streams(clip_set, read_only=True)
    wide = make(SETTINGS + [{"crop": (50, 0, 60, 30)}])  # starts right of the 48-pixel-wide clips
    with pytest.raises(ValueError, match=r"crop starts outside video boundary of clip 2 \(48x40\) in setting 7"):
        wide.run_clips(streams, gts)
    assert all(v.reads == [] for v in streams)  # refused before any frame is read
    assert wide.videos == 0
    with pytest.raises(ValueError, match="duration and end_time cannot be set at the same time!"):
        sw.run_clips(_streams(clip_set), gts, duration=1, end_time=2)
    with pytest.raises(ValueError, match="duration must be greater than or equal to 0!"):
        sw.run(_streams(clip_set)[1], gts[1], duration=-1)
    with pytest.raises(ValueError, match="end_time must be greater than or equal to 0!"):
        sw.run_clips(_streams(clip_set), gts, end_time=-2.0)
    assert ([(t.hard, t.fades) for t in sw.totals()], sw.videos) == before
    small = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, max_cuts_per_cell=1,
                           settings=[{"frame_skip": 1}, {}])
    with pytest.raises(RuntimeError, match=r"cell \d+ \(.*\) of setting \d \(\{.*\}\) found \d+ cuts in clip \d+, "
                                           r"more than max_cuts_per_cell=1"):
        small.run_clips(_streams(clip_set), gts)
    assert small.videos == 0


def test_tables_twin_with_one_table_is_the_existing_twins(twin):
    """psd_clip_cuts_tables / psd_clip_eval_tables with one table equal psd_clip_cuts_step / psd_clip_eval (twins),
    and with several tables one call per table."""
    from pyscenedetect_b200 import _capi
    lib = sweep_settings_twin.Lib()
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
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        tabs = []
        for step in (1, 3):
            first, end = clip_window_cases.first_and_end(sizes, step, gi + step)
            t = Buf(8 * (3 * c + 1))
            t.upload(np.concatenate([off, first, end]).astype(np.int64))
            tabs.append((t, step))
        mfb = Buf(mf.nbytes)
        mfb.upload(mf)

        def run_step(t, step):
            o, cuts = Buf(8 * (k * c + 1)), Buf(8 * CAP)
            lib.psd_clip_cuts_step(cells, k, t.ptr, t.ptr + 8 * (c + 1), c, mfb.ptr, cuts.ptr, CAP, o.ptr, step,
                                   t.ptr + 8 * (2 * c + 1), None)
            return _array_of(o, k * c + 1), cuts

        tables = (_capi.PsdClipTable * 2)(*[_capi.PsdClipTable(t.ptr, t.ptr + 8 * (c + 1), t.ptr + 8 * (2 * c + 1),
                                                                step) for t, step in tabs])
        # one table
        for i in range(2):
            want_o, want_c = run_step(*tabs[i])
            o, cuts = Buf(8 * (k * c + 1)), Buf(8 * CAP)
            lib.psd_clip_cuts_tables(cells, k, C.cast(C.byref(tables, i * 32), C.POINTER(_capi.PsdClipTable)), 1,
                                     None, c, mfb.ptr, cuts.ptr, CAP, o.ptr, None)
            got_o = _array_of(o, k * c + 1)
            assert (got_o == want_o).all() and 0 < got_o[-1] <= CAP
            assert (cuts.data[:8 * got_o[-1]] == want_c.data[:8 * got_o[-1]]).all()
        # two tables: cells 0 .. k-1 over table 1, then the same cells over table 0
        both = (_capi.PsdSweepCell * (2 * k))(*(list(cells) + list(cells)))
        mf2 = Buf(2 * mf.nbytes)
        mf2.upload(np.concatenate([mf, mf]))
        o, cuts = Buf(8 * (2 * k * c + 1)), Buf(16 * CAP)
        lib.psd_clip_cuts_tables(both, 2 * k, tables, 2, (C.c_int32 * (2 * k))(*([1] * k + [0] * k)), c, mf2.ptr,
                                 cuts.ptr, 2 * CAP, o.ptr, None)
        got_o = _array_of(o, 2 * k * c + 1)
        lists = [cuts.data[8 * got_o[t]:8 * got_o[t + 1]].view(np.int64).tolist() for t in range(2 * k * c)]
        for half, i in ((0, 1), (1, 0)):
            want_o, want_c = run_step(*tabs[i])
            want = [want_c.data[8 * want_o[t]:8 * want_o[t + 1]].view(np.int64).tolist() for t in range(k * c)]
            assert lists[half * k * c:(half + 1) * k * c] == want

        # the evaluator: one table equals psd_clip_eval on the same lists
        gt_off = np.arange(c + 1, dtype=np.int64)
        gt = np.array([int(x) + 2 for x in np.frombuffer(tabs[0][0].data[8 * (c + 1):8 * (2 * c + 1)].tobytes(),
                                                           np.int64)], np.int64)
        gtab = Buf(8 * (2 * (c + 1) + c + 2 * c))
        gtab.upload(np.concatenate([gt_off, gt_off, gt, np.stack([gt - 1, gt + 1], 1).ravel()]))
        tols = (C.c_int32 * 2)(0, 2)
        outs = []
        for which in ("eval", "tables"):
            co, cc = run_step(*tabs[0])
            total = int(co[-1])
            ws = Buf(sweep_clip_twin.workspace_bytes(k, c, 2, total, c, c))
            arrays = [Buf(4 * k * c), Buf(40 * 2 * k * c), Buf(24 * k * c), Buf(40 * 2 * k), Buf(24 * k), Buf(8)]
            truth = (gtab.ptr, gtab.ptr + 16 * (c + 1), c, gtab.ptr + 8 * (c + 1), gtab.ptr + 16 * (c + 1) + 8 * c, c,
                     tols, 2, ws.ptr, ws.nbytes, *[a.ptr for a in arrays], None)
            cptr = Buf(8 * max(1, total))
            cptr.data[:8 * total] = cc.data[:8 * total]
            co_buf = Buf(8 * (k * c + 1))
            co_buf.upload(co)
            if which == "eval":
                lib.psd_clip_eval(cptr.ptr, co_buf.ptr, k, c, total, 64, tabs[0][0].ptr + 8 * (2 * c + 1), *truth)
            else:
                lib.psd_clip_eval_tables(cptr.ptr, co_buf.ptr, k, c, total, 64, tables, 1, None, *truth)
            outs.append([a.data.copy() for a in arrays] + [cptr.data.copy()])
        for a, b in zip(*outs):
            assert (a == b).all()


CAP = 1 << 17


def _array_of(buf, n):
    return buf.data[:8 * n].view(np.int64).copy()


def test_c_abi_rejects_bad_tables_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    p = 4096
    cells = (_capi.PsdSweepCell * 2)(*[_capi.PsdSweepCell(kind=_capi.SWEEP_HASH, metric=p, threshold=0.5)] * 2)
    good = (_capi.PsdClipTable * 2)(_capi.PsdClipTable(p, p, p, 1), _capi.PsdClipTable(p, p, p, 3))

    def cuts(tables=good, n_tables=2, cell_table=(C.c_int32 * 2)(0, 1)):
        return lib.psd_clip_cuts_tables(cells, 2, tables, n_tables, cell_table, 3, p, p, 16, p, None)

    assert cuts(tables=None) == _capi.PSD_ERR_INVALID
    assert b"no clip table" in lib.psd_last_error()
    assert cuts(n_tables=0) == _capi.PSD_ERR_INVALID
    assert cuts(cell_table=(C.c_int32 * 2)(0, 2)) == _capi.PSD_ERR_INVALID
    assert b"cell 1 names table 2 of 2" in lib.psd_last_error()
    assert cuts(tables=(_capi.PsdClipTable * 2)(_capi.PsdClipTable(p, p, p, 1), _capi.PsdClipTable(p, p, p, 0))) == \
        _capi.PSD_ERR_INVALID
    assert b"frame_step must be >= 1" in lib.psd_last_error()
    assert cuts(tables=(_capi.PsdClipTable * 2)(_capi.PsdClipTable(p, p, p, 1), _capi.PsdClipTable(p, None, p, 1))) \
        == _capi.PSD_ERR_INVALID
    assert b"no clip first frames" in lib.psd_last_error()
    one = (C.c_int32 * 1)(1)
    need = sweep_clip_twin.workspace_bytes(2, 3, 1, 10, 4, 2)

    def ev(tables=good, n_tables=2, cell_table=(C.c_int32 * 2)(1, 0)):
        return lib.psd_clip_eval_tables(p, p, 2, 3, 10, 16, tables, n_tables, cell_table, p, p, 4, p, p, 2, one, 1, p,
                                        need, p, p, p, p, p, p, None)

    assert ev(tables=(_capi.PsdClipTable * 2)(_capi.PsdClipTable(p, p, p, 1), _capi.PsdClipTable(p, p, None, 1))) \
        == _capi.PSD_ERR_INVALID
    assert b"psd_clip_eval_tables: no clip tables" in lib.psd_last_error()
    assert ev(n_tables=0) == _capi.PSD_ERR_INVALID
    assert ev(cell_table=(C.c_int32 * 2)(-1, 0)) == _capi.PSD_ERR_INVALID
    assert b"cell 0 names table -1 of 2" in lib.psd_last_error()


def test_table_kernels_do_not_spill():
    import os
    import re
    import shutil
    import subprocess
    from pyscenedetect_b200 import _capi
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([tool, "-res-usage", _capi.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    pat = r"Function (\S*(?:psd_clip_cuts_kernel|clip_eval_kernel)\S*ClipTable\S*):\s*\n\s*REG:\d+ STACK:(\d+) " \
          r"SHARED:\d+ LOCAL:(\d+)"
    found = {fn: (stack, local) for fn, stack, local in re.findall(pat, out)}
    assert len(found) == 3, out[:2000]  # both cut passes and the evaluator read the tables
    assert all(v == ("0", "0") for v in found.values()), found
