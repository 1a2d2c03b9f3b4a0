"""GPU tests of `ParameterSweep.run_clips(windows=...)`: a window per clip (crop, duration / end_time, frame_skip)
under every setting of a sweep, in one read of each clip.

* psd_clip_cuts_tables_steps with one table equals psd_clip_cuts_steps, with every step equal it is bit-equal to
  psd_clip_cuts_tables, and with several tables it equals one call per table, on the adversarial metric sequences of
  tests/automata_inputs.py;
* grids of every detector and detector sets over 40 host, CUDA BGR, RGB and strided-view clips equal, for every
  (setting, cell, clip), a one-clip sweep with the setting and the clip's window;
* a windowed pass launches what a pass with one window for every clip launches."""

from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from tests import clip_window_cases
from tests.test_gpu_sweep_clips import TOLS, _clip_set, _cls, _counts, _random_grid, _render, _stream, _totals

pytestmark = pytest.mark.gpu

# crops that every test clip (160x90, 96x54, 640x360) starts inside: the first cuts each to 96x42, the second to 80x54
CROPS = [(0, 6, 95, 47), (8, 0, 87, 53)]


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


# -- 1. the entry ------------------------------------------------------------------------------------------------------
def test_tables_steps_entry(lib):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200._capi import check
    from pyscenedetect_b200.engine import DeviceBuffer
    cap = 1 << 18

    def dev(a):
        a = np.ascontiguousarray(a)
        b = DeviceBuffer(max(8, a.nbytes))
        b.upload(a)
        return b

    def run(m, call):
        o, cuts = DeviceBuffer(8 * (m + 1)), DeviceBuffer(8 * cap)
        call(cuts.ptr, o.ptr)
        off = o.download(8 * (m + 1)).view(np.int64)
        assert 0 <= off[-1] <= cap
        data = cuts.download(8 * int(off[-1])).view(np.int64) if off[-1] else np.zeros(0, np.int64)
        return off, data, [data[off[t]:off[t + 1]].tolist() for t in range(m)]

    for gi, (kind, _w, sizes, metric, metric2, params) in enumerate(clip_window_cases.groups()):
        c = len(sizes)
        keep = [dev(metric)] + ([dev(metric2)] if metric2 is not None else [])
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, keep[0].ptr,
                                                             keep[1].ptr if metric2 is not None else None, c, gi)
        mfb, mf2 = dev(mf), dev(np.concatenate([mf, mf]))
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        steps = np.random.default_rng(gi).integers(1, 5, c).astype(np.int64)
        first, end = clip_window_cases.first_and_end(sizes, 4, gi)
        mixed = dev(np.concatenate([off, first, end, steps]))
        equal = dev(np.concatenate([off, first, end, np.full(c, 3, np.int64)]))

        def steps_table(t):
            return _capi.PsdClipStepsTable(t.ptr, t.ptr + 8 * (c + 1), t.ptr + 8 * (2 * c + 1), t.ptr + 8 * (3 * c + 1))

        def tables_steps(*ts, cells=cells, n=k, cell_table=None, mfp=mfb.ptr):
            return lambda cuts, o: check(lib.psd_clip_cuts_tables_steps(
                cells, n, (_capi.PsdClipStepsTable * len(ts))(*[steps_table(t) for t in ts]), len(ts), cell_table, c,
                mfp, cuts, cap, o, None))

        # one table: psd_clip_cuts_steps with the same steps as a host array
        got = run(k * c, tables_steps(mixed))
        want = run(k * c, lambda cuts, o: check(lib.psd_clip_cuts_steps(
            cells, k, mixed.ptr, mixed.ptr + 8 * (c + 1), c, mfb.ptr, cuts, cap, o, (C.c_int64 * c)(*steps.tolist()),
            mixed.ptr + 8 * (2 * c + 1), None)))
        assert (got[0] == want[0]).all() and got[2] == want[2] and got[0][-1] > 0, (kind, gi)
        # every step equal: psd_clip_cuts_tables bit for bit
        got = run(k * c, tables_steps(equal))
        plain = _capi.PsdClipTable(equal.ptr, equal.ptr + 8 * (c + 1), equal.ptr + 8 * (2 * c + 1), 3)
        want = run(k * c, lambda cuts, o: check(lib.psd_clip_cuts_tables(
            cells, k, (_capi.PsdClipTable * 1)(plain), 1, None, c, mfb.ptr, cuts, cap, o, None)))
        assert (got[0] == want[0]).all() and got[1].tobytes() == want[1].tobytes(), (kind, gi)
        # two tables: cells over table 1, then the same cells over table 0
        both = (_capi.PsdSweepCell * (2 * k))(*(list(cells) + list(cells)))
        got = run(2 * k * c, tables_steps(mixed, equal, cells=both, n=2 * k,
                                          cell_table=(C.c_int32 * (2 * k))(*([1] * k + [0] * k)), mfp=mf2.ptr))
        assert got[2][:k * c] == run(k * c, tables_steps(equal))[2]
        assert got[2][k * c:] == run(k * c, tables_steps(mixed))[2]


def test_tables_steps_refuses_bad_tables(lib):
    from pyscenedetect_b200 import _capi
    p = 4096
    cells = (_capi.PsdSweepCell * 1)(_capi.PsdSweepCell(kind=_capi.SWEEP_HASH, metric=p, threshold=0.5))
    bad = (_capi.PsdClipStepsTable * 1)(_capi.PsdClipStepsTable(p, p, p, None))
    assert lib.psd_clip_cuts_tables_steps(cells, 1, bad, 1, None, 2, p, p, 16, p, None) == _capi.PSD_ERR_INVALID
    assert b"table 0 has no frame_step array" in lib.psd_last_error()


# -- 2. sweeps with windows against one-clip sweeps ----------------------------------------------------------------------
def _windows(clips, seed, crops_and_skips: bool):
    rng = random.Random(seed)
    ends = [{}, {"duration": 9}, {"duration": 0.5}, {"end_time": "00:00:01.200"}, {"end_time": 30}, {"duration": "2s"}]
    out = []
    for i in range(len(clips)):
        w = dict(rng.choice(ends))
        if crops_and_skips:
            if rng.random() < 0.7:
                w["crop"] = rng.choice(CROPS)
            if rng.random() < 0.7:
                w["frame_skip"] = rng.randint(0, 3)
        out.append(w or None)
    return out


def _with_strided_views(clips):
    """The clip set with every fifth CUDA clip read from a strided view: a crop of a larger tensor."""
    import torch
    from pyscenedetect_b200.video import ArrayVideoStream

    def open_clip(j, frames, fps, src):
        if src == "cuda" and j % 5 == 1:
            n, h, w, _ = frames.shape
            big = torch.zeros((n, h + 6, w + 10, 3), dtype=torch.uint8, device="cuda")
            big[:, 3:3 + h, 5:5 + w] = torch.from_numpy(frames).cuda()
            return ArrayVideoStream(big[:, 3:3 + h, 5:5 + w], fps)
        return _stream(frames, fps, src)
    return open_clip


def _one_clip(make, settings, s, clip, window, open_clip, j):
    frames, fps, gt, src = clip
    w = window or {}
    sw = make([{**settings[s], **{k: v for k, v in w.items() if k in ("crop", "frame_skip")}}])
    r = sw.run_clips([open_clip(j, frames, fps, src)], [gt], **{k: v for k, v in w.items()
                                                               if k in ("duration", "end_time")})
    return sw, r


def _check_against_one_clip_sweeps(make, settings, clips, windows):
    open_clip = _with_strided_views(clips)
    sw = make(settings)
    r = sw.run_clips([open_clip(j, f, fps, src) for j, (f, fps, _, src) in enumerate(clips)],
                     [gt for _, _, gt, _ in clips], windows=windows)
    n_cells = len(r) // len(settings)
    found = 0
    totals = None
    for s in range(len(settings)):
        for j, clip in enumerate(clips):
            one_sw, one = _one_clip(make, settings, s, clip, windows[j], open_clip, j)
            assert r.end_frame(j, setting=s) == one.end_frame(0), (s, j, windows[j])
            for g in range(n_cells):
                assert _counts(r, s * n_cells + g, j) == _counts(one, g, 0), (s, g, j, windows[j], clip[3])
                found += r.raw_count(s * n_cells + g, j)
            got = [(t.hard, t.hard_offset, t.fades) for t in one_sw.totals()]
            if totals is None:
                totals = [[None] * len(clips) for _ in settings]
            totals[s][j] = got
    assert found > 0
    for s in range(len(settings)):
        for g in range(n_cells):
            t = r.totals()[s * n_cells + g]
            for q in TOLS:
                assert (t.hard[q].matched, t.hard[q].false_positives, t.hard[q].missed) == tuple(
                    sum(getattr(totals[s][j][g][0][q], a) for j in range(len(clips)))
                    for a in ("matched", "false_positives", "missed"))
                assert t.hard_offset[q] == (float(sum(totals[s][j][g][1][q][0] for j in range(len(clips)))),
                                            sum(totals[s][j][g][1][q][1] for j in range(len(clips))))
            assert (t.fades.matched, t.fades.false_positives, t.fades.missed) == tuple(
                sum(getattr(totals[s][j][g][2], a) for j in range(len(clips)))
                for a in ("matched", "false_positives", "missed"))
    assert _totals(sw)[1] == len(clips)


@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
@pytest.mark.parametrize("crops_and_skips", [True, False], ids=["crops_and_skips", "ends_only"])
def test_windows_equal_one_clip_sweeps(lib, det, crops_and_skips):
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(len(det))
    grid = _random_grid(det, 24, rng)
    clips = _clip_set(seed=len(det) + 7)
    # the hash image (up to 32x32) must fit every scored frame: hash grids scale to full size instead of down
    scale = {"auto_downscale": False} if det == "hash" else {"auto_downscale": False, "downscale": 2}
    settings = ([{}, scale] if crops_and_skips else
                [{}, {"frame_skip": 2}, {"crop": CROPS[0], "frame_skip": 1}, scale])
    windows = _windows(clips, len(det), crops_and_skips)

    def make(st):
        return ParameterSweep(_cls(det), grid, tolerances=TOLS, batch_size=16, settings=st)

    _check_against_one_clip_sweeps(make, settings, clips, windows)


def test_detector_sets_with_windows(lib):
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    from pyscenedetect_b200.sweep import ParameterSweep
    sets = [ContentDetector(threshold=14.0), [AdaptiveDetector(), ThresholdDetector(threshold=20, add_final_scene=True)],
            [HashDetector(threshold=0.3, size=8), HistogramDetector(threshold=0.1, bins=64)],
            [ContentDetector(threshold=20.0, min_scene_len=3), HashDetector(threshold=0.2, size=16)]]
    clips = _clip_set(seed=3)
    settings = [{}, {"auto_downscale": False}]  # full size: the 32x32 hash image fits every cropped frame

    def make(st):
        return ParameterSweep(detector_sets=sets, tolerances=TOLS, batch_size=16, settings=st)

    _check_against_one_clip_sweeps(make, settings, clips, _windows(clips, 3, True))


# -- 3. launches per pass ----------------------------------------------------------------------------------------------
def test_windowed_pass_launches_what_a_uniform_window_pass_launches(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 64.0)  # no retry: the same launches whatever the cuts
    frames, cuts = _render(120, 96, 54, seed=9)
    calls = {}
    names = ("psd_clip_cuts_tables", "psd_clip_cuts_tables_steps", "psd_clip_eval_tables", "psd_scan_content",
             "psd_clip_fill")
    for name in names:
        def wrap(*a, _fn=getattr(lib, name), _name=name):
            before = lib.psd_launch_count()
            rc = _fn(*a)
            calls[_name] = calls.get(_name, 0) + lib.psd_launch_count() - before
            return rc
        monkeypatch.setattr(lib, name, wrap)
    grid = [dict(threshold=5.0 + 30.0 * i / 64, min_scene_len=(0, 2, 0.2)[i % 3]) for i in range(64)]
    settings = [{}, {"auto_downscale": False, "downscale": 2}]
    n_clips, k = 30, 4
    gts = [GroundTruth([c - i * k for c in cuts if i * k <= c < (i + 1) * k]) for i in range(n_clips)]

    def run(**kw):
        calls.clear()
        streams = [ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)]
        ParameterSweep(ContentDetector, grid, tolerances=TOLS, batch_size=16, settings=settings).run_clips(
            streams, gts, **kw)
        return dict(calls)

    uniform = run(duration=3)
    # two crops of one size and skips 0 to 2: one group, one pass, one stepped automaton launch
    windowed = run(windows=[{"crop": ((0, 0, 95, 47), (0, 6, 95, 53))[i % 2], "frame_skip": i % 3, "duration": 3}
                            for i in range(n_clips)])
    assert windowed.pop("psd_clip_cuts_tables_steps") == uniform.pop("psd_clip_cuts_tables") == 3
    assert windowed == uniform and uniform["psd_clip_eval_tables"] == 3
