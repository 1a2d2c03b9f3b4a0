"""GPU tests of the sweep over settings (`ParameterSweep(settings=...)`: psd_clip_cuts_tables + psd_clip_eval_tables
after one read of each clip for every setting):

* the table entries with one table are bit-equal to psd_clip_cuts, psd_clip_cuts_step and psd_clip_eval on the
  adversarial metric sequences of tests/automata_inputs.py, and with several tables equal one call per table;
* 64-cell grids of every detector x 5 settings over 40 pageable, page-locked and CUDA (BGR, RGB, NCHW) clips equal a
  per-setting `detect_clips` scored on the host, and the one-setting sweeps;
* the golden sweep grids as the middle clip give their recorded counts in setting {} beside other settings;
* the launches of a pass do not grow with the settings, cells or clips, and host frames cross PCIe once;
* the cut-buffer retry and the max_cuts_per_cell overflow work with several settings."""

from __future__ import annotations

import ctypes as C
import json
import os
import random

import numpy as np
import pytest

from tests import clip_window_cases, sweep_model
from tests.test_gpu_sweep_clips import TOLS, _clip_set, _cls, _counts, _random_grid, _render, _stream, _totals

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
# the settings of a letterbox / speed study, scaled to the test clips (the smallest is 96x54)
SETTINGS = [{}, {"frame_skip": 1}, {"frame_skip": 3}, {"auto_downscale": False, "downscale": 2},
            {"crop": (0, 6, 95, 47), "frame_skip": 1}]


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


def _sources(clips):
    """The clips of `_clip_set` with every other host clip page-locked."""
    out = []
    for i, (frames, fps, gt, src) in enumerate(clips):
        out.append((frames, fps, gt, "pinned" if src == "host" and i % 4 == 0 else src))
    return out


def _open(frames, fps, src, keep):
    from pyscenedetect_b200.engine import PinnedBuffer
    from pyscenedetect_b200.video import ArrayVideoStream
    if src != "pinned":
        return _stream(frames, fps, src)
    buf = PinnedBuffer(max(1, frames.nbytes))
    keep.append(buf)
    arr = buf.array[:frames.nbytes].reshape(frames.shape)
    np.copyto(arr, frames)
    return ArrayVideoStream(arr, fps, pinned=True)


# -- 1. the entries ----------------------------------------------------------------------------------------------------
def test_table_entries_equal_the_one_table_entries(lib):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200._capi import check
    from pyscenedetect_b200.engine import DeviceBuffer
    from tests.sweep_clip_twin import workspace_bytes
    cap = 1 << 18

    def dev(a):
        a = np.ascontiguousarray(a)
        b = DeviceBuffer(max(8, a.nbytes))
        b.upload(a)
        return b

    def i64(b, n):
        return b.download(8 * n).view(np.int64)

    for gi, (kind, _w, sizes, metric, metric2, params) in enumerate(clip_window_cases.groups()):
        c = len(sizes)
        keep = [dev(metric)] + ([dev(metric2)] if metric2 is not None else [])
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, keep[0].ptr,
                                                             keep[1].ptr if metric2 is not None else None, c, gi)
        mfb, mf2 = dev(mf), dev(np.concatenate([mf, mf]))
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        tabs = []
        for step in (1, 3):
            first, end = clip_window_cases.first_and_end(sizes, step, gi + step)
            tabs.append((dev(np.concatenate([off, first, end]).astype(np.int64)), step))
        table = lambda t, step, end=True: _capi.PsdClipTable(  # noqa: E731
            t.ptr, t.ptr + 8 * (c + 1), t.ptr + 8 * (2 * c + 1) if end else None, step)

        def cut(call):
            o, cuts = DeviceBuffer(8 * (k * 2 * c + 1)), DeviceBuffer(8 * cap)
            call(cuts.ptr, o.ptr)
            got_o = i64(o, k * c + 1) if call.__name__ != "two" else i64(o, 2 * k * c + 1)
            assert got_o[-1] <= cap
            data = i64(cuts, int(got_o[-1])) if got_o[-1] else np.zeros(0, np.int64)
            lists = [data[got_o[t]:got_o[t + 1]].tolist() for t in range(len(got_o) - 1)]
            o.close()
            return got_o, data, lists, cuts

        t0, st0 = tabs[0]
        t1, st1 = tabs[1]

        def plain(cuts, o):
            check(lib.psd_clip_cuts(cells, k, t0.ptr, t0.ptr + 8 * (c + 1), c, mfb.ptr, cuts, cap, o, None))

        def one_plain(cuts, o):
            check(lib.psd_clip_cuts_tables(cells, k, (_capi.PsdClipTable * 1)(table(t0, 1, False)), 1, None, c,
                                           mfb.ptr, cuts, cap, o, None))

        def step(cuts, o):
            check(lib.psd_clip_cuts_step(cells, k, t1.ptr, t1.ptr + 8 * (c + 1), c, mfb.ptr, cuts, cap, o, st1,
                                         t1.ptr + 8 * (2 * c + 1), None))

        def one_step(cuts, o):
            check(lib.psd_clip_cuts_tables(cells, k, (_capi.PsdClipTable * 1)(table(t1, st1)), 1, None, c, mfb.ptr,
                                           cuts, cap, o, None))

        def two(cuts, o):  # cells over table 1, then the same cells over table 0
            both = (_capi.PsdSweepCell * (2 * k))(*(list(cells) + list(cells)))
            check(lib.psd_clip_cuts_tables(both, 2 * k, (_capi.PsdClipTable * 2)(table(t0, 1, False), table(t1, st1)),
                                           2, (C.c_int32 * (2 * k))(*([1] * k + [0] * k)), c, mf2.ptr, cuts, cap, o,
                                           None))

        a, b = cut(plain), cut(one_plain)
        assert (a[0] == b[0]).all() and (a[1] == b[1]).all(), (gi, kind)
        s1, s2 = cut(step), cut(one_step)
        assert (s1[0] == s2[0]).all() and (s1[1] == s2[1]).all(), (gi, kind)
        both = cut(two)
        assert both[2] == s1[2] + a[2], (gi, kind)
        for x in (a, b, s1, s2, both):
            x[3].close()

        # the evaluator on the stepped lists: psd_clip_eval against psd_clip_eval_tables, bit for bit
        gt = t0.download(8 * (2 * c + 1)).view(np.int64)[c + 1:2 * c + 1] + 2
        gt_off = np.arange(c + 1, dtype=np.int64)
        gtab = dev(np.concatenate([gt_off, gt_off, gt, np.stack([gt - 1, gt + 1], 1).ravel()]).astype(np.int64))
        tols = (C.c_int32 * 2)(0, 2)
        outs = []
        for which in ("eval", "tables"):
            o_h, data, _lists, cuts = cut(step)
            total = int(o_h[-1])
            ob = dev(o_h)
            ws = DeviceBuffer(workspace_bytes(k, c, 2, total, c, c))
            arrays = [DeviceBuffer(n) for n in (4 * k * c, 80 * k * c, 24 * k * c, 80 * k, 24 * k, 8)]
            truth = (gtab.ptr, gtab.ptr + 16 * (c + 1), c, gtab.ptr + 8 * (c + 1), gtab.ptr + 16 * (c + 1) + 8 * c, c,
                     tols, 2, ws.ptr, ws.nbytes, *[x.ptr for x in arrays], None)
            if which == "eval":
                check(lib.psd_clip_eval(cuts.ptr, ob.ptr, k, c, total, 64, t1.ptr + 8 * (2 * c + 1), *truth))
            else:
                check(lib.psd_clip_eval_tables(cuts.ptr, ob.ptr, k, c, total, 64,
                                               (_capi.PsdClipTable * 1)(table(t1, st1)), 1, None, *truth))
            outs.append([x.download(x.nbytes).tobytes() for x in arrays] + [cuts.download(8 * max(1, total)).tobytes()])
            for x in (ob, ws, cuts, *arrays):
                x.close()
        assert outs[0] == outs[1], (gi, kind)
        for x in (*keep, mfb, mf2, gtab, t0, t1):
            x.close()


# -- 2. end to end: every (setting, cell, clip) ------------------------------------------------------------------------
def _per_setting(det, params, setting, clips):
    """detect_clips with setting `setting` and one detector: (predicted list, end frame) per clip."""
    from pyscenedetect_b200.clips import detect_clips
    keep = []
    res = detect_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], [_cls(det)(**params)], batch_size=16,
                       **setting)
    return [(sweep_model.predicted_list(r.cut_frames, r.end.frame_num + 1), r.end.frame_num + 1) for r in res]


@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_settings_sweep_equals_detect_clips_per_setting(lib, det):
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(100 + len(det))
    grid = _random_grid(det, 64, rng)
    if det == "hash":  # 96x54 clips downscaled by 2 are 48x27: too small for the 32x32 hash image of size 16
        grid = [{**p, "size": 8} for p in grid]
    clips = _sources(_clip_set(seed=3 + len(det)))
    gts = [gt for _, _, gt, _ in clips]
    keep = []
    sw = ParameterSweep(_cls(det), grid, tolerances=TOLS, batch_size=16, settings=SETTINGS)
    r = sw.run_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], gts)
    found = 0
    for s, setting in enumerate(SETTINGS):
        one = ParameterSweep(_cls(det), grid, tolerances=TOLS, batch_size=16, settings=[setting])
        r1 = one.run_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], gts)
        for g in range(len(grid)):
            k = s * len(grid) + g
            for j in range(len(clips)):
                assert _counts(r, k, j) == _counts(r1, g, j), (det, s, g, j)
                found += r.raw_count(k, j)
        assert [(t.hard, t.fades) for t in r.totals()[s * len(grid):(s + 1) * len(grid)]] == \
            [(t.hard, t.fades) for t in one.totals()]
        for g in rng.sample(range(len(grid)), 6):  # the contract itself: detect_clips, scored on the host
            want = _per_setting(det, grid[g], setting, clips)
            for j, (preds, end) in enumerate(want):
                assert r.end_frame(j, setting=s) == end
                assert r.cuts(s * len(grid) + g, j) == preds, (det, s, g, j)
                for t in TOLS:
                    h, f = sweep_model.score(preds, gts[j].hard_cuts, gts[j].fades, t)
                    assert r.hard(s * len(grid) + g, j, t) == h[:3] and r.fades(s * len(grid) + g, j) == f
    assert found > 0


# -- 3. the golden grids beside other settings -------------------------------------------------------------------------
@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_reference_grids_as_the_middle_clip_beside_other_settings(lib, det):
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.test_gpu_sweep import _frames, _kw
    with open(os.path.join(HERE, "golden", "sweep_v1.json")) as f:
        golden = json.load(f)
    g = next(x for x in golden["grids"] if x["det"] == det)
    _, frames = _frames(g["gen"])
    tols = golden["tolerances"]
    rev = frames[::-1]
    clips = [rev[:5], frames, rev[-4:]]
    h, w = frames.shape[1:3]
    settings = [{}, {"frame_skip": 2}, {"crop": (1, 1, w - 2, h - 2)}]
    sw = ParameterSweep(_cls(det), [_kw(c["kw"]) for c in g["cells"]], tolerances=tols, batch_size=48,
                        settings=settings)
    gts = [GroundTruth([3]), GroundTruth(g["true_cuts"], [tuple(f) for f in g["fades"]]), GroundTruth([], [(0, 2)])]
    r = sw.run_clips([ArrayVideoStream(c, g["fps"]) for c in clips], gts)
    for k, cell in enumerate(g["cells"]):
        assert r.cuts(k, 1) == cell["pred"], (k, cell["kw"])
        got = {str(t): {"hard": [*r.hard(k, 1, t), int(r.hard_offset(k, 1, t)[0]), r.hard_offset(k, 1, t)[1]],
                        "fades": list(r.fades(k, 1))} for t in tols}
        assert got == cell["want"], (k, cell["kw"])


# -- 4. launches and bytes per pass ------------------------------------------------------------------------------------
def test_pass_launches_and_uploads_do_not_grow_with_settings_cells_or_clips(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200 import fan_out
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 64.0)  # no retry: the same launches whatever the cuts
    frames, cuts = _render(120, 96, 54, seed=9)
    calls = {}
    real = lib.psd_clip_cuts_tables, lib.psd_clip_eval_tables

    def counted(name, fn):
        def wrap(*a):
            before = lib.psd_launch_count()
            rc = fn(*a)
            calls[name] = calls.get(name, 0) + lib.psd_launch_count() - before
            return rc
        return wrap

    monkeypatch.setattr(lib, "psd_clip_cuts_tables", counted("cuts", real[0]))
    monkeypatch.setattr(lib, "psd_clip_eval_tables", counted("eval", real[1]))
    uploads = []
    real_upload = fan_out.DeviceBuffer.upload

    def upload(self, arr, offset=0):  # frames only: the clip and ground-truth tables are uploaded too
        if np.asarray(arr).ndim == 4:
            uploads.append(np.asarray(arr).nbytes)
        return real_upload(self, arr, offset)

    monkeypatch.setattr(fan_out.DeviceBuffer, "upload", upload)
    for settings in (SETTINGS[1:3], SETTINGS):
        for n_cells in (8, 256):
            grid = [dict(threshold=5.0 + 30.0 * i / n_cells, min_scene_len=(0, 2, 0.2)[i % 3]) for i in range(n_cells)]
            for n_clips in (3, 30):
                k = 120 // n_clips
                sw = ParameterSweep(ContentDetector, grid, tolerances=TOLS, batch_size=16, settings=settings)
                gts = [GroundTruth([c - i * k for c in cuts if i * k <= c < (i + 1) * k]) for i in range(n_clips)]
                calls.clear()
                uploads.clear()
                r = sw.run_clips([ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)], gts)
                # one pass: three automaton launches and three evaluator launches for every setting, cell and clip
                assert calls == {"cuts": 3, "eval": 3}, (len(settings), n_cells, n_clips, calls)
                # host frames: every frame some setting processes is uploaded once, whatever the number of settings
                processed = set()
                for setting in settings:
                    processed |= set(range(0, k, setting.get("frame_skip", 0) + 1))
                assert sum(uploads) == r.upload_bytes == n_clips * len(processed) * 96 * 54 * 3


# -- 5. the retry, a lowered pass bound and the overflow ---------------------------------------------------------------
def test_retry_split_passes_and_overflow_with_settings(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    rng = random.Random(5)
    grid = _random_grid("content", 32, rng)
    clips = _sources(_clip_set(seed=11, n_clips=24))
    keep = []

    def run():
        sw = ParameterSweep(_cls("content"), grid, tolerances=TOLS, batch_size=16, settings=SETTINGS)
        r = sw.run_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], [gt for _, _, gt, _ in clips])
        return [[_counts(r, k, j) for j in range(len(clips))] for k in range(len(r))], _totals(sw)

    want = run()
    passes = []
    cuts = clips_mod._Pass.cuts_tables

    def spy(self, engines, holders, done, steps):
        passes.append(sum(e.frame_count for e in engines))
        return cuts(self, engines, holders, done, steps)

    monkeypatch.setattr(clips_mod._Pass, "cuts_tables", spy)
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 0)
    monkeypatch.setattr(clips_mod, "MAX_PASS_FRAMES", 20)
    assert run() == want
    assert len(passes) > 6
    monkeypatch.undo()

    sw = ParameterSweep(ContentDetector, [dict(threshold=200.0), dict(threshold=5.0, min_scene_len=0)],
                        tolerances=TOLS, max_cuts_per_cell=4, settings=[{"frame_skip": 3}, {}])
    short, _ = _render(3, 96, 54, seed=1)
    sw.run_clips([ArrayVideoStream(short, 25)], [GroundTruth([1])])
    before = _totals(sw)
    frames, cuts_ = _render(90, 96, 54, seed=2)
    with pytest.raises(RuntimeError, match=r"cell [13] \(\{'threshold': 5.0, 'min_scene_len': 0\}\) of setting [01] "
                                           r"\(\{.*\}\) found \d+ cuts in clip 1, more than max_cuts_per_cell=4"):
        sw.run_clips([ArrayVideoStream(short, 25), ArrayVideoStream(frames, 25)], [GroundTruth([]), GroundTruth(cuts_)])
    assert _totals(sw) == before
