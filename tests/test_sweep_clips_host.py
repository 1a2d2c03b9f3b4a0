"""`ParameterSweep.run_clips` without a GPU: the oracle-backed engine of tests/fake_engine.py scores the frames, and the
Python twins of the clip kernels (tests/clip_twin.py) and of psd_clip_eval (tests/sweep_clip_twin.py) stand in for
the library.  What is checked here is the host side - passes, clip tables, ground-truth tables, workspace sizes,
result accessors, totals and refusals - against one `SceneManager` per (cell, clip) scored by tests/sweep_model.py.
The kernels themselves are checked against `ParameterSweep.run` in tests/test_gpu_sweep_clips.py."""

from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import pytest

from tests import clip_twin, sweep_clip_twin, sweep_model
from tests.test_clips_host import BATCH, LENGTHS, RATES

TOLS = (0, 1, 3)
CLIP_LENGTHS = [n for n in LENGTHS if n]


def _grids():
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    return {
        "content": (ContentDetector, [dict(threshold=20.0, min_scene_len=0.2),
                                      dict(threshold=12.0, min_scene_len=3, filter_mode=FlashFilter.Mode.SUPPRESS),
                                      dict(threshold=12.0, min_scene_len=3, filter_mode=FlashFilter.Mode.MERGE)]),
        "adaptive": (AdaptiveDetector, [dict(adaptive_threshold=2.0, min_scene_len=0.12),
                                        dict(adaptive_threshold=1.5, min_scene_len=4, window_width=1)]),
        "threshold": (ThresholdDetector, [dict(threshold=40, min_scene_len=2, add_final_scene=True),
                                          dict(threshold=30, min_scene_len=0.1, fade_bias=0.5)]),
        "histogram": (HistogramDetector, [dict(threshold=0.1, min_scene_len=0.1), dict(threshold=0.05)]),
        "hash": (HashDetector, [dict(threshold=0.3, min_scene_len=3), dict(threshold=0.2, min_scene_len="0.2s")]),
    }


def _frames(n, seed, w=64, h=36):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    plan = ScenePlan(n, seed=seed, min_len=2 if n < 100 else 36, max_len=9 if n < 100 else 60)
    return render_frames(plan.params, w, h), [int(c) for c in plan.cut_frames]


def _truth(n, plan_cuts, i):
    """Ground truth of an n-frame clip: most of its plan's cuts, some moved by a frame or two, a hard cut at the end
    frame, and fades that straddle its first and its last frame."""
    from pyscenedetect_b200.sweep import GroundTruth
    hard = sorted({c + (i + k) % 3 - 1 for k, c in enumerate(plan_cuts) if k % 4 != 3} | {n})
    fades = [(-2, 0), (max(0, n - 2), n + 4)] if i % 2 else [(n - 1, n + 1)]
    return GroundTruth([c for c in hard if c >= 0], fades=fades)


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, scene_manager, sweep
    lib = sweep_clip_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", clip_twin.ClipEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(clips, "DeviceBuffer", clip_twin.Buffer)
    monkeypatch.setattr(sweep, "DeviceBuffer", clip_twin.Buffer)
    # buffers far enough apart that a pointer into a large one is not taken for the next one
    monkeypatch.setattr(clip_twin, "_ids", itertools.count(1 << 32, 1 << 28))
    return lib


@pytest.fixture(scope="module")
def clip_set():
    out = []
    for i, n in enumerate(CLIP_LENGTHS):
        frames, cuts = _frames(n, seed=11 * i + 1)
        out.append((frames, RATES[i % 2], _truth(n, cuts, i)))
    return out


def _streams(clip_set):
    from pyscenedetect_b200.video import ArrayVideoStream
    return [ArrayVideoStream(f, fps) for f, fps, _ in clip_set]


def _expect(cls, grid, clip_set):
    """Per (cell, clip): (predicted list, hard counts per tolerance, fade counts) from one SceneManager each."""
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    out = {}
    for k, params in enumerate(grid):
        for j, (frames, fps, gt) in enumerate(clip_set):
            sm = SceneManager(batch_size=BATCH)
            sm.add_detector(cls(**params))
            sm.detect_scenes(ArrayVideoStream(frames, fps))
            preds = sweep_model.predicted_list([c.frame_num for c in sm.get_cut_list()], len(frames))
            scores = [sweep_model.score(preds, gt.hard_cuts, gt.fades, t) for t in TOLS]
            out[k, j] = (preds, [s[0] for s in scores], scores[0][1])
    return out


def _check(r, want, n_cells, clip_set):
    th = np.zeros((n_cells, len(TOLS), 5), np.int64)
    tf = np.zeros((n_cells, 3), np.int64)
    for (k, j), (preds, hard, fades) in want.items():
        assert r.end_frame(j) == len(clip_set[j][0])
        assert r.cuts(k, j) == preds, (k, j)
        for q, t in enumerate(TOLS):
            assert r.hard(k, j, t) == hard[q][:3]
            assert r.hard_offset(k, j, t) == (float(hard[q][3]), hard[q][4])
            th[k, q] += hard[q]
        assert r.fades(k, j) == fades
        tf[k] += fades
        assert r.raw_count(k, j) >= max(0, len(preds) - 1)
    for k, tot in enumerate(r.totals()):
        for q, t in enumerate(TOLS):
            e = tot.hard[t]
            assert (e.matched, e.false_positives, e.missed) == tuple(th[k, q, :3])
            assert tot.hard_offset[t] == (float(th[k, q, 3]), int(th[k, q, 4]))
        assert (tot.fades.matched, tot.fades.false_positives, tot.fades.missed) == tuple(tf[k])


@pytest.mark.parametrize("kind", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_run_clips_equals_scene_manager_per_cell_and_clip(twin, clip_set, kind):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()[kind]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    r = sw.run_clips(_streams(clip_set), [gt for _, _, gt in clip_set])
    assert len(r) == len(grid) and r.n_clips == len(clip_set)
    want = _expect(cls, grid, clip_set)
    assert any(w[0] for w in want.values()), "the clips must have cuts to compare"
    _check(r, want, len(grid), clip_set)
    assert sw.videos == len(clip_set)
    assert [t.hard for t in sw.totals()] == [t.hard for t in r.totals()]
    assert [t.fades for t in sw.totals()] == [t.fades for t in r.totals()]
    assert twin.launches["psd_clip_eval"] == 3  # one pass: one call


def test_split_passes_and_tiny_cut_buffer_change_nothing(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]
    base = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    r0 = base.run_clips(_streams(clip_set), gts)
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 10)
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 0)
    twin.launches.clear()
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    r1 = sw.run_clips(_streams(clip_set), gts)
    assert twin.launches["psd_clip_eval"] > 3  # several passes
    assert twin.launches["psd_clip_cuts"] > twin.launches["psd_clip_eval"]  # and retries
    for k in range(len(grid)):
        for j in range(len(clip_set)):
            assert r1.cuts(k, j) == r0.cuts(k, j)
            assert r1.raw_count(k, j) == r0.raw_count(k, j)
            assert r1.fades(k, j) == r0.fades(k, j)
            assert all(r1.hard_offset(k, j, t) == r0.hard_offset(k, j, t) for t in TOLS)
    assert [(t.hard, t.fades) for t in sw.totals()] == [(t.hard, t.fades) for t in base.totals()]


def test_without_ground_truth_totals_stay(twin, clip_set):
    from pyscenedetect_b200.sweep import ParameterSweep
    cls, grid = _grids()["histogram"]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    r = sw.run_clips(_streams(clip_set[:3]))
    assert sw.videos == 0 and all(t.hard[0].matched == t.fades.missed == 0 for t in sw.totals())
    # against empty truths every prediction is a false positive
    for k in range(len(grid)):
        assert r.totals()[k].hard[1].false_positives == sum(len(r.cuts(k, j)) for j in range(3))


def test_refusals_leave_totals(twin, clip_set):
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    cls, grid = _grids()["content"]
    gts = [gt for _, _, gt in clip_set]
    sw = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH)
    sw.run_clips(_streams(clip_set[:2]), gts[:2])
    before = ([(t.hard, t.fades) for t in sw.totals()], sw.videos)

    def same():
        return ([(t.hard, t.fades) for t in sw.totals()], sw.videos) == before

    with pytest.raises(ValueError, match="ground truths"):
        sw.run_clips(_streams(clip_set), gts[:-1])
    assert same()
    with pytest.raises(ValueError):
        sw.run_clips(_streams(clip_set[:2]), [gts[0], None])
    assert same()
    empty = ArrayVideoStream(np.zeros((0, 36, 64, 3), np.uint8), 25)
    with pytest.raises(ValueError, match="clip 2 has no frames"):
        sw.run_clips(_streams(clip_set[:2]) + [empty], gts[:2] + [GroundTruth([])])
    assert same()
    small = ParameterSweep(cls, grid, tolerances=TOLS, batch_size=BATCH, max_cuts_per_cell=2)
    small.run_clips(_streams(clip_set[:1]), gts[:1])  # one frame: no cut
    before = ([(t.hard, t.fades) for t in small.totals()], small.videos)
    with pytest.raises(RuntimeError, match=r"cell 0 \(.*\) found \d+ cuts in clip 7, more than max_cuts_per_cell=2"):
        small.run_clips(_streams(clip_set), gts)
    assert ([(t.hard, t.fades) for t in small.totals()], small.videos) == before


def test_c_abi_rejects_bad_arguments_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    one = (C.c_int32 * 1)(1)
    nine = (C.c_int32 * 9)(*range(9))
    p = 4096
    need = sweep_clip_twin.workspace_bytes(2, 3, 1, 10, 4, 2)

    def call(*, cuts=p, offsets=p, n_cells=2, n_clips=3, total=10, max_cuts=16, ends=p, gt=p, n_gt=4, fades=p,
             n_fades=2, tols=one, n_tol=1, ws=p, ws_bytes=need, outs=(p, p, p, p, p), over=p):
        return lib.psd_clip_eval(cuts, offsets, n_cells, n_clips, total, max_cuts, ends, p, gt, n_gt, p, fades,
                                 n_fades, tols, n_tol, ws, ws_bytes, *outs, over, None)

    assert call(offsets=None) == _capi.PSD_ERR_INVALID
    assert call(cuts=None) == _capi.PSD_ERR_INVALID
    assert call(gt=None) == _capi.PSD_ERR_INVALID
    assert call(fades=None) == _capi.PSD_ERR_INVALID
    assert call(over=None) == _capi.PSD_ERR_INVALID
    assert call(outs=(None, p, p, p, p)) == _capi.PSD_ERR_INVALID
    assert call(outs=(p, p, p, None, p)) == _capi.PSD_ERR_INVALID
    assert call(n_cells=-1) == _capi.PSD_ERR_INVALID
    assert call(max_cuts=-1) == _capi.PSD_ERR_INVALID
    assert call(max_cuts=1 << 31) == _capi.PSD_ERR_INVALID
    assert call(tols=nine, n_tol=9) == _capi.PSD_ERR_INVALID
    assert b"tolerances" in lib.psd_last_error()
    assert call(tols=None) == _capi.PSD_ERR_INVALID
    assert call(tols=(C.c_int32 * 1)(-1)) == _capi.PSD_ERR_INVALID
    assert call(ws_bytes=need - 1) == _capi.PSD_ERR_INVALID
    assert f"workspace needs {need} bytes".encode() in lib.psd_last_error()
    assert call(ws=None) == _capi.PSD_ERR_INVALID


def test_workspace_size_is_the_header_formula():
    from pyscenedetect_b200.sweep import clip_eval_workspace_bytes
    for args in ((1, 1, 1, 0, 0, 0), (2, 3, 1, 10, 4, 2), (1024, 455, 3, 98765, 1234, 17), (7, 1, 8, 33, 32, 31)):
        assert clip_eval_workspace_bytes(*args) == sweep_clip_twin.workspace_bytes(*args)


def test_new_kernels_do_not_spill():
    import os
    import re
    import shutil
    import subprocess
    from pyscenedetect_b200 import _capi
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([tool, "-res-usage", _capi.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    found = {}
    pat = r"Function (\S*(?:clip_pred_kernel|clip_eval_kernel|clip_totals_kernel|psd_sweep_eval_kernel|" \
          r"psd_sweep_pred_kernel)\S*):\s*\n\s*REG:\d+ STACK:(\d+)"
    for fn, stack in re.findall(pat, out):
        found[fn] = stack
    assert len(found) == 5, out[:2000]
    assert all(s == "0" for s in found.values()), found

