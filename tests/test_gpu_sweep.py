"""GPU tests of the parameter sweep (psd_sweep_cuts / psd_sweep_eval through `ParameterSweep`): the
reference's per-cell scene lists and evaluator counts recorded in tests/golden/sweep_v1.json, the batched
automata against the single-cell psd_cuts_* kernels on a large random grid, pixel groups against
separate SceneManager runs, totals over several videos, and overflow."""

import ctypes as C
import json
import os
import random

import numpy as np
import pytest

from tests import sweep_model

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "sweep_v1.json")) as f:
        return json.load(f)


def _cls(name):
    from pyscenedetect_b200 import detectors as D
    return {"content": D.ContentDetector, "adaptive": D.AdaptiveDetector, "threshold": D.ThresholdDetector,
            "histogram": D.HistogramDetector, "hash": D.HashDetector}[name]


def _kw(kw):
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import ContentDetector, ThresholdDetector
    kw = dict(kw)
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    if "filter_mode" in kw:
        kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
    if "method" in kw:
        kw["method"] = ThresholdDetector.Method[kw["method"]]
    return kw


def _frames(gen):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    n, w, h, seed, mn, mx, ns = gen
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    return plan, render_frames(plan.params, w, h)


def _want(r, k, tols):
    return {str(t): {"hard": [*r.hard(k, t), int(r.hard_offset(k, t)[0]), r.hard_offset(k, t)[1]],
                     "fades": list(r.fades(k))} for t in tols}


@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_reference_grids(lib, golden, det):
    """Every recorded cell's predicted list (benchmark/sweep.py:169) and its score_video counts."""
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    g = next(x for x in golden["grids"] if x["det"] == det)
    _, frames = _frames(g["gen"])
    tols = golden["tolerances"]
    sw = ParameterSweep(_cls(det), [_kw(c["kw"]) for c in g["cells"]], tolerances=tols, batch_size=48)
    r = sw.run(ArrayVideoStream(frames, g["fps"]), GroundTruth(g["true_cuts"], [tuple(f) for f in g["fades"]]))
    for k, cell in enumerate(g["cells"]):
        assert r.cuts(k) == cell["pred"], (k, cell["kw"])
        assert _want(r, k, tols) == cell["want"], (k, cell["kw"])


def _eval_one(lib, raw, end, hard, fades, tols, cap=None):
    """psd_sweep_eval on one cell whose cut slice holds `raw` (any order, repeats allowed)."""
    from pyscenedetect_b200.engine import DeviceBuffer
    cap = max(1, len(raw)) if cap is None else cap
    cuts = DeviceBuffer(cap * 8)
    if raw:
        cuts.upload(np.asarray(raw, dtype=np.int64))
    count = DeviceBuffer(8)
    count.upload(np.asarray([len(raw)], dtype=np.int32))
    gt = DeviceBuffer(max(8, 8 * len(hard)))
    if hard:
        gt.upload(np.asarray(hard, dtype=np.int64))
    fb = DeviceBuffer(max(16, 16 * len(fades)))
    if fades:
        fb.upload(np.asarray(fades, dtype=np.int64).reshape(-1, 2))
    words = -(-(cap + 1) // 32) + -(-len(hard) // 32) + -(-len(fades) // 32)
    ws = DeviceBuffer(len(tols) * 4 * words + 8)
    n_pred, out_h, out_f = DeviceBuffer(8), DeviceBuffer(len(tols) * 40), DeviceBuffer(24)
    t = (C.c_int32 * len(tols))(*tols)
    rc = lib.psd_sweep_eval(cuts.ptr, count.ptr, 1, cap, end, gt.ptr, len(hard), fb.ptr, len(fades), t, len(tols),
                            ws.ptr, ws.nbytes, n_pred.ptr, out_h.ptr, out_f.ptr, None)
    assert rc == 0, lib.psd_last_error()
    npred = int(n_pred.download(4).view(np.int32)[0])
    h = out_h.download(len(tols) * 40).view(np.int64).reshape(len(tols), 5)
    f = out_f.download(24).view(np.int64)
    pred = cuts.download(max(0, npred - 1) * 8).view(np.int64).tolist() + [end] if npred > 0 else []
    return npred, pred, h, f


def test_evaluator_cases(lib, golden):
    """Every recorded score_video case, with the cut slice shuffled and one cut repeated, so the device's
    sort and de-duplication are exercised too."""
    tols = golden["tolerances"]
    rng = random.Random(7)
    for case in golden["evaluator"]:
        preds = case["preds"]
        raw = list(preds[:-1])
        if raw:
            raw.append(rng.choice(raw))
            rng.shuffle(raw)
        end = preds[-1] if preds else 0
        npred, pred, h, f = _eval_one(lib, raw, end, case["hard"], case["fades"], tols)
        assert pred == preds and npred == len(preds), case["name"]
        for q, t in enumerate(tols):
            assert h[q].tolist() == case["want"][str(t)]["hard"], (case["name"], t)
            assert f.tolist() == case["want"][str(t)]["fades"], (case["name"], t)


def _random_grid(det, rng, n):
    grid = []
    for _ in range(n):
        msl = rng.choice([0, 1, 5, 15, 30, 0.5, "0.8s"])
        if det == "content":
            kw = dict(threshold=rng.choice([8.0, 15.0, 27.0, 40.0, 60.0]) + rng.random(), min_scene_len=msl,
                      weights=rng.choice([(1.0, 1.0, 1.0, 0.0), (0.5, 1.0, 2.0, 0.0), (1.0, 1.0, 1.0, 1.0)]),
                      kernel_size=rng.choice([None, 3, 5]))
            if rng.random() < 0.3:
                kw["filter_mode"] = "SUPPRESS"
        elif det == "adaptive":
            kw = dict(adaptive_threshold=rng.choice([1.5, 2.0, 3.0, 4.0]) + rng.random(), min_scene_len=msl,
                      window_width=rng.choice([1, 2, 3, 5]), min_content_val=rng.choice([5.0, 15.0]),
                      luma_only=rng.random() < 0.2)
        elif det == "threshold":
            kw = dict(threshold=rng.choice([8, 12, 40, 100, 140]), min_scene_len=msl,
                      fade_bias=rng.choice([-1.0, -0.5, 0.0, 0.3, 1.0, 1.5, -1.5]),
                      add_final_scene=rng.random() < 0.5, method=rng.choice(["FLOOR", "CEILING"]))
        elif det == "histogram":
            kw = dict(threshold=rng.choice([0.02, 0.05, 0.1, 0.2, 0.4]), bins=rng.choice([16, 100, 128, 256]),
                      min_scene_len=msl)
        else:
            kw = dict(threshold=rng.choice([0.1, 0.2, 0.3, 0.4]) + 0.01 * rng.random(), min_scene_len=msl,
                      size=rng.choice([8, 16]))
        grid.append(kw)
    return grid


def test_random_grid_equals_single_cell_kernels(lib):
    """~2 000 mixed cells over 20 000 frames at 256x144: batched cuts identical to the single-cell psd_cuts_*
    result of the same detector, counts identical to tests/sweep_model.py."""
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import DeviceBuffer, synth_frames_device
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan
    n, w, h, fps = 20000, 256, 144, 30.0
    plan = ScenePlan(n, seed=3, min_len=10, max_len=90)
    fbytes = w * h * 3
    frames = DeviceBuffer(n * fbytes)
    for i in range(0, n, 2000):
        synth_frames_device(frames.ptr + i * fbytes, plan.params[i:i + 2000], w, h)
    rng = random.Random(2026)
    gt = GroundTruth(plan.cut_frames, [(c - 3, c + 3) for c in plan.cut_frames[5::17]] + [(100, 400), (300, 350)])
    tols = (0, 1, 3)
    total = 0
    for det, count in (("content", 600), ("adaptive", 500), ("threshold", 300), ("histogram", 300), ("hash", 300)):
        grid = _random_grid(det, rng, count)
        kws = [_kw(k) for k in grid]
        sw = ParameterSweep(_cls(det), kws, tolerances=tols, batch_size=512, max_cuts_per_cell=n)
        engines = [g.make_engine(w, h, w, h, max_batch=512) for g in sw.groups]
        for e in engines:
            e.submit_device(frames.ptr, n, fbytes)
        r = sw.run_scored(engines, fps, gt)
        for k, kw in enumerate(kws):
            e = engines[sw.cells[k].metric[1]]
            raw = cuts_for_detector(DeviceCuts(e, max_cuts=n), _cls(det)(**kw), fps)
            if det != "threshold" or abs(kw["fade_bias"]) <= 1.0:
                assert raw == sorted(set(raw)), (det, kw)  # strictly increasing (cut_automata.cuh)
            assert r.raw_count(k) == len(raw), (det, kw)
            pred = sweep_model.predicted_list(raw, n)
            assert r.cuts(k) == pred, (det, kw)
            for t in tols:
                want_h, want_f = sweep_model.score(pred, gt.hard_cuts, gt.fades, t)
                assert (*r.hard(k, t), int(r.hard_offset(k, t)[0]), r.hard_offset(k, t)[1]) == want_h, (det, kw, t)
                assert r.fades(k) == want_f, (det, kw)
        for e in engines:
            e.close()
        total += len(grid)
    assert total == 2000


def _scene_manager_pred(det, frames, fps):
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    sm = SceneManager()
    sm.add_detector(det)
    sm.detect_scenes(ArrayVideoStream(frames, fps))
    return [s[1].frame_num for s in sm.get_scene_list()]


def test_pixel_groups_equal_separate_scene_manager_runs(lib):
    """kernel_size 3 and 5 (edge weight 1) and hash size 8 and 16, each in one run; 320x180 frames are
    auto-downscaled to 256x144 first, as SceneManager does."""
    from pyscenedetect_b200.detectors import ContentDetector, HashDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    _, frames = _frames((240, 320, 180, 12, 15, 60, 30))
    for cls, grid in (
            (ContentDetector, [dict(weights=(1.0, 1.0, 1.0, 1.0), kernel_size=k, threshold=t, min_scene_len=m)
                               for k in (3, 5) for t in (20.0, 30.0) for m in (0, 10)] + [dict(threshold=20.0)]),
            (HashDetector, [dict(size=s, threshold=t, min_scene_len=m) for s in (8, 16) for t in (0.2, 0.35)
                            for m in (0, 10)])):
        sw = ParameterSweep(cls, grid, batch_size=50)
        assert len(sw.groups) == (3 if cls is ContentDetector else 2)
        r = sw.run(ArrayVideoStream(frames, 30.0))
        for k, kw in enumerate(grid):
            assert r.cuts(k) == _scene_manager_pred(cls(**kw), frames, 30.0), kw


def test_totals_over_three_videos(lib):
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    grid = [dict(threshold=t, min_scene_len=m) for t in (15.0, 27.0, 40.0) for m in (0, 15)]
    sw = ParameterSweep(ContentDetector, grid, tolerances=(0, 2))
    per = []
    for seed in (1, 2, 3):
        plan, frames = _frames((180, 160, 90, seed, 15, 50, 30))
        gt = GroundTruth(plan.cut_frames, [(plan.cut_frames[0] - 2, plan.cut_frames[0] + 2)])
        per.append(sw.run(ArrayVideoStream(frames, 30.0), gt))
    sw.run(ArrayVideoStream(frames, 30.0))  # no ground truth: not counted
    assert sw.videos == 3
    tot = sw.totals()
    for k in range(len(grid)):
        for t in (0, 2):
            assert [tot[k].hard[t].matched, tot[k].hard[t].false_positives, tot[k].hard[t].missed] == \
                [sum(r.hard(k, t)[i] for r in per) for i in range(3)]
            assert tot[k].hard_offset[t] == (sum(r.hard_offset(k, t)[0] for r in per),
                                              sum(r.hard_offset(k, t)[1] for r in per))
        assert [tot[k].fades.matched, tot[k].fades.false_positives, tot[k].fades.missed] == \
            [sum(r.fades(k)[i] for r in per) for i in range(3)]
    assert any(c.hard[2].f1 > 0 for c in tot)


def test_overflowing_cell_raises(lib):
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    _, frames = _frames((120, 160, 90, 0, 20, 70, 30))
    sw = ParameterSweep(ContentDetector, [dict(threshold=27.0), dict(threshold=0.0, min_scene_len=0)],
                        max_cuts_per_cell=16)
    with pytest.raises(RuntimeError, match=r"cell 1 .*max_cuts_per_cell=16"):
        sw.run(ArrayVideoStream(frames, 30.0))
