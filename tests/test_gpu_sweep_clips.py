"""GPU tests of the parameter sweep over many clips (`ParameterSweep.run_clips`: psd_clip_cuts + psd_clip_eval):

* every grid of tests/golden/sweep_v1.json as the middle clip of three gives the reference's recorded predicted lists
  and evaluator counts;
* random grids of a few hundred cells of every detector over about 40 host and CUDA clips of mixed frame sizes and
  rates equal `ParameterSweep.run` per clip, (cell, clip) by (cell, clip), and in total;
* the launches of a pass depend neither on its number of clips nor on its number of cells;
* a tiny first cut buffer (the retry) and a lowered per-pass bound change nothing;
* a (cell, clip) over max_cuts_per_cell raises and leaves the totals as they were."""

from __future__ import annotations

import json
import os
import random
from fractions import Fraction

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TOLS = (0, 1, 3)
RATES = (24, 25, Fraction(30000, 1001), 30)


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


def _cls(name):
    from pyscenedetect_b200 import detectors as D
    return {"content": D.ContentDetector, "adaptive": D.AdaptiveDetector, "threshold": D.ThresholdDetector,
            "histogram": D.HistogramDetector, "hash": D.HashDetector}[name]


def _render(n, w, h, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    plan = ScenePlan(n, seed=seed, min_len=2, max_len=12 if n < 100 else 40)
    return render_frames(plan.params, w, h), [int(c) for c in plan.cut_frames]


def _counts(r, k, *j):
    """Every count of cell k (on clip j for a ClipSweepResult) as one comparable tuple."""
    return (r.cuts(k, *j), r.raw_count(k, *j), [r.hard(k, *j, t) for t in TOLS],
            [r.hard_offset(k, *j, t) for t in TOLS], r.fades(k, *j))


def _totals(sw):
    return [(t.hard, t.hard_offset, t.fades) for t in sw.totals()], sw.videos


# -- 1. the reference's grids as the middle clip of a pass --------------------------------------------------------------
@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_reference_grids_as_the_middle_clip(lib, det):
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
    sw = ParameterSweep(_cls(det), [_kw(c["kw"]) for c in g["cells"]], tolerances=tols, batch_size=48)
    gts = [GroundTruth([3]), GroundTruth(g["true_cuts"], [tuple(f) for f in g["fades"]]), GroundTruth([], [(0, 2)])]
    r = sw.run_clips([ArrayVideoStream(c, g["fps"]) for c in clips], gts)
    for k, cell in enumerate(g["cells"]):
        assert r.cuts(k, 1) == cell["pred"], (k, cell["kw"])
        got = {str(t): {"hard": [*r.hard(k, 1, t), int(r.hard_offset(k, 1, t)[0]), r.hard_offset(k, 1, t)[1]],
                        "fades": list(r.fades(k, 1))} for t in tols}
        assert got == cell["want"], (k, cell["kw"])


# -- 2. random grids over mixed clips against run per clip ---------------------------------------------------------------
def _random_grid(det, n, rng):
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import ThresholdDetector
    msl = lambda: rng.choice([0, 1, 3, 8, 0.1, 0.3, "0.2s", "5"])  # noqa: E731
    out = []
    for _ in range(n):
        if det == "content":
            out.append(dict(threshold=rng.uniform(4, 40), min_scene_len=msl(), luma_only=rng.random() < 0.3,
                            filter_mode=rng.choice([FlashFilter.Mode.MERGE, FlashFilter.Mode.SUPPRESS])))
        elif det == "adaptive":
            out.append(dict(adaptive_threshold=rng.uniform(1.0, 4.0), window_width=rng.randint(1, 4),
                            min_content_val=rng.choice([5.0, 10.0, 15.0]), min_scene_len=msl()))
        elif det == "threshold":
            out.append(dict(threshold=rng.randint(8, 80), fade_bias=rng.uniform(-1.0, 1.0),
                            add_final_scene=rng.random() < 0.5, min_scene_len=msl(),
                            method=rng.choice([ThresholdDetector.Method.FLOOR, ThresholdDetector.Method.CEILING])))
        elif det == "histogram":
            out.append(dict(threshold=rng.uniform(0.02, 0.3), bins=rng.choice([32, 128, 256]), min_scene_len=msl()))
        else:
            out.append(dict(threshold=rng.uniform(0.1, 0.5), size=rng.choice([8, 16]), min_scene_len=msl()))
    return out


def _clip_set(seed, n_clips=40):
    """[(host BGR frames, fps, GroundTruth, source)]: mixed sizes (one auto-downscaled) and rates; source is "host",
    "cuda" (packed BGR) or "rgb" (an NCHW RGB tensor permuted to NHWC)."""
    from pyscenedetect_b200.sweep import GroundTruth
    rng = random.Random(seed)
    sizes = [(160, 90), (96, 54), (640, 360)]
    out = []
    for i in range(n_clips):
        n = rng.choice([1, 2, 3, 5, 9, 16, 17, 40, 90, 150])
        w, h = sizes[i % 3]
        frames, cuts = _render(n, w, h, seed=1000 * seed + i)
        hard = sorted({c + rng.choice([-2, -1, 0, 0, 1]) for c in cuts if rng.random() < 0.8} | {n})
        fades = [(-3, 0)] if rng.random() < 0.3 else []
        if n > 6 and rng.random() < 0.5:
            a = rng.randint(1, n - 3)
            fades.append((a, a + 2))
        fades += [(n - 1, n + 2)] if rng.random() < 0.3 else []
        out.append((frames, RATES[i % 4], GroundTruth([c for c in hard if c >= 0], fades),
                    ("host", "cuda", "rgb")[i % 3 if i % 2 else 0]))
    return out


def _stream(frames, fps, source):
    import torch
    from pyscenedetect_b200.video import ArrayVideoStream
    if source == "host":
        return ArrayVideoStream(frames, fps)
    if source == "cuda":
        return ArrayVideoStream(torch.from_numpy(frames).cuda(), fps)
    rgb = torch.from_numpy(np.ascontiguousarray(frames[..., ::-1].transpose(0, 3, 1, 2))).cuda()
    return ArrayVideoStream(rgb.permute(0, 2, 3, 1), fps, channel_order="rgb")


@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_random_grids_equal_run_per_clip(lib, det):
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(["content", "adaptive", "threshold", "histogram", "hash"].index(det))
    grid = _random_grid(det, 256, rng)
    clips = _clip_set(seed=len(det))
    sw = ParameterSweep(_cls(det), grid, tolerances=TOLS, batch_size=16)
    r = sw.run_clips([_stream(f, fps, src) for f, fps, _, src in clips], [gt for _, _, gt, _ in clips])
    loop = ParameterSweep(_cls(det), grid, tolerances=TOLS, batch_size=16)
    found = 0
    for j, (frames, fps, gt, src) in enumerate(clips):
        # run submits CUDA frames as packed BGR: RGB clips go to it as the same frames in host BGR
        want = loop.run(_stream(frames, fps, "host" if src == "rgb" else src), gt)
        assert r.end_frame(j) == want.end_frame == len(frames)
        for k in range(len(grid)):
            assert _counts(r, k, j) == _counts(want, k), (det, k, j, grid[k], src)
            found += r.raw_count(k, j)
    assert found > 0
    assert _totals(sw) == _totals(loop)
    assert [(t.hard, t.fades) for t in r.totals()] == [(t.hard, t.fades) for t in loop.totals()]


# -- 3. launches per pass ----------------------------------------------------------------------------------------------
def test_pass_launches_do_not_depend_on_clips_or_cells(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 64.0)  # no retry: the same launches whatever the cuts
    frames, cuts = _render(120, 96, 54, seed=9)
    counts = {}
    for n_cells in (8, 512):
        grid = [dict(threshold=5.0 + 30.0 * i / n_cells, min_scene_len=(0, 2, 0.2)[i % 3]) for i in range(n_cells)]
        for n_clips in (3, 30):
            k = 120 // n_clips
            sw = ParameterSweep(ContentDetector, grid, tolerances=TOLS, batch_size=16)
            gts = [GroundTruth([c - i * k for c in cuts if i * k <= c < (i + 1) * k]) for i in range(n_clips)]
            before = lib.psd_launch_count()
            sw.run_clips([ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)], gts)
            counts[n_cells, n_clips] = lib.psd_launch_count() - before
    assert len(set(counts.values())) == 1, counts


# -- 4. the retry and the drain -----------------------------------------------------------------------------------------
def test_tiny_cut_buffer_and_lowered_pass_bound_change_nothing(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(5)
    grid = _random_grid("content", 64, rng)
    clips = _clip_set(seed=11, n_clips=24)

    def run():
        sw = ParameterSweep(_cls("content"), grid, tolerances=TOLS, batch_size=16)
        r = sw.run_clips([_stream(f, fps, src) for f, fps, _, src in clips], [gt for _, _, gt, _ in clips])
        return [[_counts(r, k, j) for j in range(len(clips))] for k in range(len(grid))], _totals(sw)

    want = run()
    passes = []
    cuts = clips_mod._Pass.cuts

    def spy(self, engine, holders, done):
        passes.append(engine.frame_count)
        return cuts(self, engine, holders, done)

    monkeypatch.setattr(clips_mod._Pass, "cuts", spy)
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 0)
    monkeypatch.setattr(clips_mod, "MAX_PASS_FRAMES", 20)
    assert run() == want
    assert len(passes) > 6 and max(passes) >= max(len(f) for f, _, _, _ in clips)  # a long clip is held whole


# -- 5. overflow -------------------------------------------------------------------------------------------------------
def test_overflow_leaves_the_totals(lib):
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    grid = [dict(threshold=200.0), dict(threshold=5.0, min_scene_len=0)]
    sw = ParameterSweep(ContentDetector, grid, tolerances=TOLS, max_cuts_per_cell=4)
    short, _ = _render(3, 96, 54, seed=1)
    sw.run_clips([ArrayVideoStream(short, 25)], [GroundTruth([1])])
    before = _totals(sw)
    frames, cuts = _render(90, 96, 54, seed=2)
    with pytest.raises(RuntimeError, match=r"cell 1 \(.*\) found \d+ cuts in clip 1, more than max_cuts_per_cell=4"):
        sw.run_clips([ArrayVideoStream(short, 25), ArrayVideoStream(frames, 25)], [GroundTruth([]), GroundTruth(cuts)])
    assert _totals(sw) == before
