"""`detect_clips` without a GPU: the oracle-backed engine of tests/fake_engine.py scores the frames and the Python
twin of the clip kernels (tests/clip_twin.py) stands in for the library, so what is checked here is the host side -
grouping, feeding, clip tables, passes, cut lists and scene lists - against one `SceneManager` per clip on the same
engine.  The kernels themselves are checked against one-clip engines in tests/test_gpu_clips.py."""

from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_twin

W, H = 64, 36
BATCH = 16
WINDOW = 2  # AdaptiveDetector's default window_width
LENGTHS = [0, 1, 2, 2 * WINDOW, 2 * WINDOW + 1, BATCH - 1, BATCH, BATCH + 1, 300]
RATES = [25, Fraction(30000, 1001)]


def _detectors(name):
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    return {
        "content": lambda: [ContentDetector(threshold=20.0, min_scene_len=0.2)],
        "adaptive": lambda: [AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=0.12)],
        "threshold": lambda: [ThresholdDetector(threshold=40, min_scene_len=2, add_final_scene=True)],
        "histogram": lambda: [HistogramDetector(threshold=0.1, min_scene_len=0.1)],
        "hash": lambda: [HashDetector(threshold=0.3, min_scene_len=3)],
        "mix": lambda: [ContentDetector(threshold=20.0, min_scene_len=0.2),
                        AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=4),
                        HistogramDetector(threshold=0.1), HashDetector(threshold=0.3, min_scene_len=0.3),
                        ThresholdDetector(threshold=40, min_scene_len=0.1)],
    }[name]()


def _frames(n, seed, w=W, h=H):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    if n == 0:
        return np.zeros((0, h, w, 3), np.uint8)
    # long scenes in long clips, so that some fade to black (ThresholdDetector)
    return render_frames(ScenePlan(n, seed=seed, min_len=2 if n < 100 else 36, max_len=9 if n < 100 else 60).params, w, h)


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, scene_manager
    lib = clip_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", clip_twin.ClipEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(clips, "DeviceBuffer", clip_twin.Buffer)
    clip_twin.ClipEngine.submissions = []
    return lib


def _scene_manager(dets, video, **kw):
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(batch_size=kw.get("batch_size", BATCH))
    sm.auto_downscale = kw.get("auto_downscale", True)
    for d in dets:
        sm.add_detector(d)
    n = sm.detect_scenes(video)
    return sm, n


def _check(results, arrays, name, **kw):
    from pyscenedetect_b200.video import ArrayVideoStream
    assert len(results) == len(arrays)
    for r, (frames, fps) in zip(results, arrays):
        sm, n = _scene_manager(_detectors(name), ArrayVideoStream(frames, fps), **kw)
        assert r.frames == n == len(frames)
        want = [c.frame_num for c in sm.get_cut_list()]
        assert r.cut_frames == want, (name, len(frames), r.cut_frames, want)
        assert [c.frame_num for c in r.cut_list()] == want
        assert all(c.framerate == sm.get_cut_list()[0].framerate for c in r.cut_list()[:1])
        for sis in (False, True):
            got = [(a.frame_num, b.frame_num) for a, b in r.scene_list(start_in_scene=sis)]
            exp = [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list(start_in_scene=sis)]
            assert got == exp, (name, len(frames), sis)


@pytest.mark.parametrize("name", ["content", "adaptive", "threshold", "histogram", "hash", "mix"])
def test_detect_clips_equals_scene_manager_per_clip(twin, name):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    arrays = [(_frames(n, seed=11 * i + 1), RATES[i % 2]) for i, n in enumerate(LENGTHS)]
    dets = _detectors(name)
    results = detect_clips([ArrayVideoStream(f, fps) for f, fps in arrays], dets, batch_size=BATCH)
    assert any(r.cut_frames for r in results), "the clips must have cuts to compare"
    _check(results, arrays, name)
    assert all(d._engine is None for d in dets)  # configuration only: never attached


def test_host_batches_span_clips(twin):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = _frames(10, seed=5, w=32, h=18)
    results = detect_clips([ArrayVideoStream(frames, 25) for _ in range(200)], _detectors("threshold"),
                           batch_size=64)
    assert len(clip_twin.ClipEngine.submissions) == math.ceil(2000 / 64)
    assert sum(clip_twin.ClipEngine.submissions) == 2000
    assert all(r.frames == 10 for r in results)


def test_groups_keep_input_order_and_passes_end_at_clip_boundaries(twin, monkeypatch):
    from pyscenedetect_b200 import clips
    from pyscenedetect_b200.video import ArrayVideoStream
    sizes = [(W, H), (48, 27), (W, H), (48, 27), (W, H)]
    lengths = [7, 30, 0, 12, 25]
    arrays = [(_frames(n, seed=3 + i, w=w, h=h), 25) for i, ((w, h), n) in enumerate(zip(sizes, lengths))]
    held = []
    finish = clips._Pass.finish

    def spy(self, engine, holders, done):
        held.append((engine.frame_count, [m for _, m in done]))
        return finish(self, engine, holders, done)

    monkeypatch.setattr(clips._Pass, "finish", spy)
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 5)
    results = clips.detect_clips([ArrayVideoStream(f, fps) for f, fps in arrays], _detectors("mix"),
                                 batch_size=BATCH)
    # group (64, 36): clips 0, 2, 4; group (48, 27): clips 1, 3.  Each pass ends after the clip that reached the bound
    assert held == [(7, [7]), (25, [0, 25]), (30, [30]), (12, [12])]
    _check(results, arrays, "mix")


def test_tiny_first_cut_buffer_grows_once(twin, monkeypatch):
    from pyscenedetect_b200 import clips
    from pyscenedetect_b200.video import ArrayVideoStream
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 0)
    arrays = [(_frames(n, seed=20 + n), 25) for n in (40, 60)]
    results = clips.detect_clips([ArrayVideoStream(f, fps) for f, fps in arrays], _detectors("mix"),
                                 batch_size=BATCH)
    assert twin.launches["psd_clip_cuts"] == 6  # two calls of three launches: the retry
    _check(results, arrays, "mix")


def test_refusals(twin):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.video import ArrayVideoStream
    video = ArrayVideoStream(_frames(3, seed=1), 25)
    with pytest.raises(ValueError):
        detect_clips([video], [])
    d = ContentDetector()
    d.stats_manager = StatsManager()
    with pytest.raises(ValueError):
        detect_clips([video], [d])
    with pytest.raises(ValueError):
        detect_clips([video], [ContentDetector()], auto_downscale=False, downscale=0)
    with pytest.raises(TypeError):
        detect_clips([video], [object()])
    assert detect_clips([], [ContentDetector()]) == []


def test_c_abi_rejects_bad_arguments_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_clip_fill(4096, 10, None, 1, 1, 0, 0, 0.0, None) == _capi.PSD_ERR_INVALID
    assert b"clip table" in lib.psd_last_error()
    for n, n_clips, head, tail, nan in ((-1, 1, 1, 0, 0), (10, -1, 1, 0, 0), (10, 1, -1, 0, 0), (10, 1, 1, -2, 0),
                                        (10, 1, 1, 0, 2)):
        assert lib.psd_clip_fill(4096, n, 4096, n_clips, head, tail, nan, 0.0, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_fill(None, 10, 4096, 1, 1, 0, 0, 0.0, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_fill(None, 0, 4096, 1, 1, 0, 0, 0.0, None) == _capi.PSD_OK  # nothing to do, no launch

    cells = (_capi.PsdSweepCell * 1)()
    cells[0].kind, cells[0].metric = _capi.SWEEP_CONTENT, 4096
    args = [4096, 4096, 1, 4096, 4096, 16, 4096, None]
    assert lib.psd_clip_cuts(cells, 1, None, *args[1:]) == _capi.PSD_ERR_INVALID
    assert b"clip table" in lib.psd_last_error()
    assert lib.psd_clip_cuts(cells, 1, 4096, 4096, -1, *args[3:]) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_cuts(cells, -1, *args) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_cuts(cells, 1, 4096, 4096, 1, 4096, 4096, -1, 4096, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_cuts(cells, 1, 4096, 4096, 1, 4096, 4096, 16, None, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_cuts(None, 1, *args) == _capi.PSD_ERR_INVALID
    cells[0].kind = 7
    assert lib.psd_clip_cuts(cells, 1, *args) == _capi.PSD_ERR_INVALID
    assert b"psd_clip_cuts: cell 0: unknown kind" in lib.psd_last_error()
    cells[0].kind, cells[0].window = _capi.SWEEP_ADAPTIVE, 0
    assert lib.psd_clip_cuts(cells, 1, *args) == _capi.PSD_ERR_INVALID
    cells[0].kind, cells[0].mode = _capi.SWEEP_HASH, 1
    assert lib.psd_clip_cuts(cells, 1, *args) == _capi.PSD_ERR_INVALID
    cells[0].kind, cells[0].mode, cells[0].metric = _capi.SWEEP_CONTENT, 0, None
    assert lib.psd_clip_cuts(cells, 1, *args) == _capi.PSD_ERR_INVALID
    # the sweep's own checks are the same code and keep their messages
    cells[0].kind, cells[0].metric = 9, 4096
    assert lib.psd_sweep_cuts(cells, 1, 10, 0, 4096, 4096, 4, None) == _capi.PSD_ERR_INVALID
    assert b"psd_sweep_cuts: cell 0: unknown kind 9" in lib.psd_last_error()


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
    found = 0
    for fn, stack in re.findall(r"Function (\S*psd_clip_\S*):\s*\n\s*REG:\d+ STACK:(\d+)", out):
        found += 1
        assert stack == "0", f"{fn} uses a stack frame"
    assert found == 4, out[:2000]
