"""`detect_clips(windows=...)`: a crop, duration / end_time and frame_skip per clip, without a GPU.  The oracle-backed
engine of tests/fake_engine.py scores the frames and the twin library (tests/clip_steps_twin.py, which adds
psd_clip_cuts_steps) stands in for the library.  Every clip's result must be what `detect_clips([clip], **window)`
gives alone and what one `SceneManager` per clip gives from `detect_scenes` with that window and crop: frame count, cut
list, both scene lists, start and end, where the stream stands afterwards, and with `stats=True` the CSV bytes."""

from __future__ import annotations

import io
import itertools
import logging
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_steps_twin, clip_twin, clip_window_cases, clip_window_twin
from tests.test_clip_windows_host import check_clip
from tests.test_clips_host import BATCH, _detectors, _frames

KINDS = ["content", "adaptive", "threshold", "histogram", "hash", "mix"]
# (frames, width, height, rate, how the stream is read): host streams with and without read_batch, and host arrays
# that say they are CUDA memory (read as views of read_batch, as CUDA streams are)
CLIPS = [(40, 64, 36, 25, "host"), (61, 48, 40, Fraction(30000, 1001), "cuda"), (1, 56, 36, 24, "host"),
         (90, 64, 36, 25, "read_only"), (17, 48, 40, 30, "cuda"), (2, 64, 36, 25, "cuda"),
         (75, 56, 36, Fraction(24000, 1001), "read_only"), (33, 48, 40, 25, "host"), (120, 64, 36, 30, "cuda"),
         (0, 56, 36, 25, "host"), (50, 48, 40, 24, "read_only"), (64, 64, 36, 25, "host")]
# (0, 2, 47, 29) and (8, 0, 55, 27) crop every source size above to 48x28; (2, 2, 70, 50) ends outside every frame
CROPS = [None, (0, 2, 47, 29), (8, 0, 55, 27), (5, 3, 50, 30), (60, 33, 1, 3), (2, 2, 70, 50)]
SPANS = [("duration", 20), ("duration", 1.3), ("duration", "0.9s"), ("end_time", 45), ("end_time", 2.5),
         ("end_time", "00:00:01.500")]


class CudaLike:
    """A numpy stream whose frames say they are on the GPU: FrameBatches reads it through views of read_batch."""

    def __init__(self, frames, fps):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._v = ArrayVideoStream(frames, fps)

    def __getattr__(self, name):
        return getattr(self._v, name)

    def __dlpack_device__(self):
        from pyscenedetect_b200 import _dlpack
        return (_dlpack.KDL_CUDA, 0)


class ReadOnly:
    """An ArrayVideoStream without read_batch."""

    def __init__(self, frames, fps):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._v = ArrayVideoStream(frames, fps)

    def __getattr__(self, name):
        if name == "read_batch":
            raise AttributeError(name)
        return getattr(self._v, name)


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, scene_manager
    lib = clip_steps_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", clip_twin.ClipEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(clips, "DeviceBuffer", clip_twin.Buffer)
    clip_twin.ClipEngine.submissions = []
    return lib


@pytest.fixture(scope="module")
def clip_set():
    return [(_frames(n, seed=13 * i + 2, w=w, h=h), fps, how) for i, (n, w, h, fps, how) in enumerate(CLIPS)]


def _streams(clip_set):
    from pyscenedetect_b200.video import ArrayVideoStream
    kinds = {"host": ArrayVideoStream, "cuda": CudaLike, "read_only": ReadOnly}
    return [kinds[how](frames, fps) for frames, fps, how in clip_set]


def random_windows(n, seed, stats=False):
    """None, {} and dicts of a crop (None among them), a frame_skip of 0 to 3 (not with stats) and a duration or an
    end_time as an int, a float or a string."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.12:
            out.append(None)
            continue
        w = {}
        if rng.random() < 0.7:
            w["crop"] = CROPS[rng.integers(len(CROPS))]
        if not stats and rng.random() < 0.7:
            w["frame_skip"] = int(rng.integers(0, 4))
        if rng.random() < 0.7:
            key, value = SPANS[rng.integers(len(SPANS))]
            w[key] = value
        out.append(w)
    return out


def per_clip(dets_fn, video, window, stats=False, auto_downscale=True, downscale=1):
    """What one SceneManager per clip gives: (frames, SceneManager, CSV bytes or None)."""
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager() if stats else None, batch_size=BATCH)
    sm._auto_downscale, sm._downscale = auto_downscale, downscale
    sm.crop = window.get("crop")
    for d in dets_fn():
        sm.add_detector(d)
    n = sm.detect_scenes(video, duration=window.get("duration"), end_time=window.get("end_time"),
                         frame_skip=window.get("frame_skip", 0))
    text = None
    if stats:
        f = io.StringIO()
        sm.stats_manager.save_to_csv(f)
        text = f.getvalue().encode()
    return n, sm, text


def run_lists(dets_fn, clip_set, windows, stats=False, **kw):
    """detect_clips(windows=) against detect_clips per clip and one SceneManager per clip."""
    from pyscenedetect_b200.clips import detect_clips
    dets = dets_fn()
    videos = _streams(clip_set)
    results = detect_clips(videos, dets, batch_size=BATCH, stats=stats, windows=windows, **kw)
    assert len(results) == len(clip_set)
    for j, (r, window) in enumerate(zip(results, windows)):
        window = window or {}
        alone_video = _streams([clip_set[j]])
        alone = detect_clips(alone_video, dets_fn(), batch_size=BATCH, stats=stats, **window, **kw)[0]
        assert (r.frames, r.cut_frames, r.stats_csv) == (alone.frames, alone.cut_frames, alone.stats_csv), (j, window)
        assert [(x.frame_num if x else None) for x in (r.start, r.end)] == \
            [(x.frame_num if x else None) for x in (alone.start, alone.end)]
        video = _streams([clip_set[j]])[0]
        n, sm, text = per_clip(dets_fn, video, window, stats, **kw)
        check_clip(r, n, sm, text, what=(j, window))
        assert videos[j].frame_number == video.frame_number == alone_video[0].frame_number, (j, window)
    assert all(d._engine is None for d in dets)
    return results


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_windows_equal_scene_manager_per_clip(twin, clip_set, kind, seed):
    windows = random_windows(len(clip_set), seed=31 * seed + KINDS.index(kind))
    results = run_lists(lambda: _detectors(kind), clip_set, windows)
    if kind != "threshold":
        assert any(r.cut_frames for r in results), "the clips must have cuts to compare"


@pytest.mark.parametrize("kind", ["content", "adaptive", "threshold", "mix"])
def test_stats_with_crops_and_durations(twin, clip_set, kind):
    windows = random_windows(len(clip_set), seed=7 + KINDS.index(kind), stats=True)
    assert any(w and "crop" in w for w in windows) and any(w and len(w) > 1 for w in windows)
    results = run_lists(lambda: _detectors(kind), clip_set, windows, stats=True)
    assert all(r.stats_csv.startswith(b"Frame Number,Timecode,") for r in results)


def test_windows_over_split_passes(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 9)
    run_lists(lambda: _detectors("mix"), clip_set, random_windows(len(clip_set), seed=99))


def test_fixed_downscale_and_advanced_streams(twin, clip_set):
    """auto_downscale off with a fixed factor, and streams read from past their first frame."""
    from pyscenedetect_b200.clips import detect_clips
    windows = random_windows(len(clip_set), seed=5)
    run_lists(lambda: _detectors("mix"), clip_set, windows, auto_downscale=False, downscale=2)
    videos = _streams(clip_set)
    for v in videos:
        for _ in range(3):
            v.read()
    results = detect_clips(videos, _detectors("mix"), batch_size=BATCH, windows=windows)
    for j, (r, w) in enumerate(zip(results, windows)):
        video = _streams([clip_set[j]])[0]
        for _ in range(3):
            video.read()
        n, sm, _ = per_clip(lambda: _detectors("mix"), video, w or {})
        check_clip(r, n, sm, what=(j, w))


def _engines(monkeypatch):
    from pyscenedetect_b200 import scene_manager
    made = []

    class Counted(clip_twin.ClipEngine):
        def __init__(self, src_width, src_height, features, **kw):
            made.append((src_width, src_height, kw.get("width"), kw.get("height")))
            super().__init__(src_width, src_height, features, **kw)

    monkeypatch.setattr(scene_manager, "Engine", Counted)
    return made


def test_clips_cropped_to_one_size_share_an_engine(twin, clip_set, monkeypatch):
    made = _engines(monkeypatch)
    windows = [{"crop": (0, 2, 47, 29)} if i % 2 else {"crop": (8, 0, 55, 27), "frame_skip": i % 3}
               for i in range(len(clip_set))]
    windows[9] = {"crop": (8, 0, 55, 27)}  # the 56x36 clip without frames
    run_lists(lambda: _detectors("mix"), clip_set, windows)
    # the call's engines come first: host and CUDA-view clips of three source sizes, all cropped to 48x28
    assert made[:2] == [(48, 28, 48, 28)] * 2


def test_scored_size_is_part_of_the_key(twin, monkeypatch):
    """A 256-pixel wide crop scores at 255 wide (its effective size is 257), an uncropped 256-wide frame at 256."""
    made = _engines(monkeypatch)
    clip_set = [(_frames(12, seed=1, w=256, h=16), 25, "host"), (_frames(14, seed=2, w=300, h=16), 25, "host"),
                (_frames(10, seed=3, w=300, h=16), 25, "host"), (_frames(9, seed=4, w=256, h=16), 25, "host")]
    windows = [None, {"crop": (0, 0, 255, 15)}, {"crop": (10, 0, 265, 15), "frame_skip": 1}, {}]
    run_lists(lambda: _detectors("content"), clip_set, windows)
    assert made[:2] == [(256, 16, 256, 16), (256, 16, 255, 16)]


def test_one_automaton_launch_per_pass_whatever_the_steps(twin, clip_set, monkeypatch):
    from pyscenedetect_b200 import clips
    monkeypatch.setattr(clips, "FIRST_CUTS_PER_FRAME", 8.0)  # no retry of the cut buffer
    same = [(f, fps, "host") for f, fps, _ in clip_set if f.shape[1:3] == (36, 64)]
    windows = [{"frame_skip": i % 4, "duration": 30 + i} for i in range(len(same))]
    clips.detect_clips(_streams(same), _detectors("mix"), batch_size=BATCH, windows=windows)
    assert twin.launches["psd_clip_cuts_steps"] == 3 and "psd_clip_cuts" not in twin.launches
    twin.launches.clear()
    skips = [0, 1, 1, 2, 0, 0, 3, 2, 1, 0, 0, 1]
    run_lists(lambda: _detectors("mix"), clip_set, [{"frame_skip": s} for s in skips])
    # five groups (64x36, 56x36, 48x40 host; 48x40, 64x36 CUDA views), each with mixed steps: one launch per pass
    # (the clips run alone by run_lists have one step each)
    assert twin.launches["psd_clip_cuts_steps"] == 3 * 5


def test_equal_steps_keep_the_one_step_entries(twin, clip_set):
    from pyscenedetect_b200.clips import detect_clips
    calls = []
    twin.psd_clip_cuts_step = lambda *a: calls.append(a) or clip_window_twin.Lib.psd_clip_cuts_step(twin, *a)
    windows = [{"frame_skip": 2, "crop": CROPS[i % 4], "duration": 10 + i} for i in range(len(clip_set))]
    detect_clips(_streams(clip_set), _detectors("mix"), batch_size=BATCH, windows=windows)
    assert calls and all(c[9] == 3 for c in calls) and "psd_clip_cuts_steps" not in twin.launches
    calls.clear()
    detect_clips(_streams(clip_set), _detectors("mix"), batch_size=BATCH,
                 windows=[{"crop": CROPS[i % 4], "end_time": 30} for i in range(len(clip_set))])
    assert not calls and "psd_clip_cuts_steps" not in twin.launches and twin.launches["psd_clip_cuts"]


@pytest.mark.parametrize("empty", [None, {}])
def test_empty_windows_are_no_windows(twin, clip_set, empty):
    from pyscenedetect_b200.clips import detect_clips
    want = detect_clips(_streams(clip_set), _detectors("mix"), batch_size=BATCH, stats=True)
    launches, subs = dict(twin.launches), list(clip_twin.ClipEngine.submissions)
    twin.launches.clear()
    clip_twin.ClipEngine.submissions = []
    got = detect_clips(_streams(clip_set), _detectors("mix"), batch_size=BATCH, stats=True,
                       windows=[empty] * len(clip_set))
    assert twin.launches == launches and clip_twin.ClipEngine.submissions == subs
    assert got == want


def test_crop_warnings_once_per_clip(twin, clip_set, caplog):
    windows = [{"crop": (2, 2, 70, 50)} if i % 3 else {"crop": (0, 2, 47, 29)} for i in range(len(clip_set))]
    msg = "Warning: crop ends outside of video boundary."
    from pyscenedetect_b200.clips import detect_clips
    with caplog.at_level(logging.WARNING, logger="pyscenedetect_b200"):
        detect_clips(_streams(clip_set), _detectors("content"), batch_size=BATCH, windows=windows)
    got = sum(r.getMessage() == msg for r in caplog.records)
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger="pyscenedetect_b200"):
        for (frames, fps, _), w in zip(clip_set, windows):
            per_clip(lambda: _detectors("content"), _streams([(frames, fps, "host")])[0], w)
    want = sum(r.getMessage() == msg for r in caplog.records)
    # every (2, 2, 70, 50) clip, and the 48-wide clips cropped to x 0..47
    assert got == want == sum(1 for i, c in enumerate(CLIPS) if i % 3 or c[1] == 48)


def test_refusals(twin):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.scene_manager import SceneManager

    def clips_():
        return [ReadOnly(_frames(3, seed=1), 25), ReadOnly(_frames(3, seed=2, w=16, h=9), 25),
                CudaLike(_frames(4, seed=3), 30)]

    def refused(exc, msg, windows, **kw):
        videos = clips_()
        with pytest.raises(exc) as ei:
            detect_clips(videos, [ContentDetector()], windows=windows, **kw)
        assert str(ei.value) == msg, (windows, kw, str(ei.value))
        assert all(v.frame_number == 0 for v in videos)  # refused before a frame was read

    for kw in (dict(crop=(0, 0, 5, 5)), dict(duration=3), dict(end_time=1.0), dict(frame_skip=1),
               dict(duration=0), dict(end_time=0)):
        refused(TypeError, "detect_clips takes windows or crop / duration / end_time / frame_skip, not both",
                [None] * 3, **kw)
    refused(TypeError, "window 1 has an unknown key 'start': the keys are crop, duration, end_time, frame_skip",
            [None, {"start": 3}, None])
    refused(TypeError, "window 2 must be None or a dict, not tuple", [None, {}, (0, 0, 5, 5)])
    refused(ValueError, "windows has 2 entries for 3 videos", [None, None])
    refused(ValueError, "windows has 4 entries for 3 videos", [None] * 4)
    cases = [
        (dict(duration=5, end_time=5), ValueError, "duration and end_time cannot be set at the same time!"),
        (dict(duration=-1), ValueError, "duration must be greater than or equal to 0!"),
        (dict(duration=-0.5), ValueError, "duration must be greater than or equal to 0!"),
        (dict(end_time=-2), ValueError, "end_time must be greater than or equal to 0!"),
        (dict(frame_skip=1, stats=True), ValueError, "frame_skip must be 0 when using a StatsManager."),
        (dict(crop=(1, 2, 3)), TypeError, "crop region must be tuple of 4 ints"),
        (dict(crop=(1, 2, 3, 4.0)), TypeError, "crop region must be tuple of 4 ints"),
        (dict(crop=(1, -2, 3, 4)), ValueError, "crop coordinates must be >= 0"),
    ]
    for window, exc, msg in cases:
        stats = window.pop("stats", False)
        refused(exc, msg, [{"crop": (0, 0, 3, 3)}, {"frame_skip": 0}, window], stats=stats)
        # the messages are detect_scenes' and the crop setter's
        sm = SceneManager(StatsManager() if stats else None)
        sm.add_detector(ContentDetector())
        with pytest.raises(exc) as ej:
            if "crop" in window:
                sm.crop = window["crop"]
            else:
                sm.detect_scenes(clips_()[0], **window)
        assert str(ej.value) == msg
    refused(ValueError, "crop starts outside video boundary of clip 1 (16x9)",
            [{"crop": (20, 0, 30, 5)}, {"crop": (0, 9, 3, 12)}, None])
    # the scalar arguments keep their refusals
    refused(TypeError, "crop region must be tuple of 4 ints", None, crop=(1, 2, 3))
    assert twin.launches == {}


# -- the per-clip-step twin against the stepped twin --
def test_twin_equal_steps_is_the_step_twin():
    """With every clip at one step, psd_clip_cuts_steps' twin (each clip alone) gives the stepped twin's lists over
    all the clips at once, with and without end frames; with mixed steps each clip's lists are its own step's."""
    for kind, _w, sizes, metric, metric2, params in clip_window_cases.groups():
        mbuf = clip_twin.Buffer(max(8, metric.nbytes))
        mbuf.upload(metric)
        m2 = None
        if metric2 is not None:
            m2 = clip_twin.Buffer(metric2.nbytes)
            m2.upload(metric2)
        c = len(sizes)
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, mbuf.ptr, m2.ptr if m2 else None, c, 3)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        for step in (1, 2, 5):
            first, end = clip_window_cases.first_and_end(sizes, step, 4)
            for e in (None, end):
                want = clip_window_twin.clip_cut_lists(cells, k, off, first, c, mf, step, e)
                assert clip_steps_twin.clip_cut_lists_steps(cells, k, off, first, c, mf, [step] * c, e) == want
        steps = [1 + j % 4 for j in range(c)]
        first, end = clip_window_cases.first_and_end(sizes, 4, 6)
        got = clip_steps_twin.clip_cut_lists_steps(cells, k, off, first, c, mf, steps, end)
        for step in set(steps):
            want = clip_window_twin.clip_cut_lists(cells, k, off, first, c, mf, step, end)
            for t in itertools.product(range(k), range(c)):
                if steps[t[1]] == step:
                    assert got[t[0] * c + t[1]] == want[t[0] * c + t[1]], (kind, t)
        mbuf.close()
        if m2:
            m2.close()
