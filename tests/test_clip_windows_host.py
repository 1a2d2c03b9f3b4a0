"""`detect_clips` with `crop`, `frame_skip`, `duration` and `end_time`, without a GPU: the oracle-backed engine of
tests/fake_engine.py scores the frames and the twin library (tests/clip_window_twin.py, which adds
psd_clip_cuts_step) stands in for the library.  Every clip's result must be what one `SceneManager` per clip gives
from `detect_scenes(video, duration=..., end_time=..., frame_skip=...)` with the same crop, on the same engine: frame
count, cut list, both scene lists, start and end, and with `stats=True` the CSV bytes."""

from __future__ import annotations

import io
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_twin, clip_window_cases, clip_window_twin
from tests.test_clips_host import BATCH, H, W, _detectors, _frames

LENGTHS = [0, 1, BATCH - 1, BATCH, BATCH + 1, 300]
RATES = [25, Fraction(30000, 1001)]
KINDS = ["content", "adaptive", "threshold", "histogram", "hash", "mix"]


def _tc(n, fps):
    from pyscenedetect_b200.compat import FrameTimecode
    return FrameTimecode(n, fps)


WINDOWS = {
    "skip1": dict(frame_skip=1),
    "skip2": dict(frame_skip=2),
    "skip7": dict(frame_skip=7),
    "dur_int": dict(duration=20),
    "dur_float": dict(duration=1.3),
    "dur_str": dict(duration="0.5s"),
    "end_time": dict(end_time=3.0),
    "end_str": dict(end_time="00:00:02.5"),
    "crop": dict(crop=(5, 3, 50, 30)),
    "crop_corners": dict(crop=(60, 30, 2, 4)),
    "skip2_dur": dict(frame_skip=2, duration=2.1),
    "skip1_end_crop": dict(frame_skip=1, end_time=70, crop=(0, 0, 31, 17)),
    "all": dict(frame_skip=3, duration="4s", crop=(8, 2, 47, 33)),
}


@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, scene_manager
    lib = clip_window_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", clip_twin.ClipEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(clips, "DeviceBuffer", clip_twin.Buffer)
    clip_twin.ClipEngine.submissions = []
    return lib


def _streams(arrays, advance=0):
    from pyscenedetect_b200.video import ArrayVideoStream
    out = []
    for frames, fps in arrays:
        v = ArrayVideoStream(frames, fps)
        for _ in range(min(advance, len(frames))):
            v.read()
        out.append(v)
    return out


def per_clip(dets_fn, video, window, stats=False):
    """What one SceneManager per clip gives: (frames, cuts, scene lists, start, end, csv)."""
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager() if stats else None, batch_size=BATCH)
    sm.auto_downscale = True
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


def check_clip(r, n, sm, text=None, what=""):
    assert r.frames == n, what
    want = [c.frame_num for c in sm.get_cut_list()]
    assert r.cut_frames == want, (what, r.cut_frames, want)
    for sis in (False, True):
        got = [(a.frame_num, b.frame_num) for a, b in r.scene_list(start_in_scene=sis)]
        exp = [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list(start_in_scene=sis)]
        assert got == exp, (what, sis)
    if sm._start_pos is None:
        assert r.start is None and r.end is None, what
    else:
        assert r.start.frame_num == sm._start_pos.frame_num, what
        assert r.end.frame_num == sm._last_pos.frame_num, what
    if text is not None:
        assert r.stats_csv == text, (what, r.stats_csv[:300], text[:300])


def run_and_check(dets_fn, arrays, window, stats=False, advance=0, **kw):
    from pyscenedetect_b200.clips import detect_clips
    dets = dets_fn()
    results = detect_clips(_streams(arrays, advance), dets, batch_size=BATCH, stats=stats, **window, **kw)
    assert len(results) == len(arrays)
    for j, (r, video) in enumerate(zip(results, _streams(arrays, advance))):
        n, sm, text = per_clip(dets_fn, video, window, stats)
        check_clip(r, n, sm, text, what=(j, window))
    assert all(d._engine is None for d in dets)
    return results


def _arrays(lengths=LENGTHS, rates=RATES, seed=0):
    return [(_frames(n, seed=seed + 11 * i + 1), rates[i % len(rates)]) for i, n in enumerate(lengths)]


@pytest.mark.parametrize("window", list(WINDOWS))
@pytest.mark.parametrize("kind", KINDS)
def test_windows_equal_scene_manager_per_clip(twin, kind, window):
    results = run_and_check(lambda: _detectors(kind), _arrays(), WINDOWS[window])
    short = "duration" in WINDOWS[window] or "end_time" in WINDOWS[window]
    if kind != "threshold" or not short:  # the first fade to black comes after the shorter windows end
        assert any(r.cut_frames for r in results), "the clips must have cuts to compare"


def test_frame_timecode_duration(twin):
    arrays = _arrays(rates=[25])
    for window in (dict(duration=_tc(17, 25)), dict(end_time=_tc(40, 25), frame_skip=2)):
        run_and_check(lambda: _detectors("mix"), arrays, window)


@pytest.mark.parametrize("window", [dict(duration=10_000), dict(end_time="01:00:00"), dict(duration=0),
                                    dict(duration=0, frame_skip=3), dict(end_time=0), dict(end_time=0.0, frame_skip=1),
                                    dict(frame_skip=1000)])
def test_edge_windows(twin, window):
    """windows longer than the clip, empty windows (the first frame is processed anyway), skips past the end"""
    results = run_and_check(lambda: _detectors("mix"), _arrays(), window)
    if window.get("duration") == 0 or window.get("end_time") in (0, 0.0) or window.get("frame_skip") == 1000:
        assert all(r.cut_frames == [] for r in results)


@pytest.mark.parametrize("window", ["skip2", "dur_int", "end_time", "all"])
def test_streams_already_advanced(twin, window):
    run_and_check(lambda: _detectors("mix"), _arrays(), WINDOWS[window], advance=7)


@pytest.mark.parametrize("bias", [-1.0, 0.0, 0.5, 1.0, 1.5])
@pytest.mark.parametrize("skip", [1, 2, 5])
def test_threshold_placements_on_skipped_frames(twin, bias, skip):
    from pyscenedetect_b200.detectors import ThresholdDetector
    arrays = _arrays(lengths=[300, 7, 120, 301], seed=5)

    def dets():
        return [ThresholdDetector(threshold=40, min_scene_len=3, fade_bias=bias, add_final_scene=True),
                ThresholdDetector(threshold=40, min_scene_len=8, fade_bias=bias, add_final_scene=True,
                                  method=ThresholdDetector.Method.CEILING)]
    results = run_and_check(dets, arrays, dict(frame_skip=skip))
    step = skip + 1
    off_grid = [c for r in results for c in r.cut_frames if (c - r.start.frame_num) % step]
    if bias not in (-1.0, 1.0):
        assert off_grid, "some fade placement must land on a skipped frame"


def test_add_final_scene_sees_the_end_position(twin):
    """A threshold clip whose last fade-out is closer than min_scene_len to the last processed frame but not to the
    stream's position after the frames skipped behind it."""
    from pyscenedetect_b200.detectors import ThresholdDetector
    frames = np.full((33, H, W, 3), 200, np.uint8)
    frames[10:20] = 0
    frames[25:] = 0
    # frame_skip 4 processes 0, 5, .. 30: a fade out at 10, the cut at the fade in at 20, a fade out at 25; the last
    # processed frame is 30 and the position after the loop 32 (31 and 30 for the shorter clips)
    for min_len in range(8, 15):
        results = run_and_check(
            lambda: [ThresholdDetector(threshold=40, min_scene_len=min_len, add_final_scene=True)],
            [(frames, 25), (frames[:32], 25), (frames[:31], 25)], dict(frame_skip=4))
        if min_len in (11, 12):
            assert 25 in results[0].cut_frames and 25 not in results[2].cut_frames


def test_stats_with_crop_and_duration(twin):
    arrays = _arrays()
    for window in (dict(crop=(5, 3, 50, 30)), dict(duration="1.5s"), dict(end_time=40, crop=(9, 9, 40, 20))):
        for kind in ("content", "adaptive", "threshold", "mix"):
            results = run_and_check(lambda: _detectors(kind), arrays, window, stats=True)
            assert all(r.stats_csv.startswith(b"Frame Number,Timecode,") for r in results)


def test_windows_over_split_passes(twin, monkeypatch):
    from pyscenedetect_b200 import clips
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 7)
    arrays = _arrays(lengths=[3, 9, 0, 1, 16, 5, 30, 40, 17], seed=40)
    for window in (WINDOWS["skip2"], WINDOWS["dur_float"], WINDOWS["all"], dict(frame_skip=1, end_time=20)):
        run_and_check(lambda: _detectors("mix"), arrays, window)


def test_host_batches_run_across_clips_with_a_skip(twin):
    frames = _frames(20, seed=5, w=32, h=18)
    arrays = [(frames, 25)] * 30
    results = run_and_check(lambda: _detectors("threshold"), arrays, dict(frame_skip=1))
    assert sum(clip_twin.ClipEngine.submissions) // 2 == 30 * 10  # detect_clips', then the per-clip SceneManagers'
    assert all(r.frames == 20 for r in results)


def test_default_window_launches_psd_clip_cuts(twin):
    from pyscenedetect_b200.clips import detect_clips
    calls = []
    twin.psd_clip_cuts_step = lambda *a: calls.append(a) or clip_window_twin.Lib.psd_clip_cuts_step(twin, *a)
    detect_clips(_streams(_arrays()), _detectors("mix"), batch_size=BATCH, duration=30, crop=(0, 0, 40, 30))
    assert not calls and twin.launches["psd_clip_cuts"] == 3
    detect_clips(_streams(_arrays()), _detectors("mix"), batch_size=BATCH, frame_skip=1)
    assert calls and all(c[9] == 2 for c in calls)  # frame_step (a second call: the cut buffer's retry)


def test_refusals(twin):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.video import ArrayVideoStream

    def clips_():
        return [ArrayVideoStream(_frames(3, seed=1), 25), ArrayVideoStream(_frames(3, seed=2, w=16, h=9), 25)]
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
    for kw, exc, msg in cases:
        with pytest.raises(exc) as ei:
            detect_clips(clips_(), [ContentDetector()], **kw)
        assert str(ei.value) == msg, kw
        # the messages are detect_scenes' and the crop setter's
        from pyscenedetect_b200 import StatsManager
        from pyscenedetect_b200.scene_manager import SceneManager
        sm = SceneManager(StatsManager() if kw.get("stats") else None)
        sm.add_detector(ContentDetector())
        with pytest.raises(exc) as ej:
            if "crop" in kw:
                sm.crop = kw["crop"]
            else:
                sm.detect_scenes(clips_()[0], **{k: v for k, v in kw.items() if k != "stats"})
        assert str(ej.value) == msg
    videos = clips_()
    with pytest.raises(ValueError, match=r"crop starts outside video boundary of clip 1"):
        detect_clips(videos, [ContentDetector()], crop=(20, 0, 30, 5))
    assert all(v.frame_number == 0 for v in videos)  # refused before a frame was read
    assert twin.launches == {}


# -- the stepped automata twin against clip_twin's at step 1 --
def test_twin_step_one_is_clip_twin():
    """On the adversarial metric sequences, the stepped twin with step 1 and no end frames gives clip_twin's lists,
    and with end frames at the last element + 1 too."""
    for kind, _w, sizes, metric, metric2, params in clip_window_cases.groups():
        mbuf = clip_twin.Buffer(max(8, metric.nbytes))
        mbuf.upload(metric)
        m2 = None
        if metric2 is not None:
            m2 = clip_twin.Buffer(metric2.nbytes)
            m2.upload(metric2)
        c = len(sizes)
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, mbuf.ptr, m2.ptr if m2 else None, c, 1)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        first, _ = clip_window_cases.first_and_end(sizes, 1, 2)
        want = []
        for kk in range(k):
            for j in range(c):
                out = []
                clip_twin.run_cell(cells[kk], int(off[j]), sizes[j], int(first[j]), int(mf[kk * c + j]), out)
                want.append(out)
        assert clip_window_twin.clip_cut_lists(cells, k, off, first, c, mf, 1, None) == want, kind
        assert clip_window_twin.clip_cut_lists(cells, k, off, first, c, mf, 1, first + np.maximum(sizes, 1)) == want
        assert any(want), kind
        mbuf.close()
        if m2:
            m2.close()


def test_reference_settings_as_the_middle_clip(twin):
    """The reference's recorded SceneManager settings (end_time, duration, frame_skip, crop, an advanced stream) on
    golden case content_default_nostats, as the middle clip of three."""
    import gzip
    import json
    import os

    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from tests.golden_util import case_frames, get_case
    from tests.test_reference_scene_manager import FrameStream
    with gzip.open(os.path.join(os.path.dirname(__file__), "golden", "reference_compat.json.gz"), "rt") as f:
        cases = json.load(f)["scene_manager_settings"]
    frames = case_frames(get_case("content_default_nostats"))
    rev = frames[::-1]
    for case in cases:
        st = case["settings"]
        streams = [FrameStream(rev[:5]), FrameStream(frames), FrameStream(rev[-4:])]
        for _ in range(st.get("start", 0)):
            streams[1].read(decode=False)
        window = {k: v for k, v in st.items() if k in ("end_time", "duration", "frame_skip")}
        r = detect_clips(streams, [ContentDetector()], auto_downscale=bool(st.get("auto", False)), batch_size=7,
                         crop=tuple(st["crop"]) if "crop" in st else None, **window)[1]
        assert (r.frames, r.cut_frames, [[a.frame_num, b.frame_num] for a, b in r.scene_list()]) == \
            (case["frames"], case["cuts"], case["scenes"]), st
