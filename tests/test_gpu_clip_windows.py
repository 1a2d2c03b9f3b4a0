"""`detect_clips` with `crop`, `frame_skip`, `duration` and `end_time` on the GPU (clips.py, psd_clip_cuts_step):

* psd_clip_cuts_step with step 1 equals psd_clip_cuts bit for bit, and with a step it equals the stepped twin
  (tests/clip_window_twin.py), on the recorded metric arrays of the adversarial sequences;
* every clip's result equals one `SceneManager` per clip running `detect_scenes` with the same window and crop, for
  numpy clips (pageable and page-locked), CUDA `ArrayVideoStream` clips read as views (BGR, RGB and an NCHW
  permutation) and CUDA streams without `read_batch`;
* ThresholdDetector's fade placements and add_final_scene on skipped frames, AdaptiveDetector with skips, stats with
  a crop and a duration byte for byte, a lowered per-pass bound, launches per pass that do not grow with the clip
  count, and the reference's recorded SceneManager settings as the middle clip of a pass."""

from __future__ import annotations

import gzip
import io
import json
import os
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_window_cases, clip_window_twin

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
BATCH = 16
LENGTHS = [0, 1, BATCH - 1, BATCH, BATCH + 1, 300]
RATES = [25, Fraction(30000, 1001)]
SOURCES = ["host", "pinned", "cuda", "read_only"]
WINDOWS = {
    "skip1": dict(frame_skip=1),
    "skip2": dict(frame_skip=2),
    "skip7": dict(frame_skip=7),
    "dur_int": dict(duration=40),
    "dur_float": dict(duration=1.3),
    "dur_str": dict(duration="0.5s"),
    "end_time": dict(end_time=3.0),
    "crop": dict(crop=(7, 5, 120, 70)),
    "skip2_dur": dict(frame_skip=2, duration=2.1),
    "all": dict(frame_skip=3, duration="6s", crop=(8, 2, 147, 83)),
}


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


# -- 1. the step entry point on adversarial metric sequences -----------------------------------------------------------
def _upload(a):
    from pyscenedetect_b200.engine import DeviceBuffer
    b = DeviceBuffer(max(8, a.nbytes))
    if a.nbytes:
        b.upload(np.ascontiguousarray(a))
    return b


def _run(lib, entry, cells, k, sizes, first, mf, step=None, end=None):
    """(offsets, cuts) from psd_clip_cuts or psd_clip_cuts_step, with a buffer large enough in one call."""
    from pyscenedetect_b200.engine import DeviceBuffer
    c = len(sizes)
    bufs = [_upload(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)), _upload(first), _upload(mf)]
    ebuf = _upload(end) if end is not None else None
    cap = 1 << 20
    cuts, obuf = DeviceBuffer(cap * 8), DeviceBuffer((k * c + 1) * 8)
    try:
        args = [cells, k, bufs[0].ptr, bufs[1].ptr, c, bufs[2].ptr, cuts.ptr, cap, obuf.ptr]
        if entry == "psd_clip_cuts":
            rc = lib.psd_clip_cuts(*args, None)
        else:
            rc = lib.psd_clip_cuts_step(*args, step, ebuf.ptr if ebuf else None, None)
        assert rc == 0, lib.psd_last_error()
        offs = obuf.download((k * c + 1) * 8).view(np.int64)
        total = int(offs[-1])
        assert total <= cap
        return offs.tobytes(), cuts.download(total * 8).tobytes()
    finally:
        for b in bufs + [cuts, obuf] + ([ebuf] if ebuf else []):
            b.close()


def _lists(offs: bytes, cuts: bytes) -> list:
    o, v = np.frombuffer(offs, np.int64), np.frombuffer(cuts, np.int64)
    return [v[o[t]:o[t + 1]].tolist() for t in range(len(o) - 1)]


@pytest.mark.parametrize("step", [1, 2, 3, 8])
def test_step_entry_on_adversarial_sequences(lib, step):
    for kind, _w, sizes, metric, metric2, params in clip_window_cases.groups():
        mbuf = _upload(metric)
        m2 = _upload(metric2) if metric2 is not None else None
        c = len(sizes)
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, mbuf.ptr, m2.ptr if m2 else None, c,
                                                              seed=step)
        first, end = clip_window_cases.first_and_end(sizes, step, seed=10 + step)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        try:
            if step == 1:
                want = _run(lib, "psd_clip_cuts", cells, k, sizes, first, mf)
                assert _run(lib, "psd_clip_cuts_step", cells, k, sizes, first, mf, 1) == want, kind
                assert _run(lib, "psd_clip_cuts_step", cells, k, sizes, first, mf, 1, end) == want, kind
                assert any(_lists(*want)), kind
                continue
            for e in (None, end):
                got = _lists(*_run(lib, "psd_clip_cuts_step", cells, k, sizes, first, mf, step, e))
                # the twin reads the metric arrays from its own memory: give it host copies at the same pointers
                twin_cells = (type(cells[0]) * k)(*cells)
                with _TwinMemory(metric, metric2, twin_cells):
                    want = clip_window_twin.clip_cut_lists(twin_cells, k, off, first, c, mf, step, e)
                assert got == want, (kind, step, e is None)
        finally:
            mbuf.close()
            if m2:
                m2.close()


class _TwinMemory:
    """Host copies of the metric arrays registered in the twin's memory, the cells pointed at them."""

    def __init__(self, metric, metric2, cells):
        from tests import clip_twin
        self._bufs = [clip_twin.Buffer(max(8, metric.nbytes))]
        self._bufs[0].upload(metric)
        if metric2 is not None:
            self._bufs.append(clip_twin.Buffer(max(8, metric2.nbytes)))
            self._bufs[1].upload(metric2)
        for c in cells:
            c.metric = self._bufs[0].ptr
            c.metric2 = self._bufs[1].ptr if metric2 is not None else None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for b in self._bufs:
            b.close()


def test_step_entry_rejects_bad_steps(lib):
    from pyscenedetect_b200 import _capi
    cells = (_capi.PsdSweepCell * 1)()
    cells[0].kind, cells[0].metric = _capi.SWEEP_CONTENT, 4096
    for step in (0, -1):
        assert lib.psd_clip_cuts_step(cells, 1, 4096, 4096, 1, 4096, 4096, 16, 4096, step, None, None) \
            == _capi.PSD_ERR_INVALID
        assert b"psd_clip_cuts_step: frame_step must be >= 1" in lib.psd_last_error()


# -- 2. detect_clips against one SceneManager per clip -------------------------------------------------------------------
def _render(n, w, h, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    if n == 0:
        return np.zeros((0, h, w, 3), np.uint8)
    return render_frames(ScenePlan(n, seed=seed, min_len=2 if n < 100 else 36, max_len=12 if n < 100 else 60).params,
                         w, h)


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
                        ContentDetector(weights=ContentDetector.Components(1.0, 1.0, 1.0, 1.0), kernel_size=7,
                                        threshold=25.0),
                        AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=4, window_width=3),
                        HistogramDetector(threshold=0.1, bins=64), HashDetector(threshold=0.3, min_scene_len=0.3),
                        HashDetector(size=16, threshold=0.25), ThresholdDetector(threshold=40, min_scene_len=0.1)],
    }[name]()


def _clip_set(lengths=LENGTHS, seed=0):
    sizes = [(160, 90), (200, 96)]
    return [(_render(n, *sizes[(i // 2) % 2], seed=seed + 13 * i + 2), RATES[i % 2]) for i, n in enumerate(lengths)]


class _ReadOnlyStream:
    """A CUDA stream with `read()` only (no read_batch)."""

    def __init__(self, frames, fps, channel_order="bgr"):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._inner = ArrayVideoStream(frames, fps, channel_order=channel_order)

    frame_rate = property(lambda self: self._inner.frame_rate)
    frame_size = property(lambda self: self._inner.frame_size)
    frame_number = property(lambda self: self._inner.frame_number)
    position = property(lambda self: self._inner.position)
    base_timecode = property(lambda self: self._inner.base_timecode)
    channel_order = property(lambda self: self._inner.channel_order)

    def __dlpack_device__(self):
        return self._inner.__dlpack_device__()

    def read(self, decode=True):
        return self._inner.read(decode)


_PINNED = []  # page-locked copies stay alive for the module


def _streams(clips, source):
    import torch
    from pyscenedetect_b200.engine import PinnedBuffer
    from pyscenedetect_b200.video import ArrayVideoStream
    out = []
    for i, (f, fps) in enumerate(clips):
        if source == "host":
            out.append(ArrayVideoStream(f, fps))
        elif source == "pinned":
            p = PinnedBuffer(max(1, f.nbytes))
            _PINNED.append(p)
            a = p.array[:f.nbytes].reshape(f.shape)
            a[...] = f
            out.append(ArrayVideoStream(a, fps, pinned=True))
        else:
            layout = i % 3
            if layout == 0:
                t, order = torch.from_numpy(f).cuda(), "bgr"
            elif layout == 1:
                t, order = torch.from_numpy(np.ascontiguousarray(f[..., ::-1])).cuda(), "rgb"
            else:
                nchw = np.ascontiguousarray(f[..., ::-1].transpose(0, 3, 1, 2))
                t, order = torch.from_numpy(nchw).cuda().permute(0, 2, 3, 1), "rgb"
            cls = _ReadOnlyStream if source == "read_only" else ArrayVideoStream
            out.append(cls(t, fps, channel_order=order))
    return out


def _per_clip(dets_fn, video, window, stats=False):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager() if stats else None, batch_size=BATCH)
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
    start = sm._start_pos.frame_num if sm._start_pos is not None else None
    end = sm._last_pos.frame_num if sm._last_pos is not None else None
    return (n, [c.frame_num for c in sm.get_cut_list()],
            [[(a.frame_num, b.frame_num) for a, b in sm.get_scene_list(start_in_scene=s)] for s in (0, 1)],
            start, end, text)


def _got(r, stats=False):
    return (r.frames, r.cut_frames,
            [[(a.frame_num, b.frame_num) for a, b in r.scene_list(start_in_scene=s)] for s in (0, 1)],
            r.start.frame_num if r.start is not None else None, r.end.frame_num if r.end is not None else None,
            r.stats_csv if stats else None)


def _compare(clips, source, dets_fn, window, stats=False, **kw):
    from pyscenedetect_b200.clips import detect_clips
    results = detect_clips(_streams(clips, source), dets_fn(), batch_size=BATCH, stats=stats, **window, **kw)
    want = [_per_clip(dets_fn, v, window, stats) for v in _streams(clips, source)]
    got = [_got(r, stats) for r in results]
    for j, (g, w) in enumerate(zip(got, want)):
        assert g == w, (j, window, source)
    return results


@pytest.mark.parametrize("window", list(WINDOWS))
@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("name", ["content", "adaptive", "threshold", "histogram", "hash", "mix"])
def test_windows_equal_scene_manager_per_clip(lib, name, source, window):
    results = _compare(_clip_set(), source, lambda: _detectors(name), WINDOWS[window])
    if name != "threshold":
        assert any(r.cut_frames for r in results)


@pytest.mark.parametrize("source", SOURCES)
def test_streams_already_advanced_and_edge_windows(lib, source):
    clips = _clip_set(seed=3)
    for window in (dict(duration=10_000), dict(duration=0), dict(end_time=0, frame_skip=2), dict(frame_skip=1000),
                   dict(duration=25, frame_skip=2, crop=(3, 3, 100, 60))):
        _compare(clips, source, lambda: _detectors("mix"), window)
    from pyscenedetect_b200.clips import detect_clips
    for window in (dict(frame_skip=2), dict(duration=30), dict(end_time=2.0, frame_skip=1)):
        streams = _streams(clips, source)
        again = _streams(clips, source)
        for s, t in zip(streams, again):
            for _ in range(7):
                s.read()
                t.read()
        results = detect_clips(streams, _detectors("mix"), batch_size=BATCH, **window)
        assert [_got(r) for r in results] == [_per_clip(lambda: _detectors("mix"), v, window) for v in again]


@pytest.mark.parametrize("source", ["host", "cuda"])
@pytest.mark.parametrize("skip", [1, 2, 5])
def test_threshold_fade_bias_and_adaptive_with_skips(lib, source, skip):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ThresholdDetector
    clips = _clip_set([300, 7, 120, 301, 0, 45], seed=5)
    for bias in (-1.0, 0.0, 0.5, 1.0, 1.5):
        def dets(bias=bias):
            return [ThresholdDetector(threshold=40, min_scene_len=3, fade_bias=bias, add_final_scene=True),
                    ThresholdDetector(threshold=40, min_scene_len=9, fade_bias=bias, add_final_scene=True,
                                      method=ThresholdDetector.Method.CEILING)]
        results = _compare(clips, source, dets, dict(frame_skip=skip))
        if bias not in (-1.0, 1.0):
            assert any((c - r.start.frame_num) % (skip + 1) for r in results for c in r.cut_frames)
    for w in (1, 2, 4):
        _compare(clips, source, lambda: [AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=6, window_width=w)],
                 dict(frame_skip=skip))


def test_add_final_scene_sees_the_end_position(lib):
    from pyscenedetect_b200.detectors import ThresholdDetector
    frames = np.full((33, 64, 36, 3), 200, np.uint8)
    frames[10:20] = 0
    frames[25:] = 0
    for source in ("host", "cuda"):
        for min_len in (10, 11, 12, 13):
            results = _compare([(frames, 25), (frames[:32], 25), (frames[:31], 25)], source,
                               lambda: [ThresholdDetector(threshold=40, min_scene_len=min_len, add_final_scene=True)],
                               dict(frame_skip=4))
            if min_len in (11, 12):
                assert 25 in results[0].cut_frames and 25 not in results[2].cut_frames


@pytest.mark.parametrize("source", SOURCES)
def test_stats_with_crop_and_duration(lib, source):
    clips = _clip_set(seed=9)
    for window in (dict(crop=(7, 5, 120, 70)), dict(duration="1.5s"), dict(end_time=40, crop=(9, 9, 60, 50))):
        results = _compare(clips, source, lambda: _detectors("mix"), window, stats=True)
        assert all(r.stats_csv.startswith(b"Frame Number,Timecode,") for r in results)


@pytest.mark.parametrize("source", ["host", "cuda"])
def test_lowered_pass_bound(lib, monkeypatch, source):
    from pyscenedetect_b200 import clips as clips_mod
    passes = []
    finish = clips_mod._Pass.finish

    def spy(self, engine, holders, done):
        passes.append(engine.frame_count)
        finish(self, engine, holders, done)

    monkeypatch.setattr(clips_mod._Pass, "finish", spy)
    monkeypatch.setattr(clips_mod, "MAX_PASS_FRAMES", 7)
    clips = _clip_set([3, 9, 0, 1, 16, 5, 30, 40, 17, 300], seed=11)
    for window in (WINDOWS["skip2"], WINDOWS["dur_float"], WINDOWS["all"], dict(frame_skip=1, end_time=20)):
        _compare(clips, source, lambda: _detectors("mix"), window)
    assert len(passes) > 12


def test_pass_launches_do_not_depend_on_the_clip_count(lib, monkeypatch):
    import torch
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = torch.from_numpy(_render(2000, 64, 36, seed=4)).cuda()
    counts = []
    finish = clips_mod._Pass.finish

    def spy(self, engine, holders, done):
        before = lib.psd_launch_count()
        finish(self, engine, holders, done)
        counts.append(lib.psd_launch_count() - before)

    monkeypatch.setattr(clips_mod._Pass, "finish", spy)
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 4.0)  # no retry of psd_clip_cuts in either arm
    for window in (dict(frame_skip=2, crop=(2, 1, 60, 34)), dict(duration=0.5), dict(frame_skip=1, end_time=9)):
        counts.clear()
        for n_clips in (1, 1000):
            k = 2000 // n_clips
            streams = [ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)]
            clips_mod.detect_clips(streams, _detectors("mix"), batch_size=64, **window)
        assert counts[0] == counts[1] > 0, (window, counts)


# -- 3. the reference's recorded SceneManager settings as the middle clip ----------------------------------------------
def _settings():
    with gzip.open(os.path.join(HERE, "golden", "reference_compat.json.gz"), "rt") as f:
        return json.load(f)["scene_manager_settings"]


@pytest.mark.parametrize("source", ["host", "cuda", "read_only"])
def test_reference_settings_as_the_middle_clip(lib, source):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from tests.golden_util import case_frames, get_case
    frames = case_frames(get_case("content_default_nostats"))
    rev = np.ascontiguousarray(frames[::-1])
    cases = _settings()
    names = {("crop",): 0, ("frame_skip",): 0, ("end_time",): 0}
    for case in cases:
        st = case["settings"]
        for key in names:
            names[key] += key[0] in st
        clips = [(rev[:5], 30), (frames, 30), (rev[-4:], 30)]
        streams = _streams(clips, source)
        for _ in range(st.get("start", 0)):
            streams[1].read()
        window = {k: v for k, v in st.items() if k in ("end_time", "duration", "frame_skip")}
        results = detect_clips(streams, [ContentDetector()], auto_downscale=bool(st.get("auto", False)),
                               batch_size=7, crop=tuple(st["crop"]) if "crop" in st else None, **window)
        r = results[1]
        assert (r.frames, r.cut_frames, [[a.frame_num, b.frame_num] for a, b in r.scene_list()]) == \
            (case["frames"], case["cuts"], case["scenes"]), st
    assert all(names.values()), names
