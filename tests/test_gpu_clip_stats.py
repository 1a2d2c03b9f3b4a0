"""`detect_clips(stats=True)` on the GPU (psd_clip_stats_csv, csrc/stats_csv.cuh):

* the device formatter equals `str()` on 10^7 random bit patterns and the adversarial values, and its twin
  (tests/stats_csv_twin.py) on a sample of them;
* psd_clip_stats_csv on made-up columns, clip tables, large first frames and odd rates equals the twin's text;
* every golden case with recorded stats, as the middle clip of a pass, gives the reference's CSV sha256 (hist_diff
  cases: the bytes of this package's SceneManager, which agree with the reference to 1e-9, not bit for bit);
* 40 mixed host / CUDA clips of varied size and rate equal one `SceneManager(StatsManager())` per clip;
* a short first text buffer (the retry) changes nothing, and the launches a pass adds do not depend on its clip count."""

from __future__ import annotations

import hashlib
import io
from fractions import Fraction

import numpy as np
import pytest

from tests import stats_csv_twin as T
from tests.test_clip_stats_host import adversarial_doubles
from tests.test_gpu_clips import _golden_cases, _render, _source

pytestmark = pytest.mark.gpu
BATCH = 16


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


def device_format(lib, xs: np.ndarray) -> list[str]:
    from pyscenedetect_b200 import _capi
    xs = np.ascontiguousarray(xs, dtype=np.float64)
    out = np.zeros(len(xs) * _capi.F64_TEXT, dtype=np.uint8)
    _capi.check(lib.psd_test_format_f64(0, xs.ctypes.data, len(xs), out.ctypes.data), "psd_test_format_f64")
    return [s.rstrip(b"\0").decode() for s in out.reshape(-1, _capi.F64_TEXT).view(f"S{_capi.F64_TEXT}")[:, 0]]


def test_device_formatter_equals_str_and_twin(lib):
    adv = np.array(adversarial_doubles())
    got = device_format(lib, adv)
    assert got == [str(x) for x in adv.tolist()] == [T.format_f64(x) for x in adv.tolist()]
    xs = T.random_doubles(10_000_000, seed=7)
    got = device_format(lib, xs)
    want = [str(x) for x in xs.tolist()]
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, [(xs[i], got[i], want[i]) for i in bad[:5]]
    assert all(T.format_f64(x) == g for x, g in zip(xs[:200_000].tolist(), got[:200_000]))
    metric = np.random.default_rng(8).random(1_000_000) * 255.0
    assert device_format(lib, metric) == [str(x) for x in metric.tolist()]


def test_stats_kernel_equals_twin_on_made_up_columns(lib):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import DeviceBuffer
    rng = np.random.default_rng(9)
    lengths = [0, 1, 5, 0, 2, 400, 3, 33, 1, 90]
    n = sum(lengths)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    first = np.array([0, 7, 999_000, 0, 1, 1_000_000 - 200, 12, 3_600 * 120 - 10, 5, 86_399 * 30], np.int64)
    rates = np.array([float(Fraction(r)) for r in (24, 25, Fraction(30000, 1001), Fraction(60000, 1001), 120, 4000,
                                                   Fraction(24000, 1001), 120, 2000, 30)])
    values = np.concatenate([T.random_doubles(n, 10), rng.random(n) * 255.0, rng.random(4 * n)])
    spec = [(0, 1, 1, 0), (n, 1, 0, 0), (2 * n, 4, 1, 0), (2 * n + 3, 4, 2, 2), (n, 1, 3, 5)]
    vbuf = DeviceBuffer(values.nbytes)
    vbuf.upload(values)
    table = DeviceBuffer((len(lengths) * 3 + 1) * 8)
    table.upload(np.concatenate([offsets, first, rates.view(np.int64)]))
    rows, cb = DeviceBuffer((n + 1) * 8), DeviceBuffer((len(lengths) + 1) * 8)
    out = DeviceBuffer(1 << 20)
    cols = (_capi.PsdStatsColumn * len(spec))()
    for i, (o, stride, head, tail) in enumerate(spec):
        cols[i] = _capi.PsdStatsColumn(values=vbuf.ptr + 8 * o, stride=stride, head=head, tail=tail)
    c = len(lengths)
    _capi.check(lib.psd_clip_stats_csv(cols, len(spec), table.ptr, table.ptr + (c + 1) * 8, table.ptr + (2 * c + 1) * 8,
                                       c, n, rows.ptr, out.ptr, out.nbytes, cb.ptr, None))
    offs = cb.download((c + 1) * 8).view(np.int64).tolist()
    text = out.download(offs[-1]).tobytes()
    want, want_offs = T.pass_csv([(values[o:], s, h, t) for o, s, h, t in spec], offsets, first, rates)
    for b in (vbuf, table, rows, cb, out):
        b.close()
    assert offs == want_offs
    assert text == want


def _golden_stats_cases():
    return [f"{f}:{c['name']}" for f, c in _golden_cases() if c.get("stats") and f in ("golden_v1", "golden_v2")]


def reference_csv(dets, stream, batch_size, auto_downscale=True, downscale=1) -> tuple[bytes, list]:
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager(), batch_size=batch_size)
    sm.auto_downscale = auto_downscale
    if not auto_downscale:
        sm.downscale = downscale
    for d in dets:
        sm.add_detector(d)
    sm.detect_scenes(stream)
    f = io.StringIO()
    sm.stats_manager.save_to_csv(f)
    return f.getvalue().encode(), [c.frame_num for c in sm.get_cut_list()]


@pytest.mark.parametrize("which", _golden_stats_cases())
def test_golden_case_as_the_middle_clip(lib, which):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.golden_util import case_frames
    from tests.test_gpu_parity import _build
    f, case = next((f, c) for f, c in _golden_cases() if f"{f}:{c['name']}" == which)
    frames = case_frames(case)
    auto = case.get("mode", "scene_manager") == "scene_manager" and bool(case.get("auto_downscale"))
    downscale = 1 if auto else case.get("downscale", 1)
    rev = frames[::-1]
    clips = [rev[:5], frames, rev[-4:]]
    results = detect_clips([ArrayVideoStream(c, case["fps"]) for c in clips], [_build(case)], auto_downscale=auto,
                           downscale=downscale, batch_size=7, stats=True)
    r = results[1]
    assert r.cut_frames == case["cuts"]
    if any(k.startswith("hist_diff") for k in case["metric_keys"]):
        want, _ = reference_csv([_build(case)], ArrayVideoStream(frames, case["fps"]), 7, auto, downscale)
        assert r.stats_csv == want
    else:
        assert r.stats_csv.decode().splitlines()[:4] == case["csv_head"]
        assert hashlib.sha256(r.stats_csv).hexdigest() == case["csv_sha256"]


def _detectors():
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    return [ContentDetector(threshold=20.0, min_scene_len=0.2),
            ContentDetector(weights=ContentDetector.Components(1.0, 1.0, 1.0, 1.0), kernel_size=7, threshold=25.0),
            AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=4, window_width=3),
            AdaptiveDetector(adaptive_threshold=2.0, luma_only=True),
            HistogramDetector(threshold=0.1, bins=64), HashDetector(threshold=0.3, min_scene_len=0.3),
            HashDetector(size=16, threshold=0.25), ThresholdDetector(threshold=40, min_scene_len=0.1)]


def _clips40():
    """(frames, fps, kind) of 40 clips: mixed sizes, lengths (empty ones included), rates, host and CUDA frames"""
    sizes = [(160, 90), (96, 64), (640, 360)]
    rates = [25, Fraction(30000, 1001), 24, Fraction(60000, 1001), 120]
    lengths = [0, 1, 2, 3, 6, 7, 15, 16, 17, 40, 61, 150]
    out = []
    for i in range(40):
        w, h = sizes[i % 3]
        n = lengths[i % len(lengths)]
        out.append((_render(n, w, h, seed=17 * i + 5), rates[i % 5], "host" if i % 4 < 2 else "cuda"))
    return out


def _streams(clips):
    from pyscenedetect_b200.video import ArrayVideoStream
    out = []
    for f, fps, kind in clips:
        if kind == "host":
            out.append(ArrayVideoStream(f, fps))
        else:
            t, order = _source(f, "aligned" if len(f) % 2 else "nchw_rgb")
            out.append(ArrayVideoStream(t, fps, channel_order=order))
    return out


def test_forty_mixed_clips_equal_scene_manager_per_clip(lib):
    from pyscenedetect_b200.clips import detect_clips
    clips = _clips40()
    results = detect_clips(_streams(clips), _detectors(), batch_size=BATCH, stats=True)
    plain = detect_clips(_streams(clips), _detectors(), batch_size=BATCH)
    for r, p, stream in zip(results, plain, _streams(clips)):
        want, cuts = reference_csv(_detectors(), stream, BATCH)
        assert r.stats_csv == want
        assert r.cut_frames == p.cut_frames == cuts
    assert sum(r.stats_csv.count(b"\n") - 1 for r in results) > 900


def test_short_text_buffer_and_split_passes_change_nothing(lib, monkeypatch):
    from pyscenedetect_b200 import clips as clips_mod
    clips = _clips40()[:16]
    want = [r.stats_csv for r in clips_mod.detect_clips(_streams(clips), _detectors(), batch_size=BATCH, stats=True)]
    calls = []
    orig = clips_mod._Pass.stats_csv

    def spy(self, engine, pc):
        before = lib.psd_launch_count()
        out = orig(self, engine, pc)
        calls.append(lib.psd_launch_count() - before)
        return out

    monkeypatch.setattr(clips_mod._Pass, "stats_csv", spy)
    monkeypatch.setattr(clips_mod, "FIRST_STATS_BYTES", (1, 0))
    monkeypatch.setattr(clips_mod, "MAX_PASS_FRAMES", 20)
    got = [r.stats_csv for r in clips_mod.detect_clips(_streams(clips), _detectors(), batch_size=BATCH, stats=True)]
    assert got == want
    assert len(calls) > 3 and calls[0] == 6  # the first pass grows the buffer once: two calls of three launches


def test_pass_launches_do_not_depend_on_the_clip_count(lib, monkeypatch):
    import torch
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = torch.from_numpy(_render(2000, 64, 36, seed=4)).cuda()
    counts = {}
    finish = clips_mod._Pass.finish

    def spy(self, engine, holders, done):
        before = lib.psd_launch_count()
        finish(self, engine, holders, done)
        counts.setdefault(self.columns is not None, []).append(lib.psd_launch_count() - before)

    monkeypatch.setattr(clips_mod._Pass, "finish", spy)
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 8.0)  # no cut-buffer retry: the one clip has more cuts
    for n_clips in (1, 1000):
        k = 2000 // n_clips
        for stats in (False, True):
            streams = [ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)]
            clips_mod.detect_clips(streams, _detectors(), batch_size=64, stats=stats)
    # the stats pass adds the three psd_clip_stats_csv launches (the text buffer is large enough at once)
    assert counts[False][0] == counts[False][1] > 0, counts
    assert counts[True][0] == counts[True][1] == counts[False][0] + 3, counts
