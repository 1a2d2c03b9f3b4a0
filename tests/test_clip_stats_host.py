"""`detect_clips(stats=True)` and the CSV formatter without a GPU.

* tests/stats_csv_twin.py, the statement-by-statement twin of csrc/stats_csv.cuh, equals `str(float)`,
  `str(numpy.float64)` and `FrameTimecode.get_timecode()`, and its power-of-ten table is the one the header holds.
* With the oracle-backed engine and the twin library (tests/stats_clip_twin.py), every clip's `stats_csv` equals what a
  `SceneManager(StatsManager())` per clip saves, byte for byte, and the cut lists equal `stats=False`'s.
The kernels themselves are checked against the twin and per-clip SceneManagers in tests/test_gpu_clip_stats.py."""

from __future__ import annotations

import io
import math
import os
import re
import struct
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_twin, stats_clip_twin
from tests import stats_csv_twin as T
from tests.test_clips_host import BATCH, LENGTHS, RATES, _detectors, _frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def adversarial_doubles() -> list:
    """Powers of ten and their neighbours, the fixed / exponent switch points, every power of two and its neighbours
    (subnormals included), the extremes, signed zeros, NaNs, infinities and 17-digit values"""
    out = [0.0, -0.0, math.inf, -math.inf, math.nan, -math.nan, 5e-324, 1e-323, 2.2250738585072014e-308,
           2.225073858507201e-308, 1.7976931348623157e308, 0.1, 0.2, 0.30000000000000004, 1 / 3, 2 / 3, 27.0, 255.0,
           9007199254740991.0, 9007199254740992.0, 9007199254740993.0, 1.2345678901234567e-5, 123456789012345.67,
           0.0001, 0.00009999999999999999, 1e-5, 9.999999999999999e15, 1e16, 1.5e16, 999999999999999.9]
    for k in range(-324, 309):
        for m in (1, 2, 5, 9):
            v = float(f"{m}e{k}")
            out += [v, float(np.nextafter(v, 0.0)), float(np.nextafter(v, math.inf))]
    for e in range(-1074, 1024):
        v = math.ldexp(1.0, e)
        out += [v, float(np.nextafter(v, 0.0)), float(np.nextafter(v, math.inf))]
    for t in range(1, 4096):  # the smallest subnormals
        out.append(struct.unpack("<d", struct.pack("<Q", t))[0])
    out = [x for x in out if not math.isinf(x)] + [math.inf, -math.inf]
    return out + [-x for x in out]


def test_formatter_twin_equals_str_on_adversarial_values():
    for x in adversarial_doubles():
        assert T.format_f64(x) == str(x) == str(np.float64(x)), x


def test_formatter_twin_equals_str_on_random_bit_patterns():
    xs = T.random_doubles(1_000_000, seed=1)
    bad = [x for x in xs.tolist() if T.format_f64(x) != str(x)]
    assert not bad, bad[:5]
    sample = xs[:: 50]
    assert all(T.format_f64(x) == str(x) for x in sample.tolist())
    assert [str(x) for x in sample] == [str(x) for x in sample.tolist()]  # numpy.float64 prints as float does


def test_formatter_twin_on_metric_like_values():
    rng = np.random.default_rng(2)
    xs = np.concatenate([rng.random(200_000) * 255.0, rng.random(50_000), rng.integers(0, 64, 20_000) / 64.0,
                         rng.integers(0, 1 << 20, 20_000) / 3.0])
    assert all(T.format_f64(x) == str(x) for x in xs.tolist())


def test_round_millis_is_round_3():
    rng = np.random.default_rng(3)
    xs = rng.random(300_000) * 60.0
    ties = [k / 16 for k in range(0, 960)] + [k / 2048 for k in range(0, 4096)]  # exact binary halves of a millisecond
    for x in xs.tolist() + ties + [59.9995, 59.99949999999999, 59.99950000000001, 0.0005, 0.0015]:
        assert T.round_millis(x) == round(round(x, 3) * 1000), x


@pytest.mark.parametrize("rate", [24, 25, Fraction(30000, 1001), Fraction(60000, 1001), 120])
def test_timecode_twin_equals_get_timecode(rate):
    from pyscenedetect_b200.compat import FrameTimecode
    r = float(Fraction(rate))
    bad = [f for f in range(0, 1_000_001) if T.timecode(f, r) != FrameTimecode(f, rate).get_timecode()]
    assert not bad, bad[:5]


def test_timecode_rounding_edge():
    from pyscenedetect_b200.compat import FrameTimecode
    # 59.9995 s and its neighbours round up into the next minute (and hour) at these rates
    for rate, frames in ((2000, [119999, 120000, 7199999]), (4000, [239998, 239999, 14399999]),
                         (Fraction(30000, 1001), [1798, 1799, 107891, 107892])):
        for f in frames:
            assert T.timecode(f, float(rate)) == FrameTimecode(f, rate).get_timecode(), (rate, f)
    assert T.timecode(119999, 2000.0) == "00:00:59.999"  # 59.9995 is 59.99949999... in binary
    assert T.timecode(239999, 4000.0) == "00:01:00.000"  # 59.99975 carries into the minute
    assert T.timecode(14399999, 4000.0) == "01:00:00.000"  # and the hour


def test_header_table_is_the_twins():
    src = open(os.path.join(ROOT, "pyscenedetect_b200", "csrc", "stats_csv.cuh")).read()
    got = [(int(a, 16), int(b, 16)) for a, b in re.findall(r"\{0x([0-9a-f]{16})ull, 0x([0-9a-f]{16})ull\}", src)]
    assert got == T.G and len(got) == T.K_MAX - T.K_MIN + 1


# -- detect_clips(stats=True) against one SceneManager(StatsManager()) per clip --
@pytest.fixture
def twin(monkeypatch):
    from pyscenedetect_b200 import _capi, clips, scene_manager
    lib = stats_clip_twin.Lib()
    monkeypatch.setattr(_capi, "load", lambda: lib)
    monkeypatch.setattr(scene_manager, "Engine", clip_twin.ClipEngine)
    monkeypatch.setattr(scene_manager, "PinnedBuffer", clip_twin.PinnedHost)
    monkeypatch.setattr(clips, "DeviceBuffer", clip_twin.Buffer)
    clip_twin.ClipEngine.submissions = []
    return lib


def _stats_detectors(name):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    if name == "writers":  # several writers of content_val / delta_* / the adaptive ratio: the last one's values stand
        return [AdaptiveDetector(adaptive_threshold=2.0, window_width=3, weights=(1.0, 0.5, 1.0, 0.0)),
                ContentDetector(threshold=20.0, weights=(1.0, 1.0, 1.0, 0.5)),
                AdaptiveDetector(adaptive_threshold=2.5, weights=(0.5, 1.0, 1.0, 0.0), luma_only=True),
                AdaptiveDetector(adaptive_threshold=1.5, window_width=3, weights=(1.0, 1.0, 0.0, 0.0))]
    return _detectors(name)


def reference_csv(dets, frames, fps, batch_size=BATCH) -> tuple[bytes, list]:
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    sm = SceneManager(StatsManager(), batch_size=batch_size)
    for d in dets:
        sm.add_detector(d)
    sm.detect_scenes(ArrayVideoStream(frames, fps))
    f = io.StringIO()
    sm.stats_manager.save_to_csv(f)
    return f.getvalue().encode(), [c.frame_num for c in sm.get_cut_list()]


def _run(name, arrays, stats):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    return detect_clips([ArrayVideoStream(f, fps) for f, fps in arrays], _stats_detectors(name), batch_size=BATCH,
                        stats=stats)


@pytest.mark.parametrize("name", ["content", "adaptive", "threshold", "histogram", "hash", "mix", "writers"])
def test_stats_csv_equals_scene_manager_per_clip(twin, name):
    arrays = [(_frames(n, seed=11 * i + 1), RATES[i % 2]) for i, n in enumerate(LENGTHS)]
    results = _run(name, arrays, stats=True)
    plain = _run(name, arrays, stats=False)
    assert any(r.cut_frames for r in results)
    for r, p, (frames, fps) in zip(results, plain, arrays):
        want, cuts = reference_csv(_stats_detectors(name), frames, fps)
        assert r.stats_csv == want, (name, len(frames), r.stats_csv[:400], want[:400])
        assert r.cut_frames == p.cut_frames == cuts
        assert p.stats_csv is None
    header = results[0].stats_csv
    assert results[0].stats_csv.count(b"\n") == 1 and header.startswith(b"Frame Number,Timecode,")  # empty clip
    if name in ("content", "adaptive", "writers"):
        assert results[1].stats_csv == header  # one frame: no content-family row
    assert twin.launches["psd_clip_stats_csv"] == 3  # one pass


def test_stats_over_split_passes(twin, monkeypatch):
    from pyscenedetect_b200 import clips
    monkeypatch.setattr(clips, "MAX_PASS_FRAMES", 7)
    arrays = [(_frames(n, seed=40 + n), RATES[n % 2]) for n in (3, 9, 0, 1, 16, 5, 30)]
    results = _run("mix", arrays, stats=True)
    for r, (frames, fps) in zip(results, arrays):
        assert r.stats_csv == reference_csv(_stats_detectors("mix"), frames, fps)[0]
    assert twin.launches["psd_clip_stats_csv"] == 3 * 3  # passes [3, 9], [0, 1, 16], [5, 30]


def test_short_text_buffer_grows_once(twin, monkeypatch):
    from pyscenedetect_b200 import clips
    monkeypatch.setattr(clips, "FIRST_STATS_BYTES", (1, 0))
    arrays = [(_frames(n, seed=60 + n), 25) for n in (20, 33)]
    results = _run("mix", arrays, stats=True)
    assert twin.launches["psd_clip_stats_csv"] == 6  # two calls of three launches: the retry
    for r, (frames, fps) in zip(results, arrays):
        assert r.stats_csv == reference_csv(_stats_detectors("mix"), frames, fps)[0]


def test_stats_leaves_detectors_unchanged(twin):
    from pyscenedetect_b200.detectors import ContentDetector
    d = ContentDetector()
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    detect_clips([ArrayVideoStream(_frames(4, seed=1), 25)], [d], stats=True)
    assert d.stats_manager is None and d._engine is None and d.required_features() == 1


def test_c_abi_rejects_bad_arguments_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    cols = (_capi.PsdStatsColumn * 2)()
    cols[0].values, cols[0].stride = 4096, 1
    cols[1].values, cols[1].stride = 4096, 4
    args = [4096, 4096, 4096, 1, 10, 4096, 4096, 64, 4096, None]
    assert lib.psd_clip_stats_csv(cols, 2, None, *args[1:]) == _capi.PSD_ERR_INVALID
    assert b"clip table" in lib.psd_last_error()
    assert lib.psd_clip_stats_csv(cols, 2, *args[:8], None, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_stats_csv(None, 2, *args) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_stats_csv(cols, 0, *args) == _capi.PSD_ERR_INVALID
    assert lib.psd_clip_stats_csv(cols, _capi.STATS_MAX_COLUMNS + 1, *args) == _capi.PSD_ERR_INVALID
    for bad in (dict(n=-1), dict(n_clips=-1), dict(cap=-1)):
        a = list(args)
        a[3 if "n_clips" in bad else 4 if "n" in bad else 7] = -1
        assert lib.psd_clip_stats_csv(cols, 2, *a) == _capi.PSD_ERR_INVALID, bad
    for field, value in (("values", None), ("stride", 0), ("head", -1), ("tail", -1)):
        c = (_capi.PsdStatsColumn * 2)(*cols)
        setattr(c[1], field, value)
        assert lib.psd_clip_stats_csv(c, 2, *args) == _capi.PSD_ERR_INVALID
        assert b"column 1" in lib.psd_last_error()
    a = list(args)
    a[1] = None  # no first frames
    assert lib.psd_clip_stats_csv(cols, 2, *a) == _capi.PSD_ERR_INVALID
    a = list(args)
    a[6] = None  # text buffer with a capacity
    assert lib.psd_clip_stats_csv(cols, 2, *a) == _capi.PSD_ERR_INVALID
    assert lib.psd_test_format_f64(0, None, 4, None) == _capi.PSD_ERR_INVALID
    assert lib.psd_test_format_f64(0, None, 0, None) == _capi.PSD_OK
    assert lib.psd_test_format_f64(0, 4096, -1, 4096) == _capi.PSD_ERR_INVALID


def test_new_kernels_do_not_spill():
    import shutil
    import subprocess
    from pyscenedetect_b200 import _capi
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([tool, "-res-usage", _capi.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    found = dict(re.findall(r"Function (\S*(?:stats_rows_kernel|format_f64_kernel)\S*):\s*\n\s*REG:\d+ STACK:(\d+)",
                            out))
    assert len(found) == 3, out[:2000]
    assert all(s == "0" for s in found.values()), found
