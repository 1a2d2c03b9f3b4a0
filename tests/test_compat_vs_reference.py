"""The minimal boundary types in pyscenedetect_b200/compat.py (used when the real `scenedetect`
package is not importable, e.g. where only this package is installed) behave like the reference's classes for the
constant-frame-rate, frame-number-backed cases the hot path produces.  The reference's results for
the same inputs are stored in tests/golden/reference_compat.json.gz (tests/golden/make_reference_compat.py)."""

import gzip
import io
import os
import random
import zlib
from fractions import Fraction

import pytest

import pyscenedetect_b200.compat as compat_mod

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_compat.json.gz")


@pytest.fixture(scope="module")
def ref():
    import json
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def ours():
    c = compat_mod
    if c.USING_REFERENCE:
        pytest.skip("compat is already delegating to the reference")
    return c


def compare_bits(others, a, b) -> int:
    bits = [(a - b) >= o for o in others] + [a < o for o in others] + [a == b, a >= b]
    return sum(int(v) << i for i, v in enumerate(bits))


@pytest.mark.parametrize("fps", [30.0, 25.0, 24000 / 1001, 29.97, 60.0])
def test_frame_timecode_semantics(ref, ours, fps):
    want = ref["frame_timecode"][repr(fps)]
    rng = random.Random(1)
    for row in want["rows"]:
        a, b = rng.randrange(0, 200000), rng.randrange(0, 200000)
        oa, ob = ours.FrameTimecode(a, fps), ours.FrameTimecode(b, fps)
        frame_num, timecode, seconds, diff, plus7, bits, h = row
        assert oa.frame_num == frame_num and oa.get_timecode() == timecode
        assert oa.seconds == seconds and oa.frame_rate == Fraction(want["frame_rate"])
        assert (oa - ob).frame_num == diff
        assert (oa + 7).frame_num == plus7
        assert compare_bits(ref["others"], oa, ob) == bits, (a, b)
        assert hash(oa) == h
    assert str(ours.FrameTimecode("00:01:02.500", fps)) == want["str_of_timecode"]
    assert ours.FrameTimecode(1.5, fps).frame_num == want["frame_of_1.5s"]


@pytest.mark.parametrize("mode", ["MERGE", "SUPPRESS"])
@pytest.mark.parametrize("length", [15, 0, 1, 40, 0.5, "0.6s", "00:00:00.700", "20"])
def test_flash_filter_sequences(ref, ours, mode, length):
    rng = random.Random(zlib.crc32(f"{mode}|{length}".encode()) & 0xFFFF)
    for fps, want in zip((30.0, 24000 / 1001), ref["flash_filter"][f"{mode}|{length}"]):
        of = ours.FlashFilter(ours.FlashFilter.Mode[mode], length)
        assert of.max_behind == want["max_behind"]
        p = rng.choice([0.05, 0.2, 0.5])
        for t in range(600):
            above = rng.random() < p
            got = [c.frame_num for c in of.filter(ours.FrameTimecode(t, fps), above)]
            assert got == want["cuts"].get(str(t), []), (t, above)


def test_stats_manager_csv(ref, ours):
    want = ref["stats_manager"]
    os_ = ours.StatsManager()
    keys = want["keys"]
    os_.register_metrics(keys)
    rng = random.Random(3)
    import numpy as np
    for t in range(1, 80):
        row = {"content_val": np.float64(rng.random() * 50), "delta_hue": np.float64(rng.random())}
        if t % 3:
            row["adaptive_ratio (w=2)"] = rng.random() * 4
        os_.set_metrics(ours.FrameTimecode(t, 30.0), row)
    assert os_.metrics_exist(ours.FrameTimecode(5, 30.0), ["content_val"]) and not os_.metrics_exist(
        ours.FrameTimecode(0, 30.0), ["content_val"])
    assert os_.get_metrics(ours.FrameTimecode(3, 30.0), keys) == want["metrics_at_3"]
    b = io.StringIO()
    os_.save_to_csv(b)
    assert b.getvalue() == want["csv"]
