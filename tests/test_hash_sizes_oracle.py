"""CPU side of HashDetector at sizes above 16 and hash images above 64x64: the oracle against the cases recorded
from the reference (tests/golden/hash_sizes_v1.json), the folded float64 DCT model against cv2, the hash stride
and the detector's argument range."""

import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from tests import hash_twin as T
from tests.hash_sizes_util import case_names, get_case, near_median
from tests.hash_sizes_util import plan_frames as _frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _factor(case):
    w = case["gen"][1]
    return R.compute_downscale_factor(w) if case.get("auto_downscale") else float(case.get("downscale", 1))


@pytest.mark.parametrize("name", case_names())
def test_oracle_reproduces_recorded_case(name):
    case = get_case(name)
    frames = _frames(case["gen"])
    kw = case["kw"]
    det = R.RefHashDetector(threshold=kw.get("threshold", 0.35), size=kw["size"], lowpass=kw["lowpass"],
                            fps=case["fps"], with_stats=True)
    assert R.run_detector(det, frames, _factor(case)) == case["cuts"]
    got = {t: float(v[det.metric_key]).hex() for t, v in det.metrics.items()}
    assert got == {int(t): v[0] for t, v in case["metrics"].items()}


def phash_bits_columns(bgr, size, factor):
    """intmath.phash_bits with the column loops vectorised (same per-column accumulation order): the stage twin
    of the device hash, tests/hash_twin.py."""
    return T.stages(bgr, size, factor).bits.reshape(size, size)


@pytest.mark.parametrize("shape,size,lowpass", [((160, 90), 8, 2), ((131, 97), 4, 2), ((64, 64), 16, 4),
                                                ((120, 90), 17, 1), ((100, 100), 12, 8)])
def test_vectorised_model_equals_intmath(shape, size, lowpass):
    w, h = shape
    frames = _frames((3, w, h, size, 1, 2, 30))
    for f in frames:
        assert np.array_equal(phash_bits_columns(f, size, lowpass), M.phash_bits(f, size, lowpass))


@pytest.mark.parametrize("name", case_names())
def test_model_equals_cv2_on_recorded_sizes(name):
    """The folded float64 model equals cv2 except where a coefficient is within float32 rounding of the median."""
    case = get_case(name)
    kw = case["kw"]
    frames = _frames(case["gen"])[:4]
    for i, f in enumerate(frames):
        f = R.downscale_frame(f, _factor(case))
        want = R.hash_frame(f, kw["size"], kw["lowpass"]).ravel()
        diff = phash_bits_columns(f, kw["size"], kw["lowpass"]).ravel() != want
        if diff.any():
            near, bound = near_median(f, kw["size"], kw["lowpass"])
            assert not (diff & ~near).any(), (i, int(diff.sum()), bound)


def test_hash_words_match_header_macro(tmp_path):
    from pyscenedetect_b200._capi import HASH_WORDS, hash_words
    assert HASH_WORDS == 4 and [hash_words(s) for s in (1, 8, 16, 17, 32, 256)] == [4, 4, 4, 5, 16, 1024]
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to evaluate include/psd_b200.h"
    src = tmp_path / "w.c"
    src.write_text('#include <stdio.h>\n#include "psd_b200.h"\n'
                   'int main(void) { for (int s = 1; s <= 300; ++s) printf("%d\\n", PSD_HASH_WORDS_FOR(s)); }\n')
    exe = tmp_path / "w"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [hash_words(s) for s in range(1, 301)]


def test_hash_detector_accepts_reference_range():
    from pyscenedetect_b200.detectors import HashDetector
    for size, lowpass in ((32, 3), (17, 1), (256, 1), (100, 10), (1, 256), (256, 256)):
        det = HashDetector(size=size, lowpass=lowpass)
        assert det.engine_kwargs() == {"hash_size": size, "hash_lowpass": lowpass}
        assert det.get_metrics() == [f"hash_dist [size={size} lowpass={lowpass}]"]
    for size, lowpass in ((0, 2), (8, 0), (-1, 1)):
        with pytest.raises(ValueError):
            HashDetector(size=size, lowpass=lowpass)
