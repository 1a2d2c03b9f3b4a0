"""CPU checks of the stage twin of the hash pass (tests/hash_twin.py) at every geometry of the GPU hash matrix: its
bits equal oracle/intmath.py:phash_bits, its area image equals cv2.resize(INTER_AREA), and the engine's libm cosine
table equals numpy's (which the oracle uses), so that a GPU test pinned to the twin is pinned to the oracle."""

import math

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from tests import hash_twin as T
from tests.hash_matrix_cases import AREA_TIES, CASES, SUB_BATCH, WIDE_FRAMES, frame


def _geometries():
    out = {}
    for c in CASES + [SUB_BATCH]:
        for size, lowpass in c.geos:
            out.setdefault((c.W, c.H, size, lowpass), c.content)
    for (w, h), geos in WIDE_FRAMES:
        for size, lowpass in geos:
            out.setdefault((w, h, size, lowpass), ("plan", "hgrad"))
    return [k + (v,) for k, v in sorted(out.items())]


GEOMETRIES = _geometries()


@pytest.mark.parametrize("w,h,size,lowpass,kinds", GEOMETRIES,
                         ids=[f"{g[0]}x{g[1]}-{g[2]}x{g[3]}" for g in GEOMETRIES])
def test_twin_equals_intmath_and_cv2(w, h, size, lowpass, kinds):
    n = size * lowpass
    # intmath's pure-Python DCT costs seconds per frame at large n: one frame there, two content kinds elsewhere
    kinds = kinds[:1] if n > 256 else kinds[:2]
    for i, kind in enumerate(kinds):
        f = frame(kind, w, h, 11 * i + n)
        gray = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
        st = T.stages(f, size, lowpass, gray=gray)
        assert np.array_equal(st.area, cv2.resize(gray, (n, n), interpolation=cv2.INTER_AREA)), kind
        assert np.array_equal(st.bits, M.phash_bits(f, size, lowpass).ravel()), kind
        assert st.words.size == (4 if size <= 16 else (size * size + 63) // 64)
        bits = np.unpackbits(st.words.view(np.uint8), bitorder="little")
        assert np.array_equal(bits[:size * size].astype(bool), st.bits) and not bits[size * size:].any()


def test_libm_cosine_table_equals_numpy():
    for n in sorted({g[2] * g[3] for g in GEOMETRIES} | set(range(1, 257))):
        assert np.array_equal(T.costab(n), np.cos(np.pi * np.arange(4 * n) / (2.0 * n))), n


def test_rows_stage_chain_is_sequential_float32():
    """The float path's row buffer is the first / run / last chain with separate roundings: not a float64 sum, and
    not a fused multiply-add - a row where they differ pins the order."""
    W, n = 131, 21
    rng = np.random.default_rng(5)
    gray = rng.integers(0, 256, (1, W), dtype=np.uint8)
    got = T.rows_stage(gray, n)[0]
    tab = M.area_tab(W, n)
    want = np.zeros(n, np.float32)
    for d, s, a in tab:
        want[d] = np.float32(want[d] + np.float32(np.float32(gray[0, s]) * a))
    assert np.array_equal(got, want)
    exact = np.zeros(n)
    for d, s, a in tab:
        exact[d] += float(gray[0, s]) * float(a)
    assert not np.array_equal(got, exact.astype(np.float32))


def test_integer_rows_are_raw_sums():
    gray = np.arange(4 * 12, dtype=np.uint8).reshape(4, 12)
    rb = T.rows_stage(gray, 4)
    assert rb.dtype == np.float32
    assert np.array_equal(rb.view(np.uint32), gray.astype(np.uint32).reshape(4, 4, 3).sum(axis=2))


def test_median_and_words():
    low = np.array([3, 1, 2, 2], np.float32)
    assert T.median(low) == np.float32(2)
    assert T.median(np.array([1, 2, 4, 8], np.float32)) == np.float32(3)
    assert T.median(np.array([5], np.float32)) == np.float32(5)
    bits = np.zeros(17 * 17, bool)
    bits[[0, 63, 64, 288]] = True
    w = T.pack_words(bits, 17)
    assert w.tolist() == [1 | 1 << 63, 1, 0, 0, 1 << 32]
    assert math.isclose(float(T.costab(2)[1]), math.cos(math.pi / 4))


@pytest.mark.parametrize("wh", sorted(AREA_TIES))
def test_area_tie_frames_pin_the_reciprocal(wh):
    """The matrix's `area_tie` frames hold one integer-path cell whose sum OpenCV rounds through float32(1 / area);
    dividing by the area instead gives another grey level there."""
    W, H = wh
    bw, bh, levels, extra = AREA_TIES[wh]
    f = frame("area_tie", W, H, 0)
    gray = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
    s = int(gray[:bh, :bw].sum(dtype=np.int64))
    assert s == bw * bh * sum(levels) // 2 + extra
    n = W // bw
    size = n if n in (3, 8) else None
    area = cv2.resize(gray, (n, n), interpolation=cv2.INTER_AREA)
    st = T.stages(f, size, 1, gray=gray)
    assert np.array_equal(st.area, area)
    quotient = int(np.rint(np.float32(s) / np.float32(bw * bh)))
    assert int(area[0, 0]) != quotient and int(area[0, 0]) == int(np.rint(np.float32(s) * (np.float32(1) / np.float32(bw * bh))))
