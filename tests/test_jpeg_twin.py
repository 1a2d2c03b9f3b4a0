"""The numpy restatement of the baseline JPEG encoder (tests/jpeg_twin.py) writes the bytes cv2.imencode writes on
the whole parity matrix (tests/jpeg_cases.py), and the reciprocal quantisation it restates equals rounding division
wherever it can be reached."""

from __future__ import annotations

import cv2
import numpy as np
import pytest

from tests import jpeg_cases as K
from tests import jpeg_twin as J


def cv2_jpeg(bgr, q):
    return cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


@pytest.mark.parametrize("width,height", K.SIZES)
def test_twin_equals_cv2(width, height):
    for c, w, h, q in K.cases(large=True):
        if (w, h) != (width, height):
            continue
        f = K.frame(c, w, h)
        assert J.encode(f, q) == cv2_jpeg(f, q), (c, w, h, q)


def test_matrix_reaches_stuffing_zrl_and_largest_dc():
    f = K.frame("stuffing", 37, 53)
    assert J.encode(f, 100).count(b"\xff\x00") > 10
    coefs = J.mcu_coefficients(K.frame("zrl", 37, 53), 50)
    runs = [np.diff(np.concatenate([[0], np.nonzero(b[1:])[0] + 1])) - 1 for b in coefs]
    assert max(r.max() for r in runs if len(r)) >= 16   # a ZRL ahead of some coefficient
    dc = J.mcu_coefficients(K.frame("dc_jump", 64, 64), 100)[:, 0]
    assert np.abs(np.diff(dc[::6])).max() >= 1024   # luma DC differences of category 11


def test_reciprocal_equals_rounding_division():
    """|x| -> ((|x| + corr) * recip) >> shift equals (|x| + d // 2) // d for every divisor 8 * q and every
    magnitude the islow FDCT can produce (below 2^14)"""
    a = np.arange(1 << 14, dtype=np.int64)
    for q in range(1, 256):
        d = 8 * q
        recip, corr, shift = J.reciprocal(d)
        assert np.array_equal(((a + corr) * recip) >> shift, (a + d // 2) // d), q
