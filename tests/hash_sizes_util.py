"""Helpers of the HashDetector size tests: the recorded cases, and the bits where cv2's float32 DCT may
legitimately disagree with an exact transform."""

from __future__ import annotations

import json
import math
import os

import cv2
import numpy as np
import scipy.fft

from pyscenedetect_b200.synth import ScenePlan, render_frames

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hash_sizes_v1.json")


def golden() -> dict:
    with open(GOLDEN) as f:
        return json.load(f)


def case_names() -> list[str]:
    return [c["name"] for c in golden()["cases"]]


def get_case(name: str) -> dict:
    return next(c for c in golden()["cases"] if c["name"] == name)


def plan_frames(gen) -> np.ndarray:
    n, w, h, seed, mn, mx, ns = gen
    return render_frames(ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx).params, w, h)


def near_median(frame: np.ndarray, size: int, lowpass: int) -> tuple[np.ndarray, float]:
    """(size*size bools, bound): the bits whose coefficient in an independent float64 transform
    (scipy.fft.dctn, norm="ortho") lies within 2 * bound of the float64 median, with
    bound = log2(2n) * 2^-24 * ||x||_2 - float32 rounding per butterfly stage of a fast transform, scaled by the
    norm of the input (= the norm of the orthonormal output).  cv2.dct runs in float32, so its coefficient and
    its median may each be off by that much; only these bits may differ from an exact hash."""
    n = size * lowpass
    gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
    r = cv2.resize(gray, (n, n), interpolation=cv2.INTER_AREA)
    x = (np.float32(r) / (np.max(r) or 1)).astype(np.float64)
    d = scipy.fft.dctn(x, norm="ortho")[:size, :size]
    bound = math.log2(2 * n) * 2.0 ** -24 * float(np.linalg.norm(x))
    return (np.abs(d - np.median(d)) <= 2 * bound).ravel(), bound


def check_recorded_dist(got: dict, case: dict, scored_frames: np.ndarray) -> int:
    """Compare hash_dist per frame ({frame: float}) with the recording.  A value may differ only by the bits of
    frame t and t-1 that `near_median` allows, divided by size * size; returns how many frames differ."""
    kw = case["kw"]
    m = kw["size"] ** 2
    want = {int(t): float.fromhex(v[0]) for t, v in case["metrics"].items() if v[0] is not None}
    assert sorted(got) == sorted(want)
    differ = 0
    for t, w in want.items():
        if got[t] == w:
            continue
        slack = sum(int(near_median(scored_frames[k], kw["size"], kw["lowpass"])[0].sum()) for k in (t - 1, t))
        assert abs(got[t] - w) <= slack / m, (t, got[t], w, slack)
        differ += 1
    return differ
