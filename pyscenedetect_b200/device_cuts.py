"""Whole-sequence detection with the cut state machines on the device (SURVEY.md §8(f) N2).

`DeviceCuts(engine)` turns the integer results an `Engine` already holds into cut lists without
any per-frame Python: trailing device scans (psd_scan_*) produce the metric arrays, the psd_cuts_*
automata walk them, and only the cut frame numbers come back.  Constant-frame-rate,
frame-number timecodes (what `VideoStream.position` yields); every `min_scene_len` form is
converted to frames with FrameTimecode's own rounding (common.py:480-486,627-638).
The per-frame Python detectors remain the reference-facing API; tests/test_gpu_parity.py checks
both give the same cuts on the golden cases.
"""

from __future__ import annotations

import ctypes as C
from fractions import Fraction

import numpy as np

from . import _capi
from ._capi import check
from .compat import FrameTimecode, _to_fraction
from .engine import DeviceBuffer, Engine


def flash_filter_frames(length, fps) -> int:
    """FlashFilter's threshold in frames (detector.py:130-137,179-180): ints become seconds with the
    first frame's rate and are compared through round(seconds * rate)."""
    rate: Fraction = _to_fraction(fps)
    if isinstance(length, float):
        secs = length
    elif isinstance(length, str) and not length.strip().isdigit():
        secs = FrameTimecode(length, 100.0).seconds
    elif isinstance(length, FrameTimecode):
        secs = length.seconds
    else:
        n = int(length)
        if n <= 0:
            return 0
        secs = n / float(rate)
    if secs <= 0.0:
        return 0
    return round(secs * rate)


def min_len_frames(length, fps) -> int:
    """`(tc_a - tc_b) >= length` for frame-number timecodes (common.py:627-638)."""
    rate: Fraction = _to_fraction(fps)
    if isinstance(length, int):
        return length
    if isinstance(length, float):
        return round(length * rate)
    if isinstance(length, FrameTimecode):
        return length.frame_num
    if isinstance(length, str):
        return FrameTimecode(length, rate).frame_num if not length.strip().isdigit() else round(
            (int(length) / float(rate)) * rate)
    raise TypeError("unsupported min_scene_len")


class DeviceCuts:
    def __init__(self, engine: Engine, max_cuts: int = 1 << 16):
        self._e = engine
        self._lib = _capi.load()
        self._dev = engine.device
        self._cap = int(max_cuts)
        self._cuts = DeviceBuffer(self._cap * 8, self._dev)
        self._count = DeviceBuffer(8, self._dev)
        self._stream = engine.compute_stream

    def _tmp(self, n_doubles: int) -> DeviceBuffer:
        return DeviceBuffer(max(8, n_doubles * 8), self._dev)

    def _fetch(self) -> list[int]:
        self._e.sync()
        count = int(self._count.download(4).view(np.int32)[0])
        if count > self._cap:
            raise RuntimeError(f"{count} cuts exceed the device cut buffer ({self._cap})")
        return self._cuts.download(count * 8).view(np.int64).tolist() if count else []

    def _content_scores(self, weights, n):
        sums, _ = self._e.device_results()
        val, comps = self._tmp(n), self._tmp(4 * n)
        w = (C.c_double * 4)(*[float(x) for x in weights])
        check(self._lib.psd_scan_content(sums, n, self._e.n_pixels, w, float(sum(abs(x) for x in weights)),
                                         comps.ptr, val.ptr, self._stream), "psd_scan_content")
        return val, comps

    def content(self, weights=(1.0, 1.0, 1.0, 0.0), threshold=27.0, min_scene_len=15, fps=30.0,
                suppress: bool = False, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        val, _comps = self._content_scores(weights, n)
        flags = DeviceBuffer(max(1, n), self._dev)
        check(self._lib.psd_scan_compare(val.ptr, n, float(threshold), 0, flags.ptr, self._stream))
        check(self._lib.psd_cuts_flash_filter(flags.ptr, n, first_frame, flash_filter_frames(min_scene_len, fps),
                                              1 if suppress else 0, self._cuts.ptr, self._count.ptr, self._cap,
                                              self._stream), "psd_cuts_flash_filter")
        return self._fetch()

    def adaptive(self, weights=(1.0, 1.0, 1.0, 0.0), adaptive_threshold=3.0, min_scene_len=15,
                 window_width=2, min_content_val=15.0, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        val, _comps = self._content_scores(weights, n)
        ratio = self._tmp(n)
        check(self._lib.psd_scan_adaptive(val.ptr, n, int(window_width), float(min_content_val), ratio.ptr,
                                          self._stream), "psd_scan_adaptive")
        check(self._lib.psd_cuts_adaptive(ratio.ptr, val.ptr, n, first_frame, int(window_width),
                                          float(adaptive_threshold), float(min_content_val),
                                          min_len_frames(min_scene_len, fps), self._cuts.ptr, self._count.ptr,
                                          self._cap, self._stream), "psd_cuts_adaptive")
        return self._fetch()

    def histogram(self, threshold=0.20, bins=128, min_scene_len=15, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        _, hist = self._e.device_results()
        corr = self._tmp(n)
        check(self._lib.psd_scan_hist_correl(hist, n, int(bins), None, corr.ptr, self._stream))
        check(self._lib.psd_cuts_histogram(corr.ptr, n, first_frame, histogram_threshold(threshold),
                                           min_len_frames(min_scene_len, fps), self._cuts.ptr, self._count.ptr,
                                           self._cap, self._stream), "psd_cuts_histogram")
        return self._fetch()

    def hash(self, threshold=0.35, min_scene_len=15, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        hashes = self._e.device_hash()
        dist = self._tmp(n)
        check(self._lib.psd_scan_hash_dist(hashes, n, int(self._e.hash_size), None, dist.ptr, self._stream))
        check(self._lib.psd_cuts_hash(dist.ptr, n, first_frame, float(threshold), min_len_frames(min_scene_len, fps),
                                      self._cuts.ptr, self._count.ptr, self._cap, self._stream), "psd_cuts_hash")
        return self._fetch()

    def threshold(self, threshold=12, min_scene_len=15, fade_bias=0.0, add_final_scene=False,
                  ceiling: bool = False, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        sums, _ = self._e.device_results()
        avg = self._tmp(n)
        check(self._lib.psd_scan_average(sums, n, self._e.n_pixels * 3, avg.ptr, self._stream))
        check(self._lib.psd_cuts_threshold(avg.ptr, n, first_frame, float(int(threshold)), 1 if ceiling else 0,
                                           float(fade_bias), min_len_frames(min_scene_len, fps),
                                           1 if add_final_scene else 0, self._cuts.ptr, self._count.ptr,
                                           self._cap, self._stream), "psd_cuts_threshold")
        return self._fetch()


def histogram_threshold(threshold) -> float:
    """The correlation bound psd_cuts_histogram compares with: 1 - threshold, clamped (histogram_detector.py:44)."""
    return max(0.0, min(1.0, 1.0 - threshold))


def automaton_args(detector) -> tuple[str, dict]:
    """The device automaton that corresponds to a (fresh) detector object of this package, as the name of the
    `DeviceCuts` method that runs it and that method's keyword arguments, taken from the detector's own
    parameters (`fps` and `first_frame` excepted).  `cuts_for_detector` and `sweep.ParameterSweep` both map
    detectors to automata through this one function."""
    from .compat import FlashFilter
    from .detectors import AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector, ThresholdDetector
    if isinstance(detector, HashDetector):
        return "hash", dict(threshold=detector._threshold, min_scene_len=detector._min_scene_len)
    if isinstance(detector, AdaptiveDetector):
        return "adaptive", dict(weights=tuple(detector._weights), adaptive_threshold=detector.adaptive_threshold,
                                min_scene_len=detector.min_scene_len, window_width=detector.window_width,
                                min_content_val=detector.min_content_val)
    if isinstance(detector, ContentDetector):
        ff = detector._flash_filter
        length = ff._filter_secs if ff._filter_secs is not None else ff._filter_length
        return "content", dict(weights=tuple(detector._weights), threshold=detector._threshold, min_scene_len=length,
                               suppress=ff._mode == FlashFilter.Mode.SUPPRESS)
    if isinstance(detector, HistogramDetector):
        # the constructor stored 1 - threshold (clamped); DeviceCuts.histogram applies the same map
        return "histogram", dict(threshold=1.0 - detector._threshold, bins=detector._bins,
                                 min_scene_len=detector._min_scene_len)
    if isinstance(detector, ThresholdDetector):
        return "threshold", dict(threshold=detector.threshold, min_scene_len=detector.min_scene_len,
                                 fade_bias=detector.fade_bias, add_final_scene=detector.add_final_scene,
                                 ceiling=detector.method == ThresholdDetector.Method.CEILING)
    raise TypeError(f"no device automaton for {type(detector).__name__}")


def cuts_for_detector(dc: DeviceCuts, detector, fps, first_frame: int = 0) -> list[int]:
    """Run the device automaton that corresponds to a (fresh) detector object of this package with the
    detector's own parameters: the cut list its per-frame `process_frame` + `post_process` would produce."""
    method, kwargs = automaton_args(detector)
    return getattr(dc, method)(**kwargs, fps=fps, first_frame=first_frame)
