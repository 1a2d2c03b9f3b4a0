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


def scan_metric(lib, holder, key: tuple, out: int, content_val: int | None = None,
                clips: tuple[int, int] | None = None, components: int | None = None) -> None:
    """Launch the psd_scan_* that fills one metric array `out` (float64 per frame) from every frame a result holder
    (an Engine, a `SlotView` of one or `sharding.GatheredResults`) holds, on the holder's stream.  `key` is a
    `ParameterSweep` metric key without its group index: ("content_val", weights), ("adaptive_ratio", weights,
    window_width, min_content_val), which reads `content_val` (that weight vector's array), ("average_rgb",),
    ("hist_correl", bins) or ("hash_dist",).

    `clips` = (device clip table, clip count) when the holder's frames are several clips scored back to back
    (psd_clip_fill): the scan is followed by the fix-up that gives every clip's first (and, for the adaptive ratio,
    last) entries the values a one-clip engine's scan has there, so each clip's slice equals that engine's array
    byte for byte.  An adaptive ratio must read a `content_val` array that was fixed up the same way.

    `components`: for content_val, a float64[n][4] device array that also receives psd_scan_content's components
    (content_detector.py:166-176); the clip fix-up leaves them as scanned."""
    _scan_metric(lib, holder, key, out, content_val, components)
    if clips is None or key[0] == "average_rgb":  # average_rgb is per frame: nothing crosses a clip edge
        return
    table, n_clips = clips
    # the value a one-clip scan writes there, in the scan's own bits: psd_scan_adaptive and psd_scan_hist_correl
    # write CUDART_NAN (fill_nan 1), psd_scan_hash_dist the NaN with the sign bit clear, which is Python's
    fill = 0.0
    if key[0] == "content_val":      # the first frame scores 0.0 (content_detector.py:161-164)
        head, tail, nan = 1, 0, 0
    elif key[0] == "adaptive_ratio":  # the window is incomplete (adaptive_detector.py:111-115)
        head, tail, nan = int(key[2]), int(key[2]), 1
    elif key[0] == "hist_correl":     # no predecessor (histogram_detector.py:98)
        head, tail, nan = 1, 0, 1
    else:                             # hash_dist: no predecessor (hash_detector.py:82)
        head, tail, nan, fill = 1, 0, 0, float("nan")
    check(lib.psd_clip_fill(out, holder.frame_count, table, n_clips, head, tail, nan, fill, holder.compute_stream),
          "psd_clip_fill")


def _scan_metric(lib, holder, key: tuple, out: int, content_val: int | None, components: int | None = None) -> None:
    n, st = holder.frame_count, holder.compute_stream
    kind = key[0]
    if kind == "content_val":
        sums, _ = holder.device_results()
        w = (C.c_double * 4)(*[float(x) for x in key[1]])
        wsum = float(sum(abs(x) for x in key[1]))  # same expression as content_detector.py:180
        # NULL edge SADs: the sums' own sad_edges (edge slot 0)
        check(lib.psd_scan_content_edges(sums, holder.device_edge_sads(), n, holder.n_pixels, w, wsum, components, out,
                                         st), "psd_scan_content_edges")
    elif kind == "adaptive_ratio":
        check(lib.psd_scan_adaptive(content_val, n, int(key[2]), float(key[3]), out, st), "psd_scan_adaptive")
    elif kind == "average_rgb":
        sums, _ = holder.device_results()
        check(lib.psd_scan_average(sums, n, holder.n_pixels * 3, out, st), "psd_scan_average")
    elif kind == "hist_correl":
        _, yhist = holder.device_results()
        check(lib.psd_scan_hist_correl(yhist, n, int(key[1]), None, out, st), "psd_scan_hist_correl")
    else:
        check(lib.psd_scan_hash_dist(holder.device_hash(), n, int(holder.hash_size), None, out, st),
              "psd_scan_hash_dist")


class DeviceCuts:
    def __init__(self, engine: Engine, max_cuts: int = 1 << 16):
        self._e = engine
        self._lib = _capi.load()
        self._dev = engine.device
        self._cap = int(max_cuts)
        self._cuts = DeviceBuffer(self._cap * 8, self._dev)
        self._count = DeviceBuffer(8, self._dev)
        self._stream = engine.compute_stream

    def _scan(self, key: tuple, content_val: DeviceBuffer | None = None) -> DeviceBuffer:
        out = DeviceBuffer(max(8, self._e.frame_count * 8), self._dev)
        scan_metric(self._lib, self._e, key, out.ptr, content_val.ptr if content_val is not None else None)
        return out

    def _fetch(self) -> list[int]:
        self._e.sync()
        count = int(self._count.download(4).view(np.int32)[0])
        if count > self._cap:
            raise RuntimeError(f"{count} cuts exceed the device cut buffer ({self._cap})")
        return self._cuts.download(count * 8).view(np.int64).tolist() if count else []

    def content(self, weights=(1.0, 1.0, 1.0, 0.0), threshold=27.0, min_scene_len=15, fps=30.0,
                suppress: bool = False, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        val = self._scan(("content_val", weights))
        flags = DeviceBuffer(max(1, n), self._dev)
        check(self._lib.psd_scan_compare(val.ptr, n, float(threshold), 0, flags.ptr, self._stream))
        check(self._lib.psd_cuts_flash_filter(flags.ptr, n, first_frame, flash_filter_frames(min_scene_len, fps),
                                              1 if suppress else 0, self._cuts.ptr, self._count.ptr, self._cap,
                                              self._stream), "psd_cuts_flash_filter")
        return self._fetch()

    def adaptive(self, weights=(1.0, 1.0, 1.0, 0.0), adaptive_threshold=3.0, min_scene_len=15,
                 window_width=2, min_content_val=15.0, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        val = self._scan(("content_val", weights))
        ratio = self._scan(("adaptive_ratio", weights, window_width, min_content_val), val)
        check(self._lib.psd_cuts_adaptive(ratio.ptr, val.ptr, n, first_frame, int(window_width),
                                          float(adaptive_threshold), float(min_content_val),
                                          min_len_frames(min_scene_len, fps), self._cuts.ptr, self._count.ptr,
                                          self._cap, self._stream), "psd_cuts_adaptive")
        return self._fetch()

    def histogram(self, threshold=0.20, bins=128, min_scene_len=15, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        corr = self._scan(("hist_correl", bins))
        check(self._lib.psd_cuts_histogram(corr.ptr, n, first_frame, histogram_threshold(threshold),
                                           min_len_frames(min_scene_len, fps), self._cuts.ptr, self._count.ptr,
                                           self._cap, self._stream), "psd_cuts_histogram")
        return self._fetch()

    def hash(self, threshold=0.35, min_scene_len=15, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        dist = self._scan(("hash_dist",))
        check(self._lib.psd_cuts_hash(dist.ptr, n, first_frame, float(threshold), min_len_frames(min_scene_len, fps),
                                      self._cuts.ptr, self._count.ptr, self._cap, self._stream), "psd_cuts_hash")
        return self._fetch()

    def threshold(self, threshold=12, min_scene_len=15, fade_bias=0.0, add_final_scene=False,
                  ceiling: bool = False, fps=30.0, first_frame: int = 0) -> list[int]:
        n = self._e.frame_count
        avg = self._scan(("average_rgb",))
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
    detector's own parameters: the cut list its per-frame `process_frame` + `post_process` would produce.  The
    metrics come from the result holder `attach_engine` gave the detector (its slots of a shared engine), else from
    `dc`'s."""
    method, kwargs = automaton_args(detector)
    holder = detector._engine
    if holder is not None and not detector._owns_engine and holder is not dc._e:
        dc = DeviceCuts(holder, dc._cap)
    return getattr(dc, method)(**kwargs, fps=fps, first_frame=first_frame)
