"""Python twin of the two clip kernels (clip_kernels.cu) and of the device memory they work on, so that
`pyscenedetect_b200.clips` runs on a box with no GPU: psd_clip_fill, psd_clip_cuts with the five automata of
cut_automata.cuh restated statement by statement, and the psd_scan_* launches `device_cuts.scan_metric` makes,
answered from the oracle-backed engine of tests/fake_engine.py.  Device pointers are keys of `MEMORY`."""

from __future__ import annotations

import itertools

import numpy as np

from pyscenedetect_b200 import _capi
from tests.fake_engine import OracleEngine

MEMORY: dict = {}
_ids = itertools.count(1 << 20, 1 << 12)
NAN = np.frombuffer(bytes.fromhex("000000000000f8ff"), dtype=np.float64)[0]  # CUDART_NAN: sign bit set


class Buffer:
    """`engine.DeviceBuffer` over host bytes."""

    def __init__(self, nbytes: int, device: int = 0):
        self.nbytes = int(nbytes)
        self.data = np.zeros(self.nbytes, dtype=np.uint8)
        self.ptr = next(_ids)
        MEMORY[self.ptr] = self

    def upload(self, arr, offset: int = 0):
        b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        self.data[offset:offset + b.size] = b

    def download(self, nbytes: int, offset: int = 0) -> np.ndarray:
        return self.data[offset:offset + nbytes].copy()

    def close(self):
        MEMORY.pop(self.ptr, None)


def _array(ptr: int, dtype, n: int | None = None) -> np.ndarray:
    """The `dtype` array at device pointer `ptr` (which may point inside a buffer)."""
    base = max(p for p in MEMORY if p <= ptr)
    a = MEMORY[base].data[ptr - base:].view(dtype)
    return a if n is None else a[:n]


class PinnedHost:
    """`engine.PinnedBuffer` as plain host memory."""

    def __init__(self, nbytes: int):
        self.array = np.zeros(int(nbytes), dtype=np.uint8)

    def close(self):
        pass


class ClipEngine(OracleEngine):
    """OracleEngine with the device-side accessors `scan_metric` reads: every "device pointer" is the engine."""

    submissions = []

    compute_stream = None

    def submit(self, frames, pinned=False, channel_order="bgr"):
        ClipEngine.submissions.append(len(frames) if frames.ndim == 4 else 1)
        super().submit(frames, pinned)

    def device_results(self):
        return self, self

    def device_hash(self):
        return self

    def device_edge_sads(self):
        return None

    def view(self, edge_slot=0, hash_slot=0):
        assert edge_slot == 0 and hash_slot == 0, "the twin engine has one slot of each kind"
        return self


# -- the automata of cut_automata.cuh --
def flash_filter_cuts(above, n, first, min_frames, mode, out):
    if min_frames <= 0:
        out.extend(first + i for i in range(n) if above(i))
        return
    last_above, merge_enabled, merge_triggered, merge_start = first, False, False, 0
    for i in range(n):
        t = first + i
        a = above(i)
        met = (t - last_above) >= min_frames
        if mode == 1:
            if a and met:
                last_above = t
                out.append(t)
            continue
        if a:
            last_above = t
        if merge_triggered:
            if met and not a and (last_above - merge_start) >= min_frames:
                merge_triggered = False
                out.append(last_above)
            continue
        if not a:
            continue
        if met:
            merge_enabled = True
            out.append(t)
        elif merge_enabled:
            merge_triggered, merge_start = True, t


def adaptive_cuts(ratio, score, n, first, w, thr, mcv, min_frames, out):
    last_cut = first
    for i in range(w, n - w):
        met = ratio[i] >= thr and score[i] >= mcv
        if met and (first + i + w - last_cut) >= min_frames:
            last_cut = first + i
            out.append(first + i)


def histogram_cuts(correl, n, first, thr, min_frames, out):
    last_cut = first
    for i in range(1, n):
        t = first + i
        if correl[i] <= thr and (t - last_cut) >= min_frames:
            out.append(t)
            last_cut = t


def hash_cuts(dist, n, first, thr, min_frames, out):
    last_cut = first
    for i in range(n):
        d = dist[i]
        if d != d:
            continue
        t = first + i
        if d >= thr and (t - last_cut) >= min_frames:
            out.append(t)
            last_cut = t


def threshold_cuts(avg, n, first, thr, ceiling, fade_bias, min_frames, add_final, out):
    if n <= 0:
        return
    last_scene_cut = fade_frame = first
    fade_in = not (avg[0] < thr)
    for i in range(1, n):
        t = first + i
        v = avg[i]
        below = (v >= thr) if ceiling else (v < thr)
        if fade_in and below:
            fade_in, fade_frame = False, t
        elif not fade_in and not below:
            if (t - last_scene_cut) >= min_frames:
                out.append(fade_frame + round(((t - fade_frame) * (1.0 + fade_bias)) / 2.0))
                last_scene_cut = t
            fade_in, fade_frame = True, t
    if not fade_in and add_final and (first + n - 1 - last_scene_cut) >= min_frames:
        out.append(fade_frame)


def run_cell(c, base, n, first, min_frames, out):
    m = _array(c.metric, np.float64)[base:base + n]
    if c.kind == _capi.SWEEP_CONTENT:
        flash_filter_cuts(lambda i: m[i] >= c.threshold, n, first, min_frames, c.mode, out)
    elif c.kind == _capi.SWEEP_ADAPTIVE:
        adaptive_cuts(m, _array(c.metric2, np.float64)[base:base + n], n, first, c.window, c.threshold,
                      c.min_content_val, min_frames, out)
    elif c.kind == _capi.SWEEP_THRESHOLD:
        threshold_cuts(m, n, first, c.threshold, c.mode, c.fade_bias, min_frames, c.add_final_scene, out)
    elif c.kind == _capi.SWEEP_HISTOGRAM:
        histogram_cuts(m, n, first, c.threshold, min_frames, out)
    else:
        hash_cuts(m, n, first, c.threshold, min_frames, out)


class Lib:
    """The library with the clip kernels and the scans answered here; `launches` counts them as the library does."""

    def __init__(self):
        self._real = _capi.load()
        self.launches = {}

    def __getattr__(self, name):
        return getattr(self._real, name)

    def _count(self, name, k=1):
        self.launches[name] = self.launches.get(name, 0) + k

    # scans: the oracle engine's own, into device memory
    def psd_scan_content_edges(self, sums, sads, n, n_pixels, w, wsum, comps, out, st):
        self._count("scan")
        _array(out, np.float64, n)[:] = sums.scan_content(list(w))[0]
        return 0

    def psd_scan_adaptive(self, scores, n, w, mcv, out, st):
        self._count("scan")
        _array(out, np.float64, n)[:] = OracleEngine.scan_adaptive(None, _array(scores, np.float64, n), w, mcv)
        return 0

    def psd_scan_average(self, sums, n, n_values, out, st):
        self._count("scan")
        _array(out, np.float64, n)[:] = sums.scan_average()
        return 0

    def psd_scan_hist_correl(self, yhist, n, bins, prev, out, st):
        self._count("scan")
        _array(out, np.float64, n)[:] = yhist.scan_hist_correl(bins)
        return 0

    def psd_scan_hash_dist(self, hashes, n, size, prev, out, st):
        self._count("scan")
        _array(out, np.float64, n)[:] = hashes.scan_hash_dist()
        return 0

    # clip_kernels.cu
    def psd_clip_fill(self, values, n, offsets, n_clips, head, tail, fill_nan, fill, st):
        if n == 0 or n_clips * (head + tail) == 0:
            return 0
        self._count("psd_clip_fill")
        v = _array(values, np.float64, n)
        off = _array(offsets, np.int64, n_clips + 1)
        for j in range(n_clips):
            b = min(max(int(off[j]), 0), n)
            e = min(max(int(off[j + 1]), b), n)
            v[b:min(b + head, e)] = NAN if fill_nan else fill
            v[max(e - tail, b):e] = NAN if fill_nan else fill
        return 0

    def psd_clip_cuts(self, cells, n_cells, offsets, first, n_clips, min_frames, cuts, cap, cut_offsets, st):
        self._count("psd_clip_cuts", 3)
        off = _array(offsets, np.int64, n_clips + 1)
        ff = _array(first, np.int64, n_clips)
        mf = _array(min_frames, np.int64, n_cells * n_clips)
        lists = []
        for k in range(n_cells):
            for j in range(n_clips):
                b = max(int(off[j]), 0)
                e = max(int(off[j + 1]), b)
                out = []
                run_cell(cells[k], b, e - b, int(ff[j]), int(mf[k * n_clips + j]), out)
                lists.append(out)
        o = _array(cut_offsets, np.int64, n_cells * n_clips + 1)
        o[:] = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        if o[-1] <= cap and o[-1]:
            _array(cuts, np.int64, int(o[-1]))[:] = [c for x in lists for c in x]
        return 0
