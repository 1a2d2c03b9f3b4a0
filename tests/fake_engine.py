"""Oracle-backed stand-in for `pyscenedetect_b200.engine.Engine` so that the HOST logic
(detector state machines, batching, stats, SceneManager, sharding) can be tested on a box with
no GPU.  Test infrastructure only - it computes with oracle.intmath, never the product."""

from __future__ import annotations

import cv2
import numpy as np

from oracle import intmath as M
from oracle import ref_detectors as R
from pyscenedetect_b200._capi import F_BGRSUM, F_EDGES, F_HASH, F_HSV, F_YHIST, SUMS_DTYPE


class OracleEngine:
    def __init__(self, src_width, src_height, features, width=None, height=None, device=0,
                 max_batch=64, edge_kernel_size=0, hash_size=8, hash_lowpass=2):
        self.src_width, self.src_height = src_width, src_height
        self.width = width if width is not None else src_width
        self.height = height if height is not None else src_height
        self.features = features | (F_HSV if features & F_EDGES else 0)
        self.n_pixels = self.width * self.height
        self.max_batch = max_batch
        k = edge_kernel_size or R.estimated_kernel_size(self.width, self.height)
        self._kernel = np.ones((k, k), np.uint8)
        self.hash_size, self.hash_lowpass = hash_size, hash_lowpass
        self.reset()

    def reset(self):
        self._sums = []
        self._hist = []
        self._prev = None
        self._halo_hist = None
        self._hashes = []
        self._halo_hash = None

    @property
    def frame_count(self):
        return len(self._sums)

    def _score(self, frame, record=True):
        if (self.width, self.height) != (self.src_width, self.src_height):
            frame = cv2.resize(frame, (self.width, self.height), interpolation=cv2.INTER_LINEAR)
        row = np.zeros((), dtype=SUMS_DTYPE)
        h, s, v = M.bgr_to_hsv(frame)
        edges = R.detect_edges(v, self._kernel) if self.features & F_EDGES else None
        if self._prev is not None:
            row["has_prev"] = 1
            if self.features & F_HSV:
                row["sad_hue"] = M.sad(h, self._prev[0])
                row["sad_sat"] = M.sad(s, self._prev[1])
                row["sad_lum"] = M.sad(v, self._prev[2])
            if edges is not None:
                row["sad_edges"] = M.sad(edges, self._prev[3])
        if self.features & F_BGRSUM:
            row["bgr_sum"] = int(frame.astype(np.int64).sum())
        hist = np.bincount(M.bgr_to_y(frame).ravel(), minlength=256).astype(np.uint32)
        hbits = M.phash_bits(frame, self.hash_size, self.hash_lowpass) if self.features & F_HASH else None
        self._prev = (h, s, v, edges)
        if record:
            self._sums.append(row)
            self._hist.append(hist)
            self._hashes.append(hbits)
        else:
            self._halo_hist = hist
            self._halo_hash = hbits

    def set_halo(self, frame):
        assert self.frame_count == 0
        self._prev = None
        self._score(np.asarray(frame).reshape(self.src_height, self.src_width, 3), record=False)

    def submit(self, frames, pinned=False):
        frames = frames[None] if frames.ndim == 3 else frames
        for f in frames:
            self._score(np.ascontiguousarray(f))

    def sync(self):
        pass

    def close(self):
        pass

    def read_sums(self, first=0, n=None):
        n = self.frame_count - first if n is None else n
        return np.array(self._sums[first:first + n], dtype=SUMS_DTYPE)

    def read_yhist(self, first=0, n=None):
        n = self.frame_count - first if n is None else n
        return np.array(self._hist[first:first + n], dtype=np.uint32).reshape(n, 256)

    def read_hash(self, first=0, n=None):
        """(n, 4) uint64 in the engine's bit order (bit u*size+v)"""
        n = self.frame_count - first if n is None else n
        out = np.zeros((n, 4), dtype=np.uint64)
        for i in range(n):
            flat = self._hashes[first + i].ravel()
            for k in np.flatnonzero(flat):
                out[i, k >> 6] |= np.uint64(1) << np.uint64(k & 63)
        return out

    # scans: the reference's float64 operation order
    def scan_content(self, weights, first=0, n=None):
        s = self.read_sums(first, n)
        npx = float(self.n_pixels)
        val = np.zeros(len(s))
        comps = np.zeros((len(s), 4))
        for i, r in enumerate(s):
            if not r["has_prev"]:
                continue
            c = [np.float64(int(r[k])) / npx for k in ("sad_hue", "sad_sat", "sad_lum", "sad_edges")]
            comps[i] = c
            val[i] = sum(a * b for a, b in zip(c, weights)) / sum(abs(w) for w in weights)
        return val, comps

    def scan_adaptive(self, scores, window_width, min_content_val):
        scores = [np.float64(x) for x in scores]
        out = np.full(len(scores), np.nan)
        w = window_width
        for i in range(w, len(scores) - w):
            avg = sum(scores[j] for j in range(i - w, i + w + 1) if j != i) / (2.0 * w)
            if not abs(avg) < 0.00001:
                out[i] = min(scores[i] / avg, 255.0)
            else:
                out[i] = 255.0 if scores[i] >= min_content_val else 0.0
        return out

    def scan_average(self, first=0, n=None):
        s = self.read_sums(first, n)
        return np.array([np.float64(int(r["bgr_sum"])) / float(self.n_pixels * 3) for r in s])

    def scan_hash_dist(self, first=0, n=None):
        n = self.frame_count - first if n is None else n
        out = np.full(n, np.nan)
        for i in range(n):
            t = first + i
            prev = self._hashes[t - 1] if t > 0 else self._halo_hash
            if prev is not None:
                out[i] = np.count_nonzero(self._hashes[t] != prev) / float(self.hash_size * self.hash_size)
        return out

    def scan_hist_correl(self, bins, first=0, n=None):
        n = self.frame_count - first if n is None else n
        out = np.full(n, np.nan)
        for i in range(n):
            t = first + i
            prev = self._hist[t - 1] if t > 0 else self._halo_hist
            if prev is None:
                continue
            def rebin(h):
                idx = (np.arange(256) * bins) // 256
                return np.bincount(idx, weights=h, minlength=bins).astype(np.int64)
            a = M.hist_normalize_l2(rebin(prev))
            b = M.hist_normalize_l2(rebin(self._hist[t]))
            out[i] = M.hist_correl(a, b)
        return out


class OracleResults(OracleEngine):
    """`GatheredResults` stand-in: the scans of OracleEngine over gathered integer arrays."""

    def __init__(self, sums, yhist, n_pixels, device=0, hashes=None, hash_size=8, hash_lowpass=2):
        self.n_pixels = int(n_pixels)
        self._sums = list(sums)
        self._hist = list(yhist) if yhist is not None else []
        self._halo_hist = None
        self.hash_size, self.hash_lowpass = hash_size, hash_lowpass
        self._halo_hash = None
        self._hashes = []
        if hashes is not None:
            m = hash_size * hash_size
            for row in np.asarray(hashes, dtype=np.uint64):
                bits = np.array([(int(row[k >> 6]) >> (k & 63)) & 1 for k in range(m)], dtype=bool)
                self._hashes.append(bits.reshape(hash_size, hash_size))

    def read_sums(self, first=0, n=None):
        n = self.frame_count - first if n is None else n
        return np.array(self._sums[first:first + n], dtype=SUMS_DTYPE)
