"""Stage-by-stage twin of HashDetector's device hash (csrc/hash_kernels.cu: psd_hash_rows_kernel,
psd_hash_finish_kernel), vectorised over columns with the kernels' per-element order of operations, so that every
intermediate the kernels keep can be compared bit for bit:

  rowbuf  [H][n] float32   the rows kernel's output: raw uint32 column sums (as float32 bits) where both area
                           factors are integers, else the float32 chain first tap / whole-pixel run / last tap
  area    [n][n] uint8     cv2.resize(gray, (n, n), INTER_AREA)
  x       [n][n] float64   float32(area) / float32(max(area) or 1)
  low     [size][size] float32  the orthonormal DCT's low band, folded like oracle/intmath.py:dct_fold_1d
  median  float32          numpy.median of the low band
  bits    [size*size] bool low > median
  words   [PSD_HASH_WORDS_FOR(size)] uint64, bits past size * size are 0

The cosine table is the engine's: cos(pi * k / (2.0 * n)) through libm (math.cos), the host's expression."""

from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import numpy as np

from oracle import intmath as M
from pyscenedetect_b200._capi import hash_words

FOLD_CAP = 8   # hash_plan_create: at most 8 folded levels (level 0 included)


@dataclass
class Stages:
    rowbuf: np.ndarray
    area: np.ndarray
    x: np.ndarray
    low: np.ndarray
    median: np.float32
    bits: np.ndarray
    words: np.ndarray


def costab(n: int) -> np.ndarray:
    return np.array([math.cos(math.pi * k / (2.0 * n)) for k in range(4 * n)])


_costab = functools.lru_cache(maxsize=None)(costab)


@functools.lru_cache(maxsize=None)
def _by_column(ssize: int, n: int):
    """INTER_AREA taps of a length-ssize axis shrunk to n, grouped by their place in a destination cell:
    [(dst indices, src indices, float32 weights)] for tap 0, tap 1, ... of every cell that has that many."""
    tab = M.area_tab(ssize, n)
    per = [[] for _ in range(n)]
    for d, s, a in tab:
        per[d].append((s, a))
    out = []
    for j in range(max(len(p) for p in per)):
        ds = np.array([d for d in range(n) if len(per[d]) > j])
        out.append((ds, np.array([per[d][j][0] for d in ds]), np.array([per[d][j][1] for d in ds], np.float32)))
    return out


def rows_stage(gray: np.ndarray, n: int) -> np.ndarray:
    """psd_hash_rows_kernel: [H][n] float32 (uint32 sums as their bits on the integer path)."""
    H, W = gray.shape
    if W % n == 0 and H % n == 0:
        s = gray.astype(np.uint64).reshape(H, n, W // n).sum(axis=2) & 0xFFFFFFFF
        return s.astype(np.uint32).view(np.float32)
    S = gray.astype(np.float32)
    buf = np.zeros((H, n), np.float32)
    for ds, si, a in _by_column(W, n):   # tap j of every column, in source order: separate multiply and add
        buf[:, ds] = buf[:, ds] + (S[:, si] * a[None, :])
    return buf


def area_stage(rowbuf: np.ndarray, W: int, H: int, n: int) -> np.ndarray:
    """psd_hash_finish_kernel's vertical pass: the INTER_AREA image [n][n] uint8."""
    if W % n == 0 and H % n == 0:
        aw, ah = W // n, H // n
        s = (rowbuf.view(np.uint32).astype(np.uint64).reshape(n, ah, n).sum(axis=1) & 0xFFFFFFFF).astype(np.uint32)
        if aw == 2 and ah == 2:
            return ((s + np.uint32(2)) >> np.uint32(2)).astype(np.uint8)
        if aw == 1 and ah == 1:
            return s.astype(np.uint8)
        inv = np.float32(1.0) / np.float32(aw * ah)
        return np.clip(np.rint(s.astype(np.float32) * inv), 0, 255).astype(np.uint8)
    acc = np.zeros((n, n), np.float32)
    for j, (ds, si, b) in enumerate(_by_column(H, n)):   # tap j of every destination row, in source order
        term = (b[:, None] * rowbuf[si, :]).astype(np.float32)
        acc[ds] = term if j == 0 else acc[ds] + term
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def fold_levels(a: np.ndarray) -> list:
    """oracle/intmath.py:dct_fold_1d's levels, for every column of `a` at once (axis 0 folds)."""
    levels = [a]
    while levels[-1].shape[0] % 2 == 0 and levels[-1].shape[0] > 1 and len(levels) < FOLD_CAP:
        p = levels[-1]
        h = p.shape[0] // 2
        levels.append(p[:h] + p[::-1][:h])
    return levels


def dct_fold_cols(a: np.ndarray, size: int, cos: np.ndarray, n: int) -> np.ndarray:
    """dct_fold_1d applied to every column of `a` ((len, cols) float64) -> (size, cols): numpy element-wise
    float64 operations in the same order, column by column, as the pure-Python twin."""
    levels = fold_levels(a)
    out = np.zeros((size, a.shape[1]))
    for u in range(size):
        k = len(levels) - 1 if u == 0 else 0
        if u:
            while k + 1 < len(levels) and u % (2 << k) == 0:
                k += 1
        lv = levels[k]
        nk = lv.shape[0]
        acc = np.zeros(a.shape[1])
        if nk % 2 == 0 and (u >> k) & 1:
            for i in range(nk // 2):
                acc = acc + (lv[i] - lv[nk - 1 - i]) * cos[((2 * i + 1) * u) % (4 * n)]
        else:
            for i in range(nk):
                acc = acc + lv[i] * cos[((2 * i + 1) * u) % (4 * n)]
        out[u] = acc
    return out


def low_band(x: np.ndarray, size: int, cos: np.ndarray) -> np.ndarray:
    n = x.shape[0]
    t = dct_fold_cols(x, size, cos, n)             # t[u][j]
    d = dct_fold_cols(t.T.copy(), size, cos, n)     # d[v][u]
    s0, s1 = math.sqrt(1.0 / n), math.sqrt(2.0 / n)
    su = np.where(np.arange(size) > 0, s1, s0)
    return ((d.T * su[:, None]) * su[None, :]).astype(np.float32)


def median(low: np.ndarray) -> np.float32:
    """numpy.median of float32: the middle value, or the float32 mean of the two middle values."""
    flat = np.sort(low.ravel())
    m = flat.size
    return flat[m // 2] if m % 2 else np.float32(np.float32(flat[m // 2 - 1] + flat[m // 2]) * np.float32(0.5))


def pack_words(bits: np.ndarray, size: int) -> np.ndarray:
    """bit c at word c // 64, bit c % 64; PSD_HASH_WORDS_FOR(size) words, zero past size * size."""
    padded = np.zeros(hash_words(size) * 64, np.uint8)
    padded[:bits.size] = bits
    return np.packbits(padded, bitorder="little").view("<u8").astype(np.uint64)


def stages(bgr: np.ndarray, size: int, lowpass: int, gray: np.ndarray | None = None) -> Stages:
    """Every stage of one frame (`gray`: its cv2 BGR2GRAY image, if already at hand)."""
    n = size * lowpass
    H, W = bgr.shape[:2]
    rowbuf = rows_stage(M.bgr_to_gray(bgr) if gray is None else gray, n)
    area = area_stage(rowbuf, W, H, n)
    x = (area.astype(np.float32) / np.float32(int(area.max()) or 1)).astype(np.float64)
    low = low_band(x, size, _costab(n))
    med = median(low)
    bits = (low > med).ravel()
    return Stages(rowbuf, area, x, low, med, bits, pack_words(bits, size))
