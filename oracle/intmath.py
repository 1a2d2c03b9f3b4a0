"""Pure numpy/integer restatement of the cv2 primitives on the hot path.
TEST INFRASTRUCTURE - see oracle/__init__.py.

The arithmetic of this path is in OpenCV (opencv-python-headless 4.13.0.92 in this image;
not vendored in the reference, unpinned in its pyproject.toml:43-57).  Each function below
restates the published OpenCV algorithm the reference reaches through the call site cited,
and is pinned against cv2 itself by tests/test_oracle_intmath.py.  The CUDA kernels implement
exactly these formulas.
"""

from __future__ import annotations

import math

import numpy as np

# ---------------------------------------------------------------------------------------------
# BGR -> HSV (8-bit), call site content_detector.py:155  cv2.cvtColor(..., COLOR_BGR2HSV)
# OpenCV imgproc/src/color_hsv: hsv_shift = 12, sdiv_table[i] = saturate_cast<int>((255 << 12)/(1.*i)),
# hdiv_table180[i] = saturate_cast<int>((180 << 12)/(6.*i)); saturate_cast<int>(double) = cvRound
# (round half to even).
# ---------------------------------------------------------------------------------------------
HSV_SHIFT = 12


def _rint_table(num: float) -> np.ndarray:
    t = np.zeros(256, dtype=np.int64)
    for i in range(1, 256):
        t[i] = int(np.rint(num / float(i)))
    return t


SDIV_TABLE = _rint_table(float(255 << HSV_SHIFT))
HDIV_TABLE = _rint_table(float(180 << HSV_SHIFT) / 6.0)


def bgr_to_hsv(bgr: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    b = bgr[..., 0].astype(np.int64)
    g = bgr[..., 1].astype(np.int64)
    r = bgr[..., 2].astype(np.int64)
    v = np.maximum(np.maximum(b, g), r)
    vmin = np.minimum(np.minimum(b, g), r)
    diff = v - vmin
    vr = v == r
    vg = v == g
    h = np.where(vr, g - b, np.where(vg, b - r + 2 * diff, r - g + 4 * diff))
    s = (diff * SDIV_TABLE[v] + (1 << (HSV_SHIFT - 1))) >> HSV_SHIFT
    h = (h * HDIV_TABLE[diff] + (1 << (HSV_SHIFT - 1))) >> HSV_SHIFT  # arithmetic shift
    h = h + np.where(h < 0, 180, 0)
    return h.astype(np.uint8), s.astype(np.uint8), v.astype(np.uint8)


# ---------------------------------------------------------------------------------------------
# BGR -> Y of YUV, call site histogram_detector.py:156  cv2.cvtColor(..., COLOR_BGR2YUV)
# OpenCV color_yuv: yuv_shift = 14, coefficients R2Y=4899, G2Y=9617, B2Y=1868.
# ---------------------------------------------------------------------------------------------


def bgr_to_y(bgr: np.ndarray) -> np.ndarray:
    b = bgr[..., 0].astype(np.int64)
    g = bgr[..., 1].astype(np.int64)
    r = bgr[..., 2].astype(np.int64)
    return ((r * 4899 + g * 9617 + b * 1868 + (1 << 13)) >> 14).astype(np.uint8)


# ---------------------------------------------------------------------------------------------
# numpy.mean(frame) (threshold_detector.py:127) and _mean_pixel_distance (content_detector.py:29-36):
# exact integer sum followed by ONE fp64 divide.
# ---------------------------------------------------------------------------------------------


def sad(a: np.ndarray, b: np.ndarray) -> int:
    return int(np.abs(a.astype(np.int64) - b.astype(np.int64)).sum())


def mean_from_sum(total: int, count: int) -> np.float64:
    return np.float64(total) / np.float64(float(count))


# ---------------------------------------------------------------------------------------------
# cv2.resize(..., INTER_LINEAR) on 8UC3, call site scene_manager.py:670-678.
# OpenCV resize.cpp: fixed-point bilinear, INTER_RESIZE_COEF_BITS = 11; horizontal pass keeps
# int32 (x2048), vertical pass ((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2.
# ---------------------------------------------------------------------------------------------
INTER_RESIZE_COEF_SCALE = 2048


def linear_taps(src, dst: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Per destination index: source index s (second tap is s+1 clamped) and the two 11-bit
    coefficients (a0, a1).  float32 coefficient generation as in resize.cpp, where the scale is
    1 / inv_scale_x with inv_scale_x = dst / src (not src / dst, which can differ in the last bit).
    `src` may be an array of source sizes: the tables then have shape (*src.shape, dst)."""
    src = np.asarray(src, dtype=np.int64)[..., None]
    scale = 1.0 / (dst / src.astype(np.float64))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    idx = s.astype(np.int64)
    low, high = idx < 0, idx >= src - 1
    idx = np.minimum(np.maximum(idx, 0), src - 1).astype(np.int32)
    f[low | high] = 0
    c0 = (np.float32(1.0) - f) * np.float32(INTER_RESIZE_COEF_SCALE)
    c1 = f * np.float32(INTER_RESIZE_COEF_SCALE)
    return idx, np.rint(c0).astype(np.int32), np.rint(c1).astype(np.int32)


def resize_linear(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    sh, sw = img.shape[:2]
    xi, xa0, xa1 = linear_taps(sw, dw)
    yi, ya0, ya1 = linear_taps(sh, dh)
    x1 = np.minimum(xi + 1, sw - 1)
    y1 = np.minimum(yi + 1, sh - 1)
    src = img.astype(np.int64)
    # horizontal pass on the rows that are needed
    def hrow(rows):
        return src[rows][:, xi, :] * xa0[None, :, None] + src[rows][:, x1, :] * xa1[None, :, None]
    r0 = hrow(yi)
    r1 = hrow(y1)
    b0 = ya0[:, None, None].astype(np.int64)
    b1 = ya1[:, None, None].astype(np.int64)
    out = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------
# calcHist / normalize / compareHist, call sites histogram_detector.py:159,163,98.
# ---------------------------------------------------------------------------------------------


def hist_counts(y: np.ndarray, bins: int) -> np.ndarray:
    """cv2.calcHist uniform bins over [0,256): bin = floor(v * bins / 256)."""
    idx = (y.astype(np.int64).ravel() * bins) // 256
    return np.bincount(idx, minlength=bins).astype(np.int64)


def hist_normalize_l2(counts: np.ndarray) -> np.ndarray:
    """cv2.normalize(hist, hist) with defaults NORM_L2, alpha=1: fp64 norm, then the float32
    histogram is scaled by a float32... (convertTo with double scale: dst = saturate<float>(src*scale))."""
    h = counts.astype(np.float32)
    norm = math.sqrt(float((h.astype(np.float64) ** 2).sum()))
    scale = (1.0 / norm) if norm > np.finfo(np.float64).eps else 0.0
    return (h * np.float32(scale)).astype(np.float32)


def hist_correl(h1: np.ndarray, h2: np.ndarray) -> float:
    """cv2.compareHist(HISTCMP_CORREL) in fp64."""
    a = h1.astype(np.float64)
    b = h2.astype(np.float64)
    n = a.size
    s1, s2 = a.sum(), b.sum()
    s11, s22, s12 = (a * a).sum(), (b * b).sum(), (a * b).sum()
    scale = 1.0 / n
    num = s12 - s1 * s2 * scale
    den2 = (s11 - s1 * s1 * scale) * (s22 - s2 * s2 * scale)
    return num / math.sqrt(den2) if abs(den2) > np.finfo(np.float64).eps else 1.0


# ---------------------------------------------------------------------------------------------
# Edge path, call site content_detector.py:213-239: numpy.median -> cv2.Canny -> cv2.dilate.
# ---------------------------------------------------------------------------------------------


def median_u8(plane: np.ndarray) -> float:
    """numpy.median of a uint8 plane from its 256-bin histogram (mean of the two middle
    order statistics when the count is even)."""
    counts = np.bincount(plane.ravel(), minlength=256)
    n = int(plane.size)
    cum = np.cumsum(counts)
    lo = int(np.searchsorted(cum, (n - 1) // 2 + 1))
    hi = int(np.searchsorted(cum, n // 2 + 1))
    return (lo + hi) / 2.0


def canny_thresholds(median: float) -> tuple[int, int]:
    sigma = 1.0 / 3.0
    low = int(max(0, (1.0 - sigma) * median))
    high = int(min(255, (1.0 + sigma) * median))
    return low, high


TG22 = 13573  # round(tan(22.5 deg) * 2^15)


def canny(lum: np.ndarray, low: int, high: int) -> np.ndarray:
    """cv2.Canny(image, low, high) with apertureSize=3, L2gradient=False.
    Sobel 3x3 (BORDER_REPLICATE), L1 magnitude, non-maximum suppression in fixed point, double
    threshold (strictly greater), 8-connected hysteresis; output 0/255."""
    from scipy import ndimage

    if low > high:
        low, high = high, low
    h, w = lum.shape
    p = np.pad(lum.astype(np.int32), 1, mode="edge")
    gx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    gy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    mag = np.abs(gx) + np.abs(gy)
    m = np.pad(mag, 1, mode="constant")  # zero outside the image
    c = m[1:-1, 1:-1]
    ax = np.abs(gx).astype(np.int64)
    ay = np.abs(gy).astype(np.int64) << 15
    tg22x = ax * TG22
    tg67x = tg22x + (ax << 16)
    horiz = ay < tg22x
    vert = ay > tg67x
    s = np.where((gx ^ gy) < 0, -1, 1)
    left, right = m[1:-1, :-2], m[1:-1, 2:]
    up, down = m[:-2, 1:-1], m[2:, 1:-1]
    yy, xx = np.mgrid[0:h, 0:w]
    d1 = m[yy, xx + 1 - s]      # mag[y-1][x-s]  (padded coords: y-1+1, x-s+1)
    d2 = m[yy + 2, xx + 1 + s]  # mag[y+1][x+s]
    keep = np.where(horiz, (c > left) & (c >= right),
                    np.where(vert, (c > up) & (c >= down), (c > d1) & (c > d2)))
    cand = keep & (c > low)
    strong = cand & (c > high)
    lab, _n = ndimage.label(cand, structure=np.ones((3, 3), dtype=bool))
    good = np.unique(lab[strong])
    out = np.isin(lab, good[good > 0])
    return (out.astype(np.uint8)) * 255


def dilate_square(img: np.ndarray, k: int) -> np.ndarray:
    """cv2.dilate(img, ones((k,k))) - max over the k x k window centred on the pixel, pixels
    outside the image ignored."""
    r = k // 2
    h, w = img.shape
    p = np.pad(img, r, mode="constant")
    out = np.zeros_like(img)
    rows = np.zeros((h + 2 * r, w), dtype=img.dtype)
    for dx in range(k):
        rows = np.maximum(rows, p[:, dx:dx + w])
    for dy in range(k):
        out = np.maximum(out, rows[dy:dy + h, :])
    return out


# ---- HashDetector pieces (hash_detector.py:124-158), restated from OpenCV 4.13's algorithms ----
def bgr_to_gray(bgr: np.ndarray) -> np.ndarray:
    """cv2.COLOR_BGR2GRAY for 8-bit: 15-bit fixed point (B 3735, G 19235, R 9798), not the 14-bit YUV-Y."""
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    return ((b * 3735 + g * 19235 + r * 9798 + 16384) >> 15).astype(np.uint8)


def area_tab(ssize: int, dsize: int) -> list[tuple[int, int, np.float32]]:
    """computeResizeAreaTab (imgproc/resize.cpp): (dst index, src index, float32 weight) in source order."""
    import math
    scale = ssize / dsize
    tab = []
    for dx in range(dsize):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, ssize - fsx1)
        sx1, sx2 = math.ceil(fsx1), math.floor(fsx2)
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, np.float32((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, np.float32(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def resize_area(gray: np.ndarray, n: int) -> np.ndarray:
    """cv2.resize(gray, (n, n), INTER_AREA) for a shrinking 8-bit image.  Integer scale factors take OpenCV's
    integer-sum path (sum * float32(1/area), rounded; 2x2 is (sum + 2) >> 2); otherwise every destination cell
    is a float32 accumulation `buf += S * alpha` per source row and `sum += beta * buf` down the rows, in source
    order, separate multiply and add - the order matters for the last bit."""
    H, W = gray.shape
    if W % n == 0 and H % n == 0:
        sx, sy = W // n, H // n
        s = gray.astype(np.int64).reshape(n, sy, n, sx).sum(axis=(1, 3))
        if sx == 2 and sy == 2:
            return ((s + 2) >> 2).astype(np.uint8)
        if sx == 1 and sy == 1:
            return gray.copy()
        return np.clip(np.rint(s.astype(np.float32) * (np.float32(1.0) / np.float32(sx * sy))), 0, 255).astype(np.uint8)
    xt, yt = area_tab(W, n), area_tab(H, n)
    xi = np.array([t[0] for t in xt]); xs = np.array([t[1] for t in xt]); xa = np.array([t[2] for t in xt], np.float32)
    S = gray.astype(np.float32)
    out = np.zeros((n, n), np.uint8)
    sumv = np.zeros(n, np.float32)
    prev_dy = yt[0][0]
    for dy, sy, beta in yt:
        buf = np.zeros(n, np.float32)
        prod = (S[sy, xs] * xa).astype(np.float32)
        for k in range(len(xt)):                      # sequential float32 adds, source order
            buf[xi[k]] = np.float32(buf[xi[k]] + prod[k])
        if dy != prev_dy:
            out[prev_dy] = np.clip(np.rint(sumv), 0, 255).astype(np.uint8)
            sumv = (beta * buf).astype(np.float32)
            prev_dy = dy
        else:
            sumv = (sumv + (beta * buf).astype(np.float32)).astype(np.float32)
    out[prev_dy] = np.clip(np.rint(sumv), 0, 255).astype(np.uint8)
    return out


def dct_fold_1d(v, size: int, costab: np.ndarray, n: int) -> list[float]:
    """Unnormalised DCT-II coefficients u < size of `v`, computed as fast DCTs do (twin of
    csrc/hash_kernels.cu:fold_coef): fold the vector (a[i] + a[len-1-i]) while its length is even; an even
    frequency is the half frequency of the folded vector, an odd one a sum over differences a[i] - a[len-1-i],
    accumulated left to right.  Constant / mirror-symmetric inputs give exact zeros."""
    levels = [[float(t) for t in v]]
    while len(levels[-1]) % 2 == 0 and len(levels[-1]) > 1 and len(levels) < 8:
        a = levels[-1]
        h = len(a) // 2
        levels.append([a[i] + a[len(a) - 1 - i] for i in range(h)])
    out = []
    for u in range(size):
        k = 0
        if u == 0:
            k = len(levels) - 1
        else:
            while k + 1 < len(levels) and u % (2 << k) == 0:
                k += 1
        a = levels[k]
        nk = len(a)
        acc = 0.0
        if nk % 2 == 0 and (u >> k) & 1:
            for i in range(nk // 2):
                acc = acc + (a[i] - a[nk - 1 - i]) * float(costab[((2 * i + 1) * u) % (4 * n)])
        else:
            for i in range(nk):
                acc = acc + a[i] * float(costab[((2 * i + 1) * u) % (4 * n)])
        out.append(acc)
    return out


def phash_bits(bgr: np.ndarray, hash_size: int, factor: int) -> np.ndarray:
    """hash_frame with the integer stages exact and the DCT in float64 with the folding structure of a fast DCT
    (cv2.dct is float32 through IPP: a bit can differ only where a coefficient sits within rounding distance of the
    median - in practice where the exact coefficient is 0: solid-colour frames and 1-D gradients; with the folding,
    solid frames come out as cv2 gives them for power-of-two hash images)."""
    import math
    n = hash_size * factor
    r = resize_area(bgr_to_gray(bgr), n)
    mx = int(r.max()) or 1
    x = (r.astype(np.float32) / np.float32(mx)).astype(np.float64)
    costab = np.cos(np.pi * np.arange(4 * n) / (2.0 * n))
    t = [dct_fold_1d(x[:, j], hash_size, costab, n) for j in range(n)]          # t[j][u]: vertical transform of column j
    s0, s1 = math.sqrt(1.0 / n), math.sqrt(2.0 / n)
    low = np.zeros((hash_size, hash_size), np.float32)
    for u in range(hash_size):
        row = dct_fold_1d([t[j][u] for j in range(n)], hash_size, costab, n)
        for v in range(hash_size):
            low[u, v] = np.float32((row[v] * (s1 if u else s0)) * (s1 if v else s0))
    flat = np.sort(low.ravel())
    m = flat.size
    med = flat[m // 2] if m % 2 else np.float32(np.float32(flat[m // 2 - 1] + flat[m // 2]) * np.float32(0.5))
    return low > med
