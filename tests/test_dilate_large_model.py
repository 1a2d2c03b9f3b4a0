"""CPU restatement of the separable bit-plane dilation for kernel sizes >= 65 (csrc/edge_kernels.cu,
psd_edge_hdil_rows_kernel and psd_edge_vdil_cols_kernel), word for word where the bit manipulation is the risk:

  * horizontal: each row behind ceil(r / 32) zero words, window doubling W_2l(x) = W_l(x) | W_l(x + l) with
    funnel-shift reads up to the largest power of two L <= k, then out(x) = W_L(x - r) | W_L(x + r - L + 1),
    the last word masked to the image;
  * vertical: van Herk / Gil-Werman on the column padded with r zero rows, blocks of k rows, a suffix march over
    block b and a prefix march over block b + 1 per output block;
  * both radii clamped to W - 1 and H - 1 first.

The result must equal cv2.dilate with a k x k box for k up to 1025, widths that are not a multiple of 32 and
kernels wider and taller than the image.  oracle.intmath.dilate_square, the CPU twin the GPU tests lean on, is
pinned to cv2.dilate at these sizes too."""

import cv2
import numpy as np
import pytest

from oracle import intmath as M

MASK32 = np.uint64(0xFFFFFFFF)


def pack_rows(img: np.ndarray) -> np.ndarray:
    """0/255 image -> [H][Wq] row-major words as uint64 (bit i of word q = pixel 32 q + i, padding bits 0)."""
    h, w = img.shape
    wq = (w + 31) // 32
    bits = np.pad(img != 0, ((0, 0), (0, 32 * wq - w)))
    return np.packbits(bits, axis=1, bitorder="little").view("<u4").astype(np.uint64)


def unpack_rows(words: np.ndarray, w: int) -> np.ndarray:
    b = np.unpackbits(words.astype("<u4").view(np.uint8), axis=1, bitorder="little")
    return (b[:, :w] * 255).astype(np.uint8)


def row_bits(a: np.ndarray, d: int) -> np.ndarray:
    """row_bits(a, len, 32 w + d) for every word w of every row: funnel shift of words w + d // 32 and the next,
    words at or past the row's end read as 0."""
    n = a.shape[1]
    wo, s = d >> 5, np.uint64(d & 31)
    ext = np.concatenate([a, np.zeros((a.shape[0], wo + 2), np.uint64)], axis=1)
    lo, hi = ext[:, wo:wo + n], ext[:, wo + 1:wo + 1 + n]
    return (((hi << np.uint64(32)) | lo) >> s) & MASK32


def hdil_rows(plane: np.ndarray, w: int, k: int) -> np.ndarray:
    wq = plane.shape[1]
    r = min(k // 2, w - 1)
    pad = (r + 31) // 32
    big_l = 1
    while 2 * big_l <= 2 * r + 1:
        big_l *= 2
    a = np.concatenate([np.zeros((plane.shape[0], pad), np.uint64), plane], axis=1)
    l, steps = 1, 0
    while l < big_l:
        a = a | row_bits(a, l)
        l <<= 1
        steps += 1
    assert steps == big_l.bit_length() - 1          # log2 k doubling steps, nothing else grows with k
    # output word w covers image bits x = 32 w .., buffer bits 32 (pad + w) ..: positions x - r and x + r - L + 1
    out = (row_bits(a, 32 * pad - r) | row_bits(a, 32 * pad + r - big_l + 1))[:, :wq]
    last = (1 << (w & 31)) - 1 if w & 31 else 0xFFFFFFFF
    out[:, -1] &= np.uint64(last)
    return out


def vdil_cols(hdil: np.ndarray, k: int) -> np.ndarray:
    """The vertical kernel's two marches, one thread per (block, word column) - vectorised over the columns."""
    h = hdil.shape[0]
    r = min(k // 2, h - 1)
    k = 2 * r + 1
    out = np.zeros_like(hdil)
    blocks = (h + k - 1) // k
    for b in range(blocks):
        q0, y_end = b * k, min(b * k + k, h)
        acc = np.zeros(hdil.shape[1], np.uint64)
        for q in range(min(q0 + k - 1, r + h - 1), q0 - 1, -1):
            if q >= r:
                acc = acc | hdil[q - r]
            if q < h:
                out[q] = acc
        acc = np.zeros(hdil.shape[1], np.uint64)
        for y in range(q0, y_end):
            if y > q0:
                out[y] |= acc
            if y + k < r + h:
                acc = acc | hdil[y + k - r]
    return out


def dilate_bits(img: np.ndarray, k: int) -> np.ndarray:
    h, w = img.shape
    return unpack_rows(vdil_cols(hdil_rows(pack_rows(img), w, k), k), w)


def _images(h, w, seed):
    rng = np.random.default_rng(seed)
    sparse = ((rng.random((h, w)) < 0.004) * 255).astype(np.uint8)
    one = np.zeros((h, w), np.uint8)
    one[rng.integers(0, h), rng.integers(0, w)] = 255
    corners = np.zeros((h, w), np.uint8)
    corners[0, 0] = corners[h - 1, w - 1] = 255
    edges = cv2.Canny(cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (7, 7), 0), 20, 60)
    return [sparse, one, corners, edges, np.zeros((h, w), np.uint8)]


@pytest.mark.parametrize("k", [65, 101, 129, 255, 257])
@pytest.mark.parametrize("shape", [(36, 64), (90, 160), (97, 131), (180, 320)])
def test_oracle_dilate_square_equals_cv2_large_k(shape, k):
    h, w = shape
    kernel = np.ones((k, k), np.uint8)
    for img in _images(h, w, h * w + k):
        assert np.array_equal(M.dilate_square(img, k), cv2.dilate(img, kernel))


# (H, W, k): k from 65 to 1025; widths that are not a multiple of 32; k > W, k > H, k above both, k at 2W - 1 /
# 2H - 1 (the clamp) and one short of it
MODEL_CASES = [
    (90, 200, 65), (90, 200, 67), (97, 131, 95), (97, 131, 127), (97, 131, 129), (180, 320, 129),
    (64, 300, 95), (300, 29, 65), (130, 70, 101), (60, 500, 255), (131, 97, 257), (36, 64, 129),
    (97, 131, 193), (97, 131, 261), (97, 131, 263), (200, 90, 399), (200, 90, 401), (40, 1000, 1025),
    (1000, 40, 1025), (20, 33, 1025), (3, 3, 65), (1, 70, 65), (70, 1, 65), (256, 256, 511), (255, 257, 513),
]


@pytest.mark.parametrize("h,w,k", MODEL_CASES)
def test_separable_bit_dilation_equals_cv2(h, w, k):
    kernel = np.ones((k, k), np.uint8)
    for img in _images(h, w, 7 * h + w + k):
        assert np.array_equal(dilate_bits(img, k), cv2.dilate(img, kernel)), (h, w, k)


def test_separable_bit_dilation_every_k_small_frame():
    """every odd k from 65 to 1025 on a 45x77 frame (k passes W, 2W - 1, H and 2H - 1 on the way)."""
    h, w = 45, 77
    imgs = _images(h, w, 11)
    for k in range(65, 1027, 2):
        kernel = np.ones((k, k), np.uint8)
        for img in imgs[:2]:
            assert np.array_equal(dilate_bits(img, k), cv2.dilate(img, kernel)), k
