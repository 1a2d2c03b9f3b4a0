"""The edge stages (csrc/edge_kernels.cu) at the benchmark's edge batch: 512 frames of 1920x1080 in one
`Engine(..., F_EDGES, max_batch=512)` batch, so psd_hyst_bits_kernel deals its tiles in at least two passes whatever
its occupancy, then a second batch that reads the carry plane.  ScenePlan frames are mixed with V images built so
that hysteresis has real work: weak chains that must grow up and left (against the order tiles are dealt in) from
one strong segment at their far end, and one-pixel chains whose only link between two tiles is a diagonal step
through the tiles' shared corner, grown in all four diagonal directions.  Every frame's
Canny map, dilated map and edge SAD is compared with cv2."""

import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from pyscenedetect_b200.synth import ScenePlan

W, H, BATCH = 1920, 1080, 512
TILE_W, TILE_H = 64, 32
HYST_CTA_WARPS = 8       # psd_hyst_bits_kernel: 256 threads
HYST_MAX_CTAS_PER_SM = 8
BG, WEAK, STRONG = 100, 120, 140   # median 100 -> Canny thresholds (66, 133): a 20-step edge is weak, 40 strong


def _sm_count() -> int:
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    n = C.c_int(0)
    _capi.check(lib.psd_device_info(0, None, 0, None, None, C.byref(n), None), "psd_device_info")
    return n.value


def _thresholds(v):
    return M.canny_thresholds(float(np.median(v)))


BAND = 6   # weak chains are bands of this width: their two outlines are closed contours that turn every corner


def serpentine(seed: int) -> np.ndarray:
    """Horizontal bands one tile row apart, joined at alternating ends by vertical bands across the tile borders; only
    the end of the last band (bottom) is strong, so the whole chain grows from there back up, against the order the
    tiles are dealt in."""
    v = np.full((H, W), BG, np.uint8)
    rows = list(range(8 + seed % 7, H - TILE_H, TILE_H))
    x0, x1 = 40 + seed % 5, W - 40
    for i, y in enumerate(rows):
        v[y:y + BAND, x0:x1] = WEAK
        if i + 1 < len(rows):
            x = x1 - BAND if i % 2 == 0 else x0
            v[y:rows[i + 1] + BAND, x:x + BAND] = WEAK
    y = rows[-1]
    end = x1 - 24 if len(rows) % 2 == 1 else x0
    v[y:y + BAND, end:end + 24] = STRONG
    return v


def spiral(seed: int) -> np.ndarray:
    """An inward rectangular spiral band seeded by a strong piece at its innermost end: growth runs left, up, right
    and down in turn."""
    v = np.full((H, W), BG, np.uint8)
    top, left, bottom, right = 8 + seed % 3, 8, H - 9 - BAND, W - 9 - BAND
    gap = 3 * BAND
    y, x = top, left
    while bottom - top > 2 * gap and right - left > 2 * gap:
        v[top:top + BAND, left:right + BAND] = WEAK            # right along the top
        v[top:bottom + BAND, right:right + BAND] = WEAK        # down the right side
        v[bottom:bottom + BAND, left:right + BAND] = WEAK      # left along the bottom
        v[top + gap:bottom + BAND, left:left + BAND] = WEAK    # up the left side, stopping short of the top
        v[top + gap:top + gap + BAND, left:left + gap + BAND] = WEAK   # into the next ring
        y, x = top + gap, left + gap
        top, left, bottom, right = top + gap, left + gap, bottom - gap, right - gap
    v[y:y + BAND, x:x + BAND] = STRONG
    return v


def corner_chains(anti: bool, from_top: bool, seed: int) -> np.ndarray:
    """Diagonal bands whose outlines are one-pixel Canny chains that cross tile corners diagonally.

    Each band runs along x - y = c (or, `anti`, x + y = c). Its edges are soft steps: BG, BG + 8 on the
    diagonal, then BG + 16 inside. The gradient therefore peaks in a single pixel on each outline, just above
    the low threshold. With c = 0 mod 32 (or 31 mod 32) an outline steps from (32 m - 1, 64 k - 1) to
    (32 m, 64 k) (or from (32 m - 1, 64 k) to (32 m, 64 k - 1)) at every corner it meets. There the two tiles
    share no edge-adjacent pixels. Only the strip of the band nearest the top (`from_top`) or the bottom row
    is strong, so growth crosses every corner in one direction. The four frames need, in turn, the ring bit
    above-left (lane 0, `g_l`), below-right (lane 31, `g_r`), above-right (lane 0, `g_r`) and below-left
    (lane 31, `g_l`)."""
    d, width, spacing = 16, 40, 256
    v = np.full((H, W), BG, np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    s = (xx + yy) if anti else (xx - yy)
    base = 31 if anti else 0
    for c in range(-H - 2 * spacing + 32 * (seed % 8), W + H + spacing, spacing):
        c0 = c - c % 32 + base
        band = (s > c0) & (s < c0 + width)
        edge = (s == c0) | (s == c0 + width)
        if band.sum() < 4000:
            continue
        v[band] = BG + d
        v[edge] = BG + d // 2
        ys, xs = np.nonzero(band | edge)
        key = ys if from_top else -ys
        sel = key <= np.sort(key)[24 * (width + 1)]
        v[ys[sel], xs[sel]] = np.where(edge[ys[sel], xs[sel]], BG + d, BG + 2 * d)
    return v


def hysteresis_model(v: np.ndarray, corner_links: bool = True) -> np.ndarray:
    """Canny's hysteresis as the 8-connected components of the candidate map, cv2.Canny(V, low, low), that
    contain a strong pixel, cv2.Canny(V, high, high). With `corner_links` False, no step may cross a 32-row
    tile border and a 64-column tile border at once."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    low, high = _thresholds(v)
    cand = cv2.Canny(v, low, low) > 0
    strong = cv2.Canny(v, high, high) > 0
    h, w = v.shape
    idx = np.full((h, w), -1, np.int64)
    ys, xs = np.nonzero(cand)
    idx[ys, xs] = np.arange(ys.size)
    a, b = [], []
    for dy, dx in ((0, 1), (1, 0), (1, 1), (1, -1)):
        x0, x1 = max(0, -dx), w - max(0, dx)
        p, q = idx[:h - dy, x0:x1], idx[dy:, x0 + dx:x1 + dx]
        ok = (p >= 0) & (q >= 0)
        if not corner_links and dy and dx:
            ry, rx = np.mgrid[0:h - dy, x0:x1]
            ok &= ~(((ry + dy) // TILE_H != ry // TILE_H) & ((rx + dx) // TILE_W != rx // TILE_W))
        a.append(p[ok])
        b.append(q[ok])
    a, b = np.concatenate(a), np.concatenate(b)
    _, label = connected_components(coo_matrix((np.ones(a.size), (a, b)), shape=(ys.size, ys.size)), directed=False)
    keep = np.zeros(label.max() + 1 if ys.size else 0, bool)
    keep[label[strong[ys, xs]]] = True
    out = np.zeros((h, w), np.uint8)
    out[ys[keep[label]], xs[keep[label]]] = 255
    return out


def check_needs_hysteresis(v: np.ndarray, min_pixels: int, min_tiles: int):
    """The frame is shown to need hysteresis: growing from the strong pixels adds many pixels over many tiles."""
    low, high = _thresholds(v)
    full = cv2.Canny(v, low, high)
    strong_only = cv2.Canny(v, high, high)
    grown = (full > 0) & ~(strong_only > 0)
    ys, xs = np.nonzero(grown)
    assert ys.size >= min_pixels, ys.size
    assert len(set(zip((ys // TILE_H).tolist(), (xs // TILE_W).tolist()))) >= min_tiles


# (name, V image of frame t, needs links through tile corners)
ADVERSARIAL = [("serpentine", serpentine, False), ("spiral", spiral, False),
               ("corners_down_right", lambda t: corner_chains(False, True, t), True),
               ("corners_up_left", lambda t: corner_chains(False, False, t), True),
               ("corners_down_left", lambda t: corner_chains(True, True, t), True),
               ("corners_up_right", lambda t: corner_chains(True, False, t), True)]
N_FRAMES = BATCH + 40      # a second batch of 40 frames reads the carry plane of the first
ADV_FRAMES = {t: ADVERSARIAL[(t // 16) % len(ADVERSARIAL)] for t in range(3, N_FRAMES, 16)}   # every 16th frame


def test_adversarial_frames_need_hysteresis():
    """Every designed frame the GPU test submits: the model reproduces cv2.Canny, growth from the strong pixels
    adds many pixels over many tiles, and for the corner frames growth without tile-corner links loses pixels."""
    for t, (name, make, corner) in ADV_FRAMES.items():
        v = make(t)
        low, high = _thresholds(v)
        full = hysteresis_model(v)
        assert np.array_equal(full, cv2.Canny(v, low, high)), (name, t)
        if corner:
            check_needs_hysteresis(v, min_pixels=5000, min_tiles=150)
            lost = (full > 0) & ~(hysteresis_model(v, corner_links=False) > 0)
            assert lost.sum() >= 2000, (name, t, int(lost.sum()))
        else:
            check_needs_hysteresis(v, min_pixels=20000, min_tiles=500)


@pytest.mark.gpu
def test_edge_batch_512_at_1080p_and_carry():
    from pyscenedetect_b200.engine import F_EDGES, DeviceBuffer, Engine, synth_frames_device
    sms = _sm_count()
    tiles = ((W + TILE_W - 1) // TILE_W) * ((H + TILE_H - 1) // TILE_H)
    assert tiles == 1020
    # one pass deals grid x 8 warps x 32 tiles, grid <= SMs x 8 CTAs: more tiles than that means >= 2 passes
    assert BATCH * tiles > sms * HYST_MAX_CTAS_PER_SM * HYST_CTA_WARPS * 32
    fb = W * H * 3
    n = N_FRAMES
    plan = ScenePlan(n, seed=17, min_len=2, max_len=30, noise_shift=29)
    adv = ADV_FRAMES   # B = G = R = the V image
    buf = DeviceBuffer(n * fb)
    eng = Engine(W, H, F_EDGES, max_batch=BATCH)
    try:
        synth_frames_device(buf.ptr, plan.params, W, H)
        for t, (_, make, _) in adv.items():
            buf.upload(np.repeat(make(t)[..., None], 3, axis=2), offset=t * fb)
        k = eng.edge_kernel_size
        assert k == R.estimated_kernel_size(W, H)
        kernel = np.ones((k, k), np.uint8)
        prev = None
        for b0, b1 in ((0, BATCH), (BATCH, n)):
            eng.submit_device(buf.ptr + b0 * fb, b1 - b0)
            sums = eng.read_sums(b0, b1 - b0)
            for t in range(b0, b1):
                f = buf.download(fb, t * fb).reshape(H, W, 3)
                lum = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2]
                low, high = _thresholds(lum)
                assert np.array_equal(eng.debug_plane(2, t - b0), cv2.Canny(lum, low, high)), t
                want = R.detect_edges(lum, kernel)
                assert np.array_equal(eng.debug_plane(3, t - b0), want), t
                assert int(sums["sad_edges"][t - b0]) == (M.sad(want, prev) if prev is not None else 0), t
                prev = want
    finally:
        eng.close()
        buf.close()
