"""The fused score pass (csrc/score_kernel.cu) under every feature mask it compiles, against a per-geometry oracle.

For each scored geometry the oracle (cv2 HSV / YUV, exact integer sums, cv2.Canny + cv2.dilate) is computed once
and compared bit for bit with all 11 instantiations of psd_score_ws_kernel<F> (and the tail kernel): the H, S, V
SADs, the byte sum, `has_prev`, the Y histogram and, for the masks with edges, the V plane, the Canny map, the
dilated map and the edge SAD of every frame.  The geometries cover every residue P mod 16 (the tail kernel's 1..15
pixels), frames smaller than one thread slice, exactly one strip, a strip plus a 16-pixel strip, partial strips
and multi-strip frames.  The frame counts come from the twin of the kernel's work split (tests/score_split.py), for
the SM count of the device the test runs on: together they reach every `walked mod 4` with and without a halo
frame, a launch with fewer items than SMs and a launch in which one CTA walks items of different slot counts - the
test fails, not skips, when they do not.  Predecessors come from nowhere, from the previous batch, from a host
halo frame and from a device halo frame; frames are submitted from the host, from 16-byte aligned device memory
and from device memory that is not (the copy path)."""

import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from pyscenedetect_b200.synth import ScenePlan, render_frames
from tests import score_split as S

pytestmark = pytest.mark.gpu

MASKS = (1, 2, 3, 4, 5, 6, 7, 9, 11, 13, 15)
F_HSV, F_BGRSUM, F_YHIST, F_EDGES = 1, 2, 4, 8

GEOMETRIES = [
    # P < 16: only the tail kernel runs; W < 8 and H <= 2 for the edge stages
    (1, 1), (7, 1), (15, 1), (1, 15), (7, 2), (5, 9),
    # small frames of one partial strip, residues 2, 4, 5, 6, 10, 11, 12
    (46, 15), (44, 15), (41, 13), (42, 15), (70, 23), (57, 19), (60, 21),
    (128, 96),     # exactly one strip
    (769, 16),     # one strip plus a strip of 16 pixels
    (535, 23),     # the same plus a 1-pixel tail
    (1117, 11),    # one partial strip plus a 15-pixel tail
    (199, 65), (301, 49), (302, 49),   # one strip plus a partial one, tails of 7, 13 and 14 pixels
    (131, 97), (160, 90), (1000, 37), (333, 77), (640, 360), (1920, 1080),
]
# geometries searched (with the device's SM count) for a launch in which a CTA walks items of different slot counts
MIXED_CANDIDATES = [(1280, 720), (800, 600), (1920, 1080)]
MIXED_N_MAX = 160
TINY_LAUNCHES = [(1, False), (3, True), (2, False), (5, True), (4, True)]


@pytest.fixture(scope="module")
def sm_count():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    n = C.c_int(0)
    _capi.check(lib.psd_device_info(0, None, 0, None, None, C.byref(n), None), "psd_device_info")
    assert n.value > 0
    return n.value


# ---- content ----
def v_frame(kind: str, w: int, h: int) -> np.ndarray:
    """B = G = R = a V plane built for the order statistics of psd_edge_thresholds_kernel (raster order, so the
    value boundaries are long horizontal edges of a known gradient)."""
    p = w * h
    half = p // 2
    if kind == "v_half":        # half at 2, half at 3: median 2.5 for even P
        vals = [(2, half), (3, p - half)]
    elif kind == "v_lanes":     # ranks (P-1)//2 and P//2 in bins 7 and 8: lanes 0 and 1 of the warp scan
        q = max(1, p // 8) if p >= 4 else 0
        vals = [(0, half - q), (7, q), (8, q), (20, p - half - q)]
    elif kind == "v_binend":    # the count up to bin 30 is exactly P//2 + 1: the upper rank ends a bin
        n30 = min(p, half + 1)
        vals = [(30, n30), (42, p - n30)]
    elif kind == "v_med0":
        vals = [(0, min(p, half + 1)), (255, p - min(p, half + 1))]
    else:                       # v_med255
        vals = [(0, p - min(p, half + 1)), (255, min(p, half + 1))]
    flat = np.concatenate([np.full(n, v, np.uint8) for v, n in vals if n > 0])
    assert flat.size == p
    return np.repeat(flat.reshape(h, w)[..., None], 3, axis=2)


KINDS = ("plan", "random", "same", "black", "white", "black", "solid", "plan", "v_half", "v_lanes", "v_binend",
         "same", "v_med0", "v_med255", "random", "plan", "white")


def make_frames(w: int, h: int, n: int, seed: int) -> np.ndarray:
    frames = render_frames(ScenePlan(n, seed=seed, min_len=2, max_len=6).params, w, h)
    rng = np.random.default_rng(seed)
    for t in range(n):
        kind = KINDS[(t + seed) % len(KINDS)]
        if kind == "random":
            frames[t] = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        elif kind == "same" and t > 0:
            frames[t] = frames[t - 1]
        elif kind == "black":
            frames[t] = 0
        elif kind == "white":
            frames[t] = 255
        elif kind == "solid":
            frames[t] = (17, 200, 90)
        elif kind.startswith("v_"):
            frames[t] = v_frame(kind, w, h)
    return frames


class Oracle:
    """Per-frame expectations of one frame sequence; SADs against the previous frame of the sequence."""

    def __init__(self, frames: np.ndarray, edges: bool):
        n, h, w = frames.shape[:3]
        self.n = n
        self.bsum = [int(f.sum(dtype=np.int64)) for f in frames]
        self.yhist = np.stack([np.bincount(cv2.cvtColor(f, cv2.COLOR_BGR2YUV)[..., 0].ravel(), minlength=256)
                               for f in frames]).astype(np.uint32)
        hsv = [cv2.cvtColor(f, cv2.COLOR_BGR2HSV) for f in frames]
        assert np.array_equal(hsv[0][..., 2], frames[0].max(axis=2))
        self.sad = [[0, 0, 0]] + [[M.sad(hsv[t][..., c], hsv[t - 1][..., c]) for c in range(3)]
                                   for t in range(1, n)]
        self.lum = [x[..., 2].copy() for x in hsv]
        if edges:
            k = R.estimated_kernel_size(w, h)
            self.ksize = k
            kernel = np.ones((k, k), np.uint8)
            self.canny = []
            for lum in self.lum:
                low, high = M.canny_thresholds(float(np.median(lum)))
                self.canny.append(cv2.Canny(lum, low, high))
            self.dil = [R.detect_edges(lum, kernel) for lum in self.lum]
            self.sad_e = [0] + [M.sad(self.dil[t], self.dil[t - 1]) for t in range(1, n)]

    def check_sums(self, mask: int, sums, t0: int, first_has_prev: bool, tag):
        for j in range(len(sums)):
            t = t0 + j
            p = first_has_prev or j > 0
            got = [int(sums[k][j]) for k in ("sad_hue", "sad_sat", "sad_lum", "sad_edges", "bgr_sum", "has_prev")]
            want = (self.sad[t] if (mask & F_HSV and p) else [0, 0, 0]) + \
                [self.sad_e[t] if (mask & F_EDGES and p) else 0,
                 self.bsum[t] if mask & F_BGRSUM else 0, 1 if p else 0]
            assert got == want, (tag, mask, t, got, want)

    def check_planes(self, eng, t0: int, n: int, tag):
        for j in range(n):
            t = t0 + j
            assert np.array_equal(eng.debug_plane(1, j), self.lum[t]), (tag, t, "V")
            assert np.array_equal(eng.debug_plane(2, j), self.canny[t]), (tag, t, "Canny")
            assert np.array_equal(eng.debug_plane(3, j), self.dil[t]), (tag, t, "dilated")


def schedule(launches):
    """Segments (predecessor, submission, [batch sizes]) that run the given launches (n_frames, has_prev).  A
    segment starts after a reset; its later batches have the previous batch's last frame carried, and a segment
    that starts with a halo has the sequence's previous frame as its predecessor.  Segments without a predecessor
    come first, so every halo frame exists."""
    segs = [["none", [n]] for n, p in launches if not p] or [["none", [1]]]
    for i, n in enumerate(n for n, p in launches if p):
        mode = ("carry", "halo_host", "halo_device")[i % 3]
        if mode == "carry":
            segs[i % len(segs)][1].append(n)
        else:
            segs.append([mode, [n]])
    subs = ("host", "device", "device_unaligned")
    return [(pred, subs[k % 3], batches) for k, (pred, batches) in enumerate(segs)]


def launches_of(segs) -> set:
    """The launches (n_frames, has_prev) a schedule makes."""
    return {(b, pred != "none" or k > 0) for pred, _, batches in segs for k, b in enumerate(batches)}


def run_matrix(src_frames, scored_frames, segs, tag):
    """Every mask over the schedule `segs`; `src_frames` are submitted, `scored_frames` (their downscaled copy, or
    the same) are what the oracle scores."""
    from pyscenedetect_b200.engine import DeviceBuffer, Engine
    n, sh, sw = src_frames.shape[:3]
    h, w = scored_frames.shape[1:3]
    any_edges = any(m & F_EDGES for m in MASKS)
    orc = Oracle(scored_frames, any_edges)
    fb = sw * sh * 3
    dev = DeviceBuffer(n * fb + 16)
    dev.upload(src_frames, offset=0)
    dev_u = DeviceBuffer(n * fb + 16)
    dev_u.upload(src_frames, offset=1)
    max_b = max(max(b) for _, _, b in segs)
    try:
        for mask in MASKS:
            eng = Engine(sw, sh, mask, width=w, height=h, max_batch=max_b)
            if mask & F_EDGES:
                assert eng.edge_kernel_size == orc.ksize
            t = 0
            for pred, sub, batches in segs:
                eng.reset()
                if pred == "halo_host":
                    eng.set_halo(src_frames[t - 1])
                elif pred == "halo_device":
                    eng.set_halo_device(dev.ptr + (t - 1) * fb)
                t0 = t
                for k, b in enumerate(batches):
                    if sub == "host":
                        eng.submit(src_frames[t:t + b])
                    elif sub == "device":
                        eng.submit_device(dev.ptr + t * fb, b)
                    else:
                        eng.submit_device(dev_u.ptr + 1 + t * fb, b)
                    if mask & F_EDGES:
                        orc.check_planes(eng, t, b, (tag, mask, pred, sub))
                    t += b
                sums = eng.read_sums()
                assert len(sums) == t - t0
                orc.check_sums(mask, sums, t0, pred != "none", (tag, pred, sub))
                if mask & F_YHIST:
                    assert np.array_equal(eng.read_yhist(), orc.yhist[t0:t]), (tag, mask, pred, sub)
            eng.close()
    finally:
        dev.close()
        dev_u.close()


def _launches_for(w, h, sm_count):
    return TINY_LAUNCHES if w * h < 16 else S.choose_launches(w * h, sm_count)


@pytest.mark.parametrize("shape", GEOMETRIES)
def test_fused_pass_every_mask(shape, sm_count):
    w, h = shape
    launches = _launches_for(w, h, sm_count)
    if w * h >= 16:
        assert S.required_cases() <= S.coverage(w * h, launches, sm_count)
    segs = schedule(launches)
    n = sum(sum(b) for _, _, b in segs)
    frames = make_frames(w, h, n, seed=w * 7 + h)
    run_matrix(frames, frames, segs, shape)


def mixed_schedule(sm_count):
    """(geometry, schedule) of a launch in which one CTA walks items of different slot counts on this device."""
    for w, h in MIXED_CANDIDATES:
        found = S.find_mixed_launch(w * h, sm_count, MIXED_N_MAX)
        if found:
            n, has_prev = found
            return (w, h), [("none", "device", [1, n])] if has_prev else [("none", "device", [n])]
    raise AssertionError(f"no launch of <= {MIXED_N_MAX} frames has a CTA with mixed slot counts on {sm_count} SMs")


RESIZED_SCHEDULE = schedule([(5, False), (3, True), (2, True), (6, True)])


def test_fused_pass_mixed_slot_cta(sm_count):
    """A launch in which one CTA walks items of different slot counts (found with the twin for this device)."""
    (w, h), segs = mixed_schedule(sm_count)
    assert "mixed" in S.coverage(w * h, launches_of(segs), sm_count)
    frames = make_frames(w, h, sum(segs[0][2]), seed=5)
    run_matrix(frames, frames, segs, (w, h))


def test_fused_pass_resized():
    """1920x1080 submitted, 256x144 scored: the masks see the device downscale's output."""
    segs = RESIZED_SCHEDULE
    n = sum(sum(b) for _, _, b in segs)
    src = make_frames(1920, 1080, n, seed=11)
    scored = np.stack([cv2.resize(f, (256, 144), interpolation=cv2.INTER_LINEAR) for f in src])
    run_matrix(src, scored, segs, "1920x1080->256x144")


def test_matrix_reaches_every_case(sm_count):
    """The launches of the tests above, together, reach every decomposition case on this device."""
    reached = set()
    for w, h in GEOMETRIES:
        reached |= S.coverage(w * h, launches_of(schedule(_launches_for(w, h, sm_count))), sm_count)
    (w, h), segs = mixed_schedule(sm_count)
    reached |= S.coverage(w * h, launches_of(segs), sm_count)
    reached |= S.coverage(256 * 144, launches_of(RESIZED_SCHEDULE), sm_count)
    missing = (S.required_cases() | {"few", "mixed"}) - reached
    assert not missing, sorted(map(str, missing))


# ---- the production shape: 2 048 device-rendered 1080p frames in one launch ----
@pytest.mark.parametrize("mask", [7, 15])
def test_production_batch_2048_at_1080p(sm_count, mask):
    """bench.py's shape (max_batch = 2048): one launch of 2 048 frames gives the same bytes as 2 048 launches of
    one frame, and the oracle agrees at every chunk boundary of the launch and on the last frame.  The frames stay
    on the device; only the sampled ones are downloaded."""
    from pyscenedetect_b200.engine import DeviceBuffer, Engine, synth_frames_device
    w, h, n = 1920, 1080, 2048
    fb = w * h * 3
    sp = S.split(w * h, n, True, False, sm_count)
    plan = ScenePlan(n, seed=21, min_len=3, max_len=40, noise_shift=29)
    buf = DeviceBuffer(n * fb)
    try:
        synth_frames_device(buf.ptr, plan.params, w, h)
        big = Engine(w, h, mask, max_batch=n)
        big.submit_device(buf.ptr, n)
        sums, hist = big.read_sums(), big.read_yhist()
        big.close()
        one = Engine(w, h, mask, max_batch=1)
        one.submit_device(buf.ptr, n)
        assert one.read_sums().tobytes() == sums.tobytes()
        assert one.read_yhist().tobytes() == hist.tobytes()
        one.close()
        c = sp.n_chunks
        bounds = {S.chunk_first(k, n, c) for k in range(1, c)}
        sample = sorted({t for b in bounds for t in (b - 1, b)} | {0, n - 1})
        need = sorted({t for s in sample for t in (s - 1, s) if t >= 0})
        frames = {t: buf.download(fb, t * fb).reshape(h, w, 3) for t in need}
    finally:
        buf.close()
    k = R.estimated_kernel_size(w, h)
    kernel = np.ones((k, k), np.uint8)
    hsv = {t: cv2.cvtColor(f, cv2.COLOR_BGR2HSV) for t, f in frames.items()}
    dil = {t: R.detect_edges(x[..., 2], kernel) for t, x in hsv.items()} if mask & F_EDGES else {}
    for t in sample:
        f = frames[t]
        assert int(sums["bgr_sum"][t]) == int(f.sum(dtype=np.int64)), t
        assert np.array_equal(hist[t], np.bincount(cv2.cvtColor(f, cv2.COLOR_BGR2YUV)[..., 0].ravel(),
                                                   minlength=256)), t
        assert int(sums["has_prev"][t]) == (1 if t else 0)
        want = [M.sad(hsv[t][..., ch], hsv[t - 1][..., ch]) for ch in range(3)] if t else [0, 0, 0]
        assert [int(sums[key][t]) for key in ("sad_hue", "sad_sat", "sad_lum")] == want, t
        if mask & F_EDGES:
            assert int(sums["sad_edges"][t]) == (M.sad(dil[t], dil[t - 1]) if t else 0), t
