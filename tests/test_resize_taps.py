"""The INTER_LINEAR tap tables of the device downscale (engine.cu build_taps, through psd_test_resize_taps) against
oracle.intmath.linear_taps, and the oracle against cv2.resize, at the geometries SceneManager and Engine can produce.

cv2.resize takes its scale as 1 / (dst / src).  src / dst can differ from it in the last bit, and at source sides
above 10 240 pixels that bit can survive the float32 cast of a source position and move an 11-bit coefficient by
one.  `old_taps` below restates the src / dst form, so the tests can find where the two differ and show that the
recorded numbers never depended on it.  Runs without a GPU: the test entry makes no CUDA call."""

import gzip
import hashlib
import json
import os

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from pyscenedetect_b200.synth import ScenePlan, render_frames

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOWNSCALE_GOLDEN = os.path.join(GOLDEN_DIR, "downscale_v1.json")
MAX_SIDE = 32768
FACTORS = range(2, 17)
AUTO_MAX = 256   # auto-downscale scores at most 256 pixels on either side
# source -> scored side where the two scales give different taps (reached by downscale 2, 2, 7 and by Engine(width=))
TABLE = [(10241, 5120), (12287, 6144), (14335, 2048)]
ENGINE_ONLY = (7281, 4096)


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    return _capi.load()


def lib_taps(lib, src, dst):
    ofs = np.empty(dst, np.int32)
    coef = np.empty((dst, 2), np.int16)
    assert lib.psd_test_resize_taps(src, dst, ofs.ctypes.data, coef.ctypes.data) == 0
    return ofs, coef[:, 0].astype(np.int32), coef[:, 1].astype(np.int32)


def old_taps(src, dst):
    """linear_taps with scale = src / dst: the form build_taps and the oracle used before."""
    scale = float(src) / float(dst)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    idx = s.astype(np.int64)
    f[(idx < 0) | (idx >= src - 1)] = 0
    idx = np.clip(idx, 0, src - 1).astype(np.int32)
    c0 = (np.float32(1.0) - f) * np.float32(2048)
    c1 = f * np.float32(2048)
    return idx, np.rint(c0).astype(np.int32), np.rint(c1).astype(np.int32)


def same_taps(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def reachable_pairs(max_side=MAX_SIDE):
    """Every (source side, scored side) with scored < source that SceneManager reaches for sides up to max_side:
    integer downscale 2 … 16 (scored = max(1, round(side / k)), half to even as Python's round) and auto-downscale,
    whose scored sides are at most 256.  A crop reaches any source side, so these are all source sides."""
    src = np.arange(2, max_side + 1, dtype=np.int64)
    keys = [src * 65536 + np.maximum(1, np.round(src / k)).astype(np.int64) for k in FACTORS]
    keys.append((src[:, None] * 65536 + np.arange(1, AUTO_MAX + 1)[None, :]).ravel())
    k = np.unique(np.concatenate(keys))
    s, d = k >> 16, k & 65535
    keep = d < s
    return s[keep], d[keep]


def scale_split_pairs(src, dst):
    """The pairs among (src, dst) where src / dst and 1 / (dst / src) give different taps.  The taps are a function
    of the float32 source positions, so only pairs with different scale doubles are candidates, and of those only
    the ones with a position whose float32 cast differs; the candidates are then checked on the whole tables."""
    sf, df = src.astype(np.float64), dst.astype(np.float64)
    so, sn = sf / df, 1.0 / (df / sf)
    m = so != sn
    src, dst, so, sn = src[m], dst[m], so[m], sn[m]
    order = np.argsort(dst, kind="stable")
    src, dst, so, sn = src[order], dst[order], so[order], sn[order]
    found = []
    for g in np.split(np.arange(len(dst)), np.flatnonzero(np.diff(dst)) + 1):
        n = int(dst[g[0]])
        x = np.arange(n, dtype=np.float64) + 0.5
        a = (x[None, :] * so[g, None] - 0.5).astype(np.float32)
        b = (x[None, :] * sn[g, None] - 0.5).astype(np.float32)
        found += [(int(s), n) for s in src[g][(a != b).any(axis=1)]]
    return sorted(p for p in found if not same_taps(old_taps(*p), M.linear_taps(*p)))


_split: list = []


def split_pairs():
    if not _split:
        _split.extend(scale_split_pairs(*reachable_pairs()))
    return _split


# ---- the library's tables equal the oracle's ----

def test_library_taps_equal_oracle_exhaustive(lib):
    """Every src <= 1 024 and dst < src, element by element (the oracle vectorised over src per dst)."""
    top = 1024
    for dst in range(1, top):
        srcs = np.arange(dst + 1, top + 1)
        want = M.linear_taps(srcs, dst)
        ofs = np.empty((len(srcs), dst), np.int32)
        coef = np.empty((len(srcs), dst, 2), np.int16)
        for i, s in enumerate(srcs):
            assert lib.psd_test_resize_taps(int(s), dst, ofs[i].ctypes.data, coef[i].ctypes.data) == 0
        assert np.array_equal(ofs, want[0]), dst
        assert np.array_equal(coef[..., 0], want[1]), dst
        assert np.array_equal(coef[..., 1], want[2]), dst


def test_library_taps_equal_oracle_where_the_scales_split(lib):
    pairs = split_pairs() + [ENGINE_ONLY]
    for src, dst in pairs:
        assert same_taps(lib_taps(lib, src, dst), M.linear_taps(src, dst)), (src, dst)
        assert not same_taps(lib_taps(lib, src, dst), old_taps(src, dst)), (src, dst)


def test_library_taps_equal_oracle_on_reachable_pairs(lib):
    """Every integer factor and every auto-downscale side for 600 source sides up to 32 768 (those of the
    recorded cases and benchmarks included), plus upscales and equal sizes, which Engine(width=, height=) takes."""
    rng = np.random.default_rng(7)
    sides = np.array(sorted(set(rng.integers(2, MAX_SIDE + 1, 560).tolist()) | set(recorded_sides())
                            | {MAX_SIDE, 10241, 4095}))
    for dst in range(1, AUTO_MAX + 1):   # auto-downscale, the oracle vectorised over the sides
        srcs = sides[sides > dst]
        want = M.linear_taps(srcs, dst)
        for i, src in enumerate(srcs):
            got = lib_taps(lib, int(src), dst)
            assert all(np.array_equal(g, w[i]) for g, w in zip(got, want)), (src, dst)
    for src in sides.tolist():
        for dst in sorted({max(1, round(src / k)) for k in FACTORS} - set(range(1, AUTO_MAX + 1))):
            assert same_taps(lib_taps(lib, src, dst), M.linear_taps(src, dst)), (src, dst)
    for src, dst in [(1, 1), (1, 7), (2, 3), (7, 7), (100, 333), (1080, 1920), (4096, 4096), (3, 32768)]:
        assert same_taps(lib_taps(lib, src, dst), M.linear_taps(src, dst)), (src, dst)


def test_library_rejects_bad_sizes(lib):
    buf = np.zeros(8, np.int32)
    assert lib.psd_test_resize_taps(0, 4, buf.ctypes.data, buf.ctypes.data) != 0
    assert lib.psd_test_resize_taps(4, 0, buf.ctypes.data, buf.ctypes.data) != 0
    assert lib.psd_test_resize_taps(4, 2, None, buf.ctypes.data) != 0


# ---- the oracle equals cv2.resize ----

def test_search_finds_the_known_pairs():
    pairs = split_pairs()
    assert set(TABLE) <= set(pairs), pairs
    assert all(s > 10240 for s, _ in pairs)
    assert not any(d <= AUTO_MAX for s, d in pairs if s <= 16384)   # auto-downscale below 16 384: none
    assert not same_taps(old_taps(*ENGINE_ONLY), M.linear_taps(*ENGINE_ONLY))


def _probe(rng, src, dst):
    """A 2-row random probe resized along x, and its transpose along y: only the tested axis is resampled."""
    img = rng.integers(0, 256, size=(2, src, 3), dtype=np.uint8)
    assert np.array_equal(M.resize_linear(img, dst, 2), cv2.resize(img, (dst, 2), interpolation=cv2.INTER_LINEAR))
    tall = np.ascontiguousarray(img.transpose(1, 0, 2))
    assert np.array_equal(M.resize_linear(tall, 2, dst), cv2.resize(tall, (2, dst), interpolation=cv2.INTER_LINEAR))


def test_oracle_equals_cv2_where_the_scales_split():
    rng = np.random.default_rng(11)
    for src, dst in split_pairs() + [ENGINE_ONLY]:
        _probe(rng, src, dst)


def test_old_scale_differs_from_cv2_on_the_table(monkeypatch):
    """The probe is sharp enough to see the src / dst form: it moves bytes at every pair of the table."""
    monkeypatch.setattr(M, "linear_taps", old_taps)
    rng = np.random.default_rng(12)
    for src, dst in TABLE + [ENGINE_ONLY]:
        img = rng.integers(0, 256, size=(2, src, 3), dtype=np.uint8)
        want = cv2.resize(img, (dst, 2), interpolation=cv2.INTER_LINEAR)
        assert not np.array_equal(M.resize_linear(img, dst, 2), want), (src, dst)


def test_oracle_equals_cv2_on_random_geometries():
    """300 downscales (dst <= src on both axes, as SceneManager resizes).  Upscaling is not pinned: cv2 clamps the
    vertical source row but not its coefficients where a row maps above the first or below the last, and the
    oracle and the kernel clamp both, which can differ by one when the horizontal pass resamples too."""
    rng = np.random.default_rng(13)
    for _ in range(300):
        sw, sh = (int(v) for v in np.exp(rng.uniform(0, np.log(1500), 2)))
        dw, dh = int(rng.integers(1, sw + 1)), int(rng.integers(1, sh + 1))
        img = rng.integers(0, 256, size=(sh, sw, 3), dtype=np.uint8)
        want = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(M.resize_linear(img, dw, dh), want), (sw, sh, dw, dh)


EDGE_GEOMETRIES = (
    [(1, 1, 1, 1), (1, 9, 1, 4), (9, 1, 4, 1), (1, 4096, 1, 2048), (4096, 1, 2048, 1), (1, 7, 1, 1), (7, 1, 1, 1)]
    + [(n + 1, 3, n, 3) for n in (1, 2, 3, 7, 15, 255, 256, 1023, 4095)]          # src = dst + 1
    + [(3, n + 1, 3, n) for n in (1, 2, 3, 255, 4095)]
    + [(w, h, 1, 1) for w, h in ((2, 2), (3, 5), (640, 360), (10241, 2))]         # dst = 1
    + [(640, 360, 1, 144), (640, 360, 256, 1), (4095, 2, 2048, 2)]                # 4095 -> 2048: exact .5 coefficients
)


@pytest.mark.parametrize("sw,sh,dw,dh", EDGE_GEOMETRIES)
def test_oracle_equals_cv2_at_edges(sw, sh, dw, dh):
    rng = np.random.default_rng(sw * 7 + sh)
    img = rng.integers(0, 256, size=(sh, sw, 3), dtype=np.uint8)
    want = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(M.resize_linear(img, dw, dh), want)


def test_exact_half_coefficients_are_reached():
    """4095 -> 2048 (downscale 2 of a 4095-pixel side) puts source positions on odd multiples of 1/4096, so f * 2048
    is an exact half and rounding half to even (lrintf, cvRound) decides the coefficient."""
    _, a0, a1 = M.linear_taps(4095, 2048)
    f = ((np.arange(2048) + 0.5) * (1.0 / (2048 / 4095)) - 0.5).astype(np.float32)
    halves = (f - np.floor(f)) * 2048 % 1 == 0.5
    assert halves.sum() > 1000
    assert (a1[halves] % 2 == 0).all() and (a0[halves] % 2 == 0).all()


# ---- no recorded number depends on the scale form ----

def recorded_sides():
    """Every frame side of the recorded cases (the new downscale_v1.json aside) and of the benchmarks, and of the
    crops the recordings take."""
    sides = set()

    def walk(o):
        if isinstance(o, dict):
            if "gen" in o and isinstance(o["gen"], list):
                sides.update(int(v) for v in o["gen"][1:3])
            if "crop" in o and isinstance(o["crop"], list):
                x0, y0, x1, y1 = o["crop"]
                sides.update({abs(x1 - x0) + 1, abs(y1 - y0) + 1})
            for v in o.values():
                walk(v)
        elif isinstance(o, list):
            for v in o:
                walk(v)

    for name in sorted(os.listdir(GOLDEN_DIR)):
        if name.startswith("downscale_") or not name.endswith((".json", ".json.gz")):
            continue
        path = os.path.join(GOLDEN_DIR, name)
        with (gzip.open(path, "rt") if name.endswith(".gz") else open(path)) as f:
            walk(json.load(f))
    for w, h in [(1920, 1080), (640, 360), (1280, 720), (3840, 2160), (1200, 640), (274, 154), (7680, 4320),
                 (15360, 8640)]:
        sides.update({w, h})
    return sorted(sides)


def test_recorded_geometries_keep_their_taps():
    sides = recorded_sides()
    assert {160, 90, 640, 360, 1920, 1080, 15360, 8640} <= set(sides)
    for src in sides:
        dsts = {max(1, round(src / k)) for k in FACTORS} | set(range(1, min(AUTO_MAX, src) + 1))
        for dst in sorted(dsts):
            assert same_taps(old_taps(src, dst), M.linear_taps(src, dst)), (src, dst)


# ---- the reference's SceneManager at the split sizes ----

def downscale_golden():
    with open(DOWNSCALE_GOLDEN) as f:
        return json.load(f)


def _case_frames(case):
    n, w, h, seed, mn, mx, ns = case["gen"]
    frames = render_frames(ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx).params, w, h)
    assert hashlib.sha256(frames.tobytes()).hexdigest() == case["frames_sha256"]
    return frames


def cropped_and_scored(case, frames):
    """SceneManager's geometry (scene_manager.py:505-535, 657-678): the crop, then the factor from the effective
    size and the scored size from the cropped frame."""
    fh, fw = frames.shape[1:3]
    x0, y0, x1, y1, eff = 0, 0, fw, fh, (fw, fh)
    if "crop" in case:
        cx0, cy0, cx1, cy1 = case["crop"]
        x0, y0, x1, y1 = min(cx0, cx1), min(cy0, cy1), max(cx0, cx1) + 1, max(cy0, cy1) + 1
        eff = (1 + min(x1, fw) - x0, 1 + min(y1, fh) - y0)
        x1, y1 = min(x1, fw), min(y1, fh)
    w, h = x1 - x0, y1 - y0
    factor = R.compute_downscale_factor(max(eff)) if case.get("auto_downscale") else case["downscale"]
    size = (max(1, round(w / factor)), max(1, round(h / factor))) if factor > 1.0 else (w, h)
    return frames[:, y0:y1, x0:x1], size


def run_oracle(case):
    """The oracle's ContentDetector on frames downscaled by intmath.resize_linear: cuts, metrics, CSV sha256."""
    frames, (dw, dh) = cropped_and_scored(case, _case_frames(case))
    det = R.RefContentDetector(fps=case["fps"], with_stats=True, **case["kw"])
    cuts = []
    for t, frame in enumerate(frames):
        small = M.resize_linear(frame, dw, dh) if (dw, dh) != frame.shape[1::-1] else frame
        cuts += det.process_frame(t, small)
    cuts += det.post_process(len(frames) - 1)
    metrics = {str(t): [float(det.metrics[t][k]).hex() if det.metrics[t].get(k) is not None else None
                        for k in case["metric_keys"]] for t in det.metrics}
    csv = R.stats_csv(det.metrics, case["metric_keys"], case["fps"])
    return sorted(set(cuts)), metrics, hashlib.sha256(csv.encode()).hexdigest()


def test_downscale_golden_covers_the_table():
    cases = downscale_golden()["cases"]
    scored = set()
    for c in cases:
        n, w, h = c["gen"][:3]
        frames = np.zeros((1, h, w, 3), np.uint8)
        crop, (dw, dh) = cropped_and_scored(c, frames)
        scored.update({(crop.shape[2], dw), (crop.shape[1], dh)})
    assert set(TABLE) <= scored, scored
    assert any("crop" in c for c in cases)
    assert any(c.get("auto_downscale") and c["gen"][1:3] == [7680, 4320] for c in cases)


@pytest.mark.parametrize("name", [c["name"] for c in downscale_golden()["cases"]])
def test_oracle_reproduces_downscale_golden(name):
    case = next(c for c in downscale_golden()["cases"] if c["name"] == name)
    cuts, metrics, csv_sha = run_oracle(case)
    assert cuts == case["cuts"]
    assert metrics == case["metrics"]
    assert csv_sha == case["csv_sha256"]


def test_old_scale_oracle_misses_the_golden(monkeypatch):
    """With the src / dst taps in the oracle, every recorded case at a split size fails; the three whose geometries
    the two scales agree on (15360 -> 7680 and the auto-downscaled ones) still match."""
    monkeypatch.setattr(M, "linear_taps", old_taps)
    missed = []
    for case in downscale_golden()["cases"]:
        if run_oracle(case) != (case["cuts"], case["metrics"], case["csv_sha256"]):
            missed.append(case["name"])
    assert missed == ["ds2_10241x4", "ds2_12287x6", "ds7_14335x14", "ds2_4x10241", "crop_ds2_10241x4"], missed
