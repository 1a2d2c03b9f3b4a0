"""GPU parity tests: the CUDA path (through the C-ABI) against the oracle and the committed
golden fixtures recorded from the real reference.  Integer-derived metrics are compared
bit-exactly; `hist_diff` (cv2's SIMD summation order is not reproduced) to 1e-9, far inside
the 1e-4 tolerance BASELINE.json states."""

import ctypes as C
import hashlib
import io

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from tests.golden_util import case_frames, case_names, get_case, golden_metrics

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


def _build(case):
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    kw = dict(case["kw"])
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    if "filter_mode" in kw:
        kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
    if "method" in kw:
        kw["method"] = ThresholdDetector.Method[kw["method"]]
    cls = {"content": ContentDetector, "adaptive": AdaptiveDetector, "threshold": ThresholdDetector,
           "histogram": HistogramDetector, "hash": HashDetector}[case["det"]]
    return cls(**kw)


def _check_stats(case, stats, n):
    from pyscenedetect_b200 import FrameTimecode
    gold = golden_metrics(case)
    keys = case["metric_keys"]
    for t in range(n):
        vals = stats.get_metrics(FrameTimecode(t, case["fps"]), keys)
        if t not in gold:
            assert all(v is None for v in vals), (t, vals)
            continue
        for k, v in zip(keys, vals):
            want = gold[t][k]
            if want is None:
                assert v is None, (t, k, v)
            elif k.startswith("hist_diff"):
                assert abs(float(v) - want) < 1e-9, (t, k, float(v), want)
            else:
                assert float(v) == want, (t, k, float(v), want)
    if not any(k.startswith("hist_diff") for k in keys):
        buf = io.StringIO()
        stats.save_to_csv(buf)
        assert buf.getvalue().splitlines()[:4] == case["csv_head"]
        assert hashlib.sha256(buf.getvalue().encode()).hexdigest() == case["csv_sha256"]


def _scored_size(case):
    n, w, h = case["gen"][:3]
    if case["mode"] != "scene_manager":
        return None
    f = R.compute_downscale_factor(max(w, h)) if case.get("auto_downscale") else float(case.get("downscale", 1))
    return R.downscaled_size(w, h, f) if f > 1.0 else None


@pytest.mark.parametrize("name", case_names())
def test_strict_per_frame_matches_reference_golden(lib, name):
    """detector.process_frame(timecode, frame) one frame at a time, as SceneManager drives it."""
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    case = get_case(name)
    frames = case_frames(case)
    n = frames.shape[0]
    det = _build(case)
    stats = StatsManager() if case["stats"] else None
    det.stats_manager = stats
    if stats is not None:
        stats.register_metrics(det.get_metrics())
    det.configure(scored_size=_scored_size(case))
    cuts = []
    for i in range(n):
        cuts += det.process_frame(FrameTimecode(i, case["fps"]), frames[i])
    cuts += det.post_process(FrameTimecode(n - 1, case["fps"]))
    assert sorted({c.frame_num for c in cuts}) == case["cuts"]
    if stats is not None:
        _check_stats(case, stats, n)
    det.close()


@pytest.mark.parametrize("batch", [7, 64])
@pytest.mark.parametrize("name", case_names())
def test_batched_scene_manager_matches_reference_golden(lib, name, batch):
    """Same cases through the batched SceneManager (shared fused pass, on-device downscale)."""
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    case = get_case(name)
    frames = case_frames(case)
    stats = StatsManager() if case["stats"] else None
    sm = SceneManager(stats, batch_size=batch)
    sm.add_detector(_build(case))
    if case["mode"] == "scene_manager" and case.get("auto_downscale"):
        sm.auto_downscale = True
    else:
        sm.auto_downscale = False
        sm.downscale = case.get("downscale", 1)
    total = sm.detect_scenes(ArrayVideoStream(frames, case["fps"]))
    assert total == frames.shape[0]
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    if case["scene_list"] is not None:
        assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    if stats is not None:
        _check_stats(case, stats, frames.shape[0])


def test_hsv_and_y_exhaustive_2_24(lib):
    """Every BGR colour through the device functions of the fused kernel vs cv2."""
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v & 255), (v >> 8) & 255, (v >> 16) & 255], axis=-1).astype(np.uint8)
    n = img.shape[0]
    h, s, val, y = (np.empty(n, np.uint8) for _ in range(4))
    from pyscenedetect_b200 import _capi
    _capi.check(lib.psd_test_hsv(0, img.ctypes.data, n, h.ctypes.data, s.ctypes.data,
                                 val.ctypes.data, y.ctypes.data))
    want = cv2.cvtColor(img.reshape(4096, 4096, 3), cv2.COLOR_BGR2HSV).reshape(-1, 3)
    assert np.array_equal(h, want[:, 0])
    assert np.array_equal(s, want[:, 1])
    assert np.array_equal(val, want[:, 2])
    wy = cv2.cvtColor(img.reshape(4096, 4096, 3), cv2.COLOR_BGR2YUV).reshape(-1, 3)[:, 0]
    assert np.array_equal(y, wy)


def test_device_generator_matches_numpy(lib):
    from pyscenedetect_b200.engine import DeviceBuffer, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    for (w, h, ns) in [(160, 90, 30), (131, 97, 29), (64, 36, 32)]:
        plan = ScenePlan(40, seed=5, min_len=10, max_len=20, noise_shift=ns)
        want = render_frames(plan.params, w, h)
        buf = DeviceBuffer(want.nbytes)
        synth_frames_device(buf.ptr, plan.params, w, h)
        got = buf.download(want.nbytes).reshape(want.shape)
        assert np.array_equal(got, want)
        buf.close()


@pytest.mark.parametrize("shape", [(160, 90), (131, 97), (17, 5), (1, 1), (4096, 3), (640, 360), (64, 36)])
def test_integer_sums_any_shape(lib, shape):
    """Raw integer outputs vs the oracle for aligned, unaligned, tiny and partial-strip sizes; the same frames
    submitted from device memory at a base pointer that is not 16-byte aligned give the same bytes.  64x36 submits
    9 000 frames in calls of 1 000 (batches of 256), so the engine's result slots grow from 4 096 to 8 192 with
    4 000 frames' results in place and to 16 384 with 8 000; the frames right after each growth read the
    previous frame carried across it."""
    from pyscenedetect_b200.engine import F_BGRSUM, F_HSV, F_YHIST, DeviceBuffer, Engine
    w, h = shape
    n, batch, chunk = (9000, 256, 1000) if shape == (64, 36) else (9, 4, 9)
    rng = np.random.default_rng(w * 1000 + h)
    frames = rng.integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)
    eng = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, max_batch=batch)
    for i in range(0, n, chunk):
        eng.submit(frames[i:i + chunk])
    sums = eng.read_sums()
    hist = eng.read_yhist()
    buf = DeviceBuffer(frames.nbytes + 16)
    buf.upload(frames, offset=1)
    dev = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, max_batch=batch)
    for i in range(0, n, chunk):
        dev.submit_device(buf.ptr + 1 + i * frames[0].nbytes, min(chunk, n - i))
    assert dev.frame_count == n
    assert dev.read_sums().tobytes() == sums.tobytes()
    assert np.array_equal(dev.read_yhist(), hist)
    dev.close()
    buf.close()
    prev = None
    for i, f in enumerate(frames):
        hsv = M.bgr_to_hsv(f)
        assert int(sums["bgr_sum"][i]) == int(f.astype(np.int64).sum())
        assert np.array_equal(hist[i], np.bincount(M.bgr_to_y(f).ravel(), minlength=256))
        assert int(sums["has_prev"][i]) == (1 if i else 0)
        if prev is not None:
            assert int(sums["sad_hue"][i]) == M.sad(hsv[0], prev[0])
            assert int(sums["sad_sat"][i]) == M.sad(hsv[1], prev[1])
            assert int(sums["sad_lum"][i]) == M.sad(hsv[2], prev[2])
        prev = hsv
    eng.close()


def test_strided_crop_view_and_batch_invariance(lib):
    """Non-contiguous (cropped) input views and any batching give identical integer sums."""
    from pyscenedetect_b200.engine import F_BGRSUM, F_HSV, F_YHIST, Engine
    rng = np.random.default_rng(3)
    big = rng.integers(0, 256, size=(20, 120, 200, 3), dtype=np.uint8)
    view = big[:, 10:100, 20:180]  # 160x90 crop, non-contiguous rows
    ref = None
    for batches in ([20], [1] * 20, [3, 7, 10], [19, 1]):
        eng = Engine(160, 90, F_HSV | F_BGRSUM | F_YHIST, max_batch=8)
        i = 0
        for b in batches:
            eng.submit(view[i:i + b])
            i += b
        got = (eng.read_sums().tobytes(), eng.read_yhist().tobytes())
        eng.close()
        if ref is None:
            ref = got
            want = Engine(160, 90, F_HSV | F_BGRSUM | F_YHIST)
            want.submit(np.ascontiguousarray(view))
            assert want.read_sums().tobytes() == ref[0]
            want.close()
        assert got == ref


def test_halo_shards_equal_serial(lib):
    """Contiguous time shards with a one-frame halo reproduce the serial run exactly.  (131x97: a frame of
    12707 pixels, whose last 3 go through the tail kernel, staged at a stride that is not 16-byte aligned.)"""
    from pyscenedetect_b200.engine import F_BGRSUM, F_EDGES, F_HSV, F_YHIST, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    for w, h in ((192, 108), (131, 97)):
        frames = render_frames(ScenePlan(60, seed=2, min_len=10, max_len=25).params, w, h)
        feats = F_HSV | F_BGRSUM | F_YHIST | F_EDGES
        serial = Engine(w, h, feats)
        serial.submit(frames)
        want_s, want_h = serial.read_sums(), serial.read_yhist()
        want_c = serial.scan_hist_correl(256)
        for shards in (2, 3, 4):
            bounds = [round(i * 60 / shards) for i in range(shards + 1)]
            got_s, got_h, got_c = [], [], []
            for r in range(shards):
                eng = Engine(w, h, feats)
                if r > 0:
                    eng.set_halo(frames[bounds[r] - 1])
                eng.submit(frames[bounds[r]:bounds[r + 1]])
                got_s.append(eng.read_sums())
                got_h.append(eng.read_yhist())
                got_c.append(eng.scan_hist_correl(256))
                eng.close()
            assert np.concatenate(got_s).tobytes() == want_s.tobytes(), (w, h, shards)
            assert np.array_equal(np.concatenate(got_h), want_h)
            c = np.concatenate(got_c)
            assert np.array_equal(c[1:], want_c[1:]) and np.isnan(c[0]) and np.isnan(want_c[0])
        serial.close()


@pytest.mark.parametrize("src,dst", [((640, 360), (256, 144)), ((1920, 1080), (256, 144)),
                                     ((480, 270), (160, 90)), ((131, 97), (50, 37)),
                                     ((512, 288), (256, 144))])
def test_device_resize_bit_exact(lib, src, dst):
    from pyscenedetect_b200.engine import F_BGRSUM, Engine
    rng = np.random.default_rng(src[0])
    frames = rng.integers(0, 256, size=(3, src[1], src[0], 3), dtype=np.uint8)
    eng = Engine(src[0], src[1], F_BGRSUM, width=dst[0], height=dst[1])
    eng.submit(frames)
    for i in range(3):
        want = cv2.resize(frames[i], dst, interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(eng.debug_plane(0, i), want)
    eng.close()


@pytest.mark.parametrize("shape", [(320, 180), (131, 97), (70, 33), (29, 300)])
def test_edge_intermediates_match_cv2(lib, shape):
    """V plane, Canny map and dilated edges of every frame vs cv2 (content_detector.py:213-239).
    The odd sizes exercise partial 64x32 hysteresis tiles, partial 28-column classify bands, rows
    that are not a multiple of 4 bytes and images narrower than one tile."""
    from pyscenedetect_b200.engine import F_EDGES, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    w, h = shape
    frames = render_frames(ScenePlan(12, seed=4, min_len=4, max_len=8).params, w, h)
    rng = np.random.default_rng(0)
    extra = np.stack([np.zeros((h, w, 3), np.uint8), np.full((h, w, 3), 255, np.uint8),
                      rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
                      cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (9, 9), 0)])
    frames = np.concatenate([frames, extra])
    eng = Engine(w, h, F_EDGES, max_batch=16)
    eng.submit(frames)
    k = eng.edge_kernel_size
    assert k == R.estimated_kernel_size(w, h)
    kernel = np.ones((k, k), np.uint8)
    prev = None
    sums = eng.read_sums()
    for i, f in enumerate(frames):
        lum = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2]
        assert np.array_equal(eng.debug_plane(1, i), lum)
        low, high = M.canny_thresholds(float(np.median(lum)))
        assert np.array_equal(eng.debug_plane(2, i), cv2.Canny(lum, low, high)), i
        want = R.detect_edges(lum, kernel)
        assert np.array_equal(eng.debug_plane(3, i), want), i
        if prev is not None:
            assert int(sums["sad_edges"][i]) == M.sad(want, prev)
        prev = want
    eng.close()


@pytest.mark.parametrize("k", [3, 9, 17, 19, 25])
def test_edge_dilation_kernel_sizes(lib, k):
    """Explicit dilation kernel sizes: k <= 17 runs the register-ring kernel (R = 1 .. 8), larger k (the estimate for
    4K frames is 19) the one-thread-per-word kernel; dilated map and edge SAD vs cv2.dilate."""
    from pyscenedetect_b200.engine import F_EDGES, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    w, h = 200, 90
    frames = render_frames(ScenePlan(10, seed=6, min_len=4, max_len=6).params, w, h)
    eng = Engine(w, h, F_EDGES, max_batch=4, edge_kernel_size=k)   # several sub-batches: the carry plane is used
    assert eng.edge_kernel_size == k
    kernel = np.ones((k, k), np.uint8)
    prev = None
    for b in range(0, len(frames), 4):
        eng.submit(frames[b:b + 4])
        sums = eng.read_sums(b, min(4, len(frames) - b))
        for j, f in enumerate(frames[b:b + 4]):
            lum = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2]
            want = R.detect_edges(lum, kernel)
            assert np.array_equal(eng.debug_plane(3, j), want), (k, b + j)
            if prev is not None:
                assert int(sums["sad_edges"][j]) == M.sad(want, prev), (k, b + j)
            prev = want
    eng.close()


def test_edge_path_matches_cv2_at_1080p(lib):
    """BASELINE.json configs[2] size: Canny map, dilated edges and the edge SAD of 1920x1080 frames vs cv2
    (30 x 34 hysteresis tiles, k = 13, components spanning many tiles).  The blurred-noise frames are dense
    with short components, the ramp-plus-noise frame has long weak chains that only resolve over many
    rounds across tile borders, the raw noise frame is the worst case for the candidate density."""
    from pyscenedetect_b200.engine import F_EDGES, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    w, h = 1920, 1080
    frames = render_frames(ScenePlan(4, seed=9, min_len=2, max_len=3).params, w, h)
    rng = np.random.default_rng(3)
    noise = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    ramp = ((xx * 255) // (w - 1)).astype(np.uint8)
    weak = np.clip(ramp[..., None].astype(np.int16) + rng.integers(-9, 10, (h, w, 3)), 0, 255).astype(np.uint8)
    extra = np.stack([cv2.GaussianBlur(noise, (5, 5), 0), cv2.GaussianBlur(noise, (15, 15), 0), weak, noise])
    frames = np.concatenate([frames, extra])
    eng = Engine(w, h, F_EDGES, max_batch=8)
    eng.submit(frames)
    k = eng.edge_kernel_size
    assert k == R.estimated_kernel_size(w, h) == 13
    kernel = np.ones((k, k), np.uint8)
    sums = eng.read_sums()
    prev = None
    for i, f in enumerate(frames):
        lum = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2]
        low, high = M.canny_thresholds(float(np.median(lum)))
        assert np.array_equal(eng.debug_plane(2, i), cv2.Canny(lum, low, high)), i
        want = R.detect_edges(lum, kernel)
        assert np.array_equal(eng.debug_plane(3, i), want), i
        if prev is not None:
            assert int(sums["sad_edges"][i]) == M.sad(want, prev), i
        prev = want
    eng.close()


def test_histogram_path_matches_oracle_at_4k(lib):
    """BASELINE.json configs[3] size: the 256-bin Y histogram of 3840x2160 frames vs numpy.bincount of the
    oracle's Y plane (= cv2 COLOR_BGR2YUV), and hist_diff vs cv2.compareHist(CORREL) on cv2's own histograms."""
    from pyscenedetect_b200.engine import F_YHIST, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    w, h = 3840, 2160
    frames = render_frames(ScenePlan(3, seed=5, min_len=1, max_len=2).params, w, h)
    rng = np.random.default_rng(8)
    frames = np.concatenate([frames, rng.integers(0, 256, (1, h, w, 3), dtype=np.uint8)])
    eng = Engine(w, h, F_YHIST, max_batch=4)
    eng.submit(frames)
    yh = eng.read_yhist()
    diffs = eng.scan_hist_correl(256)
    eng.close()
    prev = None
    for i, f in enumerate(frames):
        y = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2YUV))[0]
        assert np.array_equal(M.bgr_to_y(f), y)
        assert np.array_equal(yh[i], np.bincount(y.ravel(), minlength=256)), i
        hist = R.calculate_histogram(f, bins=256)
        if prev is not None:
            assert abs(diffs[i] - cv2.compareHist(prev, hist, cv2.HISTCMP_CORREL)) < 1e-9, i
        prev = hist


@pytest.mark.parametrize("shape,size,lowpass", [((160, 90), 8, 2), ((256, 144), 8, 2), ((1920, 1080), 8, 2),
                                                ((3840, 2160), 8, 2), ((131, 97), 4, 2), ((640, 360), 16, 4),
                                                ((32, 32), 8, 2), ((64, 64), 16, 4), ((1280, 720), 12, 3)])
def test_frame_hashes_match_cv2(lib, shape, size, lowpass):
    """hash_detector.py:124-158: every hash bit of every frame vs the reference's own cv2 call sequence
    (non-integer area scales, the integer-scale path incl. 2x2, mixed 1920x1080, no resize at all)."""
    from pyscenedetect_b200.engine import F_HASH, Engine
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    w, h = shape
    n = 6 if w * h > 1000000 else 24
    frames = render_frames(ScenePlan(n, seed=w + size, min_len=2, max_len=5).params, w, h)
    rng = np.random.default_rng(w)
    extra = [np.zeros((h, w, 3), np.uint8), rng.integers(0, 256, (h, w, 3), dtype=np.uint8)]
    n_img = size * lowpass
    if n_img & (n_img - 1) == 0:
        # solid colours: every AC coefficient is exactly 0, the bits are decided by how the transform cancels;
        # the folded DCT reproduces cv2 for power-of-two hash images (cv2's noise for other sizes is its own)
        extra += [np.full((h, w, 3), 255, np.uint8), np.full((h, w, 3), 37, np.uint8)]
    frames = np.concatenate([frames, np.stack(extra)])
    eng = Engine(w, h, F_HASH, max_batch=8, hash_size=size, hash_lowpass=lowpass)
    eng.submit(frames)
    got = eng.read_hash()
    dist = eng.scan_hash_dist()
    eng.close()
    m = size * size
    prev = None
    for i, f in enumerate(frames):
        want = R.hash_frame(f, size, lowpass).ravel()
        bits = np.array([(int(got[i, k >> 6]) >> (k & 63)) & 1 for k in range(m)], dtype=bool)
        assert np.array_equal(bits, want), (i, int((bits != want).sum()))
        if prev is None:
            assert np.isnan(dist[i])
        else:
            assert dist[i] == np.count_nonzero(want != prev) / float(m)
        prev = want


def test_errors_are_loud(lib):
    from pyscenedetect_b200 import FrameTimecode
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector, HistogramDetector
    from pyscenedetect_b200.engine import F_HSV, Engine
    with pytest.raises(ValueError):
        ContentDetector(kernel_size=4)
    with pytest.raises(ValueError):
        AdaptiveDetector(window_width=0)
    with pytest.raises(ValueError):
        HistogramDetector().process_frame(FrameTimecode(0, 30.0), np.zeros((9, 16, 3), np.float32))
    with pytest.raises(ValueError):
        HistogramDetector().process_frame(FrameTimecode(0, 30.0), np.zeros((9, 16, 4), np.uint8))
    eng = Engine(16, 9, F_HSV)
    with pytest.raises(ValueError):
        eng.submit(np.zeros((2, 10, 16, 3), np.uint8))  # wrong size
    with pytest.raises(ValueError):
        eng.read_sums(0, 5)  # out of range
    eng.close()
    with pytest.raises(ValueError):
        Engine(16, 9, 0)
    from pyscenedetect_b200 import _capi
    cfg = _capi.PsdConfig(struct_size=C.sizeof(_capi.PsdConfig), src_width=16, src_height=9, width=16, height=9,
                          features=F_HSV, max_batch=1, flags=1)
    h = C.c_void_p()
    assert lib.psd_engine_create(C.byref(cfg), C.byref(h)) == _capi.PSD_ERR_INVALID  # no flags are defined
    assert not h.value


@pytest.mark.parametrize("shape", [(1920, 1080), (640, 360), (3840, 2160), (1000, 37)])
def test_score_pass_matches_oracle_at_full_size(lib, shape):
    """Every frame's integer sums and Y histogram from a device-resident sequence vs the integer oracle.
    (1920x1080 and 3840x2160 exercise the full and partial warp-specialised strips; 1000x37, submitted at
    its tight, not 16-byte aligned frame stride, the aligned copy and the tail kernel for the last 8 pixels.)"""
    from pyscenedetect_b200.engine import F_BGRSUM, F_HSV, F_YHIST, DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan
    w, h = shape
    n = 70 if w * h < 3000000 else 12   # > one 64-frame chunk where memory allows
    plan = ScenePlan(n, seed=9, min_len=5, max_len=12, noise_shift=29)
    buf = DeviceBuffer(n * w * h * 3)
    synth_frames_device(buf.ptr, plan.params, w, h)
    eng = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, max_batch=128)
    eng.submit_device(buf.ptr, n)
    sums, hist = eng.read_sums(), eng.read_yhist()
    eng.close()
    frames = buf.download(n * w * h * 3).reshape(n, h, w, 3)
    buf.close()
    prev = None
    for i, f in enumerate(frames):
        hsv = M.bgr_to_hsv(f)
        want = [M.sad(hsv[c], prev[c]) for c in range(3)] if prev is not None else [0, 0, 0]
        got = [int(sums[k][i]) for k in ("sad_hue", "sad_sat", "sad_lum")]
        assert got == want, (i, got, want)
        assert int(sums["sad_edges"][i]) == 0
        assert int(sums["bgr_sum"][i]) == int(f.astype(np.int64).sum()), i
        assert int(sums["has_prev"][i]) == (1 if i else 0)
        assert np.array_equal(hist[i], np.bincount(M.bgr_to_y(f).ravel(), minlength=256)), i
        prev = hsv


def test_full_size_properties_1080p(lib):
    """Size-independent properties at the benchmark's full frame size (1920x1080), device-resident:
    identical frames score 0; black<->white gives the extreme sums and the exact correlation
    -1/(bins-1); contiguous time shards with a halo equal the serial run; re-submitting is
    idempotent."""
    from pyscenedetect_b200.engine import F_BGRSUM, F_HSV, F_YHIST, DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan
    w, h = 1920, 1080
    npx, fb = w * h, w * h * 3
    feats = F_HSV | F_BGRSUM | F_YHIST
    # (1)/(2): hand-made frames
    frames = np.zeros((5, h, w, 3), np.uint8)
    frames[1] = 255                      # black -> white
    frames[2] = 255                      # white -> white (identical)
    frames[3, :, :, 2] = 255             # pure red
    frames[4, :, :, 2] = 255             # identical again
    eng = Engine(w, h, feats)
    eng.submit(frames)
    s = eng.read_sums()
    assert (int(s["sad_lum"][1]), int(s["sad_sat"][1]), int(s["sad_hue"][1])) == (255 * npx, 0, 0)
    assert (int(s["sad_lum"][2]), int(s["sad_sat"][2]), int(s["sad_hue"][2])) == (0, 0, 0)
    assert (int(s["sad_lum"][3]), int(s["sad_sat"][3]), int(s["sad_hue"][3])) == (0, 255 * npx, 0)
    assert int(s["sad_lum"][4]) == 0 and int(s["bgr_sum"][4]) == 255 * npx
    assert int(s["bgr_sum"][1]) == 3 * 255 * npx and int(s["bgr_sum"][0]) == 0
    val, comps = eng.scan_content((1.0, 1.0, 1.0, 0.0))
    assert val[1] == 85.0 and val[2] == 0.0 and comps[3][1] == 255.0
    c = eng.scan_hist_correl(256)
    assert abs(c[1] - (-1.0 / 255.0)) < 1e-12 and c[2] == 1.0
    avg = eng.scan_average()
    assert avg[1] == 255.0 and avg[0] == 0.0 and avg[3] == 85.0
    eng.close()
    # (3) shards + halo == serial, (4) idempotence, on a synthetic device-resident sequence
    n = 96
    plan = ScenePlan(n, seed=4, min_len=8, max_len=20)
    buf = DeviceBuffer(n * fb)
    synth_frames_device(buf.ptr, plan.params, w, h)
    serial = Engine(w, h, feats, max_batch=128)
    serial.submit_device(buf.ptr, n)
    want = (serial.read_sums().tobytes(), serial.read_yhist().tobytes())
    serial.reset()
    serial.submit_device(buf.ptr, n)
    assert (serial.read_sums().tobytes(), serial.read_yhist().tobytes()) == want
    serial.close()
    parts_s, parts_h = [], []
    for a, b in ((0, 31), (31, 64), (64, 96)):
        e = Engine(w, h, feats, max_batch=16)
        if a:
            e.set_halo_device(buf.ptr + (a - 1) * fb)
        e.submit_device(buf.ptr + a * fb, b - a)
        parts_s.append(e.read_sums())
        parts_h.append(e.read_yhist())
        e.close()
    assert np.concatenate(parts_s).tobytes() == want[0]
    assert np.concatenate(parts_h).tobytes() == want[1]
    buf.close()


class _PlainStream:
    """VideoStream-shaped source WITHOUT read_batch: exercises the pinned double-buffer path."""

    def __init__(self, frames, fps=30.0):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._s = ArrayVideoStream(frames, fps)

    frame_size = property(lambda self: self._s.frame_size)
    frame_rate = property(lambda self: self._s.frame_rate)
    position = property(lambda self: self._s.position)
    frame_number = property(lambda self: self._s.frame_number)

    def read(self, decode=True):
        return self._s.read(decode)


def test_scene_manager_plain_stream_crop_and_empty(lib):
    """Frame-by-frame streams (pinned staging), a crop region (strided view -> packed copy) and an
    empty stream, against the oracle."""
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.detectors import ContentDetector, ThresholdDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    case = get_case("content_default_stats")
    frames = case_frames(case)
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=16)
    sm.auto_downscale = False
    sm.add_detector(ContentDetector())
    sm.add_detector(ThresholdDetector())     # two detectors share one fused pass
    assert sm.detect_scenes(_PlainStream(frames)) == frames.shape[0]
    ref = R.RefContentDetector(with_stats=True)
    want = R.run_detector(ref, frames)
    rthr = R.RefThresholdDetector()
    want = sorted(set(want) | set(R.run_detector(rthr, frames)))
    assert [c.frame_num for c in sm.get_cut_list()] == want
    # crop
    sm2 = SceneManager(batch_size=8)
    sm2.auto_downscale = False
    sm2.crop = (143, 10, 16, 81)     # inclusive corners in any order (scene_manager.py:293-306): x 16..143, y 10..81
    sm2.add_detector(ContentDetector())
    sm2.detect_scenes(_PlainStream(frames))
    cropped = np.ascontiguousarray(frames[:, 10:82, 16:144])
    assert [c.frame_num for c in sm2.get_cut_list()] == R.run_detector(R.RefContentDetector(), cropped)
    # empty
    sm3 = SceneManager()
    sm3.add_detector(ContentDetector())
    assert sm3.detect_scenes(_PlainStream(frames[:0])) == 0
    assert sm3.get_cut_list() == [] and sm3.get_scene_list() == []


@pytest.mark.parametrize("name", case_names())
def test_device_cut_state_machines_match_golden(lib, name):
    """SURVEY §8(f) N2: scans + cut automata entirely on the device give the reference's cut list."""
    from pyscenedetect_b200.device_cuts import DeviceCuts
    from pyscenedetect_b200.engine import F_BGRSUM, F_EDGES, F_HSV, F_YHIST, Engine
    case = get_case(name)
    frames = case_frames(case)
    kw = dict(case["kw"])
    det = case["det"]
    weights = tuple(kw.get("weights", (1.0, 1.0, 1.0, 0.0)))
    if kw.get("luma_only"):
        weights = (0.0, 0.0, 1.0, 0.0)
    feats = {"content": F_HSV, "adaptive": F_HSV, "threshold": F_BGRSUM, "histogram": F_YHIST, "hash": 16}[det]
    if det in ("content", "adaptive") and weights[3] > 0.0:
        feats |= F_EDGES
    size = _scored_size(case) or (frames.shape[2], frames.shape[1])
    eng = Engine(frames.shape[2], frames.shape[1], feats, width=size[0], height=size[1], max_batch=64,
                 edge_kernel_size=kw.get("kernel_size") or 0, hash_size=kw.get("size", 8),
                 hash_lowpass=kw.get("lowpass", 2))
    eng.submit(frames)
    dc = DeviceCuts(eng)
    fps = case["fps"]
    msl = kw.get("min_scene_len", 15)
    if det == "content":
        cuts = dc.content(weights, kw.get("threshold", 27.0), msl, fps, suppress=kw.get("filter_mode") == "SUPPRESS")
    elif det == "adaptive":
        cuts = dc.adaptive(weights, kw.get("adaptive_threshold", 3.0), msl, kw.get("window_width", 2),
                           kw.get("min_content_val", 15.0), fps)
    elif det == "histogram":
        cuts = dc.histogram(kw.get("threshold", 0.20), kw.get("bins", 128), msl, fps)
    elif det == "hash":
        cuts = dc.hash(kw.get("threshold", 0.35), msl, fps)
    else:
        cuts = dc.threshold(kw.get("threshold", 12), msl, kw.get("fade_bias", 0.0), kw.get("add_final_scene", False),
                            kw.get("method") == "CEILING", fps)
    assert sorted(set(cuts)) == case["cuts"]
    eng.close()


@pytest.mark.parametrize("name", case_names())
def test_gathered_results_device_automata_match_golden(lib, name):
    """The rank-0 tail of sharding.detect_sharded: integer results uploaded as one array
    (`GatheredResults`), then scans + cut automata on the device with the DETECTOR OBJECT's own parameters
    (`cuts_for_detector`) - no per-frame Python."""
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import F_YHIST, Engine
    from pyscenedetect_b200.sharding import GatheredResults
    case = get_case(name)
    frames = case_frames(case)
    det = _build(case)
    size = _scored_size(case) or (frames.shape[2], frames.shape[1])
    eng = Engine(frames.shape[2], frames.shape[1], det.required_features(), width=size[0], height=size[1],
                 max_batch=64, edge_kernel_size=det.edge_kernel_size_arg(), **det.engine_kwargs())
    eng.submit(frames)
    sums = eng.read_sums()
    hist = eng.read_yhist() if det.required_features() & F_YHIST else None
    hashes = eng.read_hash() if det.required_features() & 16 else None
    eng.close()
    res = GatheredResults(sums, hist, size[0] * size[1], hashes=hashes, **det.engine_kwargs())
    assert sorted(set(cuts_for_detector(DeviceCuts(res), det, case["fps"]))) == case["cuts"]


def test_independent_engines_in_threads(lib):
    """SURVEY §8b threading contract: engines are single-producer but independent engines may run
    concurrently (benchmark sweeps use one SceneManager per thread)."""
    import threading

    from pyscenedetect_b200.engine import F_BGRSUM, F_HSV, F_YHIST, Engine
    rng = np.random.default_rng(11)
    data = [rng.integers(0, 256, size=(24, 90, 160, 3), dtype=np.uint8) for _ in range(4)]
    feats = F_HSV | F_BGRSUM | F_YHIST
    want = []
    for d in data:
        e = Engine(160, 90, feats)
        e.submit(d)
        want.append((e.read_sums().tobytes(), e.read_yhist().tobytes()))
        e.close()
    got = [None] * 4
    errors = []

    def work(i):
        try:
            for _ in range(5):
                e = Engine(160, 90, feats, max_batch=8)
                for j in range(0, 24, 5):
                    e.submit(data[i][j:j + 5])
                got[i] = (e.read_sums().tobytes(), e.read_yhist().tobytes())
                e.close()
        except Exception as exc:  # pragma: no cover
            errors.append(exc)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert got == want
