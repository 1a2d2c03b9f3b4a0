"""The device downscale (psd_resize_kernel with engine.cu's taps) against cv2.resize(INTER_LINEAR) of the numpy BGR
frame, byte for byte, at every geometry where cv2's scale 1 / (dst / src) and src / dst give different taps (found by
the CPU search of tests/test_resize_taps.py), at common video sizes under auto-downscale and factors 2 … 8, at
15360x8640, at 1-pixel sides and on a frame whose scored height exceeds 65 535 rows (the kernel's row loop), from
every frame layout the engine reads.  Then the cases of tests/golden/downscale_v1.json, recorded from the
reference's SceneManager, through this package's SceneManager at batch 7 and 64."""

import hashlib
import io

import cv2
import numpy as np
import pytest
import torch

from oracle import ref_detectors as R
from tests.test_resize_taps import ENGINE_ONLY, TABLE, downscale_golden, split_pairs

pytestmark = pytest.mark.gpu

F_BGRSUM = 2


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


def _check(frames, dw, dh, submit=None, tag=""):
    """Engine(F_BGRSUM, width=dw, height=dh) on `frames` (n, sh, sw, 3) BGR; every scored frame equals cv2's."""
    from pyscenedetect_b200.engine import Engine
    n, sh, sw, _ = frames.shape
    eng = Engine(sw, sh, F_BGRSUM, width=dw, height=dh, max_batch=n)
    try:
        if submit is None:
            eng.submit(frames)
        else:
            submit(eng)
        for i in range(n):
            want = cv2.resize(frames[i], (dw, dh), interpolation=cv2.INTER_LINEAR)
            got = eng.debug_plane(0, i)
            assert got.shape == want.shape and np.array_equal(got, want), (tag, sw, sh, dw, dh, i)
        sums = eng.read_sums()
        for i in range(n):   # the fused pass scores what the resize wrote
            want = cv2.resize(frames[i], (dw, dh), interpolation=cv2.INTER_LINEAR)
            assert int(sums["bgr_sum"][i]) == int(want.astype(np.int64).sum()), (tag, sw, sh, dw, dh, i)
    finally:
        eng.close()


def _noise(n, w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def test_search_pairs_are_there(lib):
    assert set(TABLE) <= set(split_pairs())


@pytest.mark.parametrize("axis", ["x", "y"])
def test_scale_split_pairs_as_thin_frames(lib, axis):
    """Every pair the CPU search finds (75 at sides up to 32 768), along x on a 2-row frame and along y on its
    transpose, plus 7281 -> 4096, which only Engine(width=) reaches."""
    for k, (src, dst) in enumerate(split_pairs() + [ENGINE_ONLY]):
        if axis == "x":
            _check(_noise(2, src, 2, k), dst, 2, tag=axis)
        else:
            _check(_noise(2, 2, src, k), 2, dst, tag=axis)


@pytest.mark.parametrize("sw,sh,dw,dh", [(10241, 4, 5120, 2), (12287, 6, 6144, 3), (14335, 14, 2048, 2),
                                         (4, 10241, 2, 5120), (15360, 8, 7680, 4)])
def test_issue_table_geometries(lib, sw, sh, dw, dh):
    _check(_noise(3, sw, sh, sw + sh), dw, dh)


VIDEO_SIZES = [(426, 240), (640, 360), (854, 480), (1280, 720), (1920, 1080), (2560, 1440), (3840, 2160),
               (7680, 4320), (1080, 1920)]


@pytest.mark.parametrize("sw,sh", VIDEO_SIZES, ids=[f"{w}x{h}" for w, h in VIDEO_SIZES])
def test_video_sizes_auto_and_factors(lib, sw, sh):
    frames = _noise(2, sw, sh, sw * 3 + sh)
    f = R.compute_downscale_factor(max(sw, sh))
    sizes = [R.downscaled_size(sw, sh, f)] + [R.downscaled_size(sw, sh, k) for k in range(2, 9)]
    for dw, dh in sizes:
        _check(frames, dw, dh, tag="auto" if (dw, dh) == sizes[0] else "factor")


def test_15360x8640(lib):
    frames = _noise(1, 15360, 8640, 5)
    for dw, dh in [R.downscaled_size(15360, 8640, R.compute_downscale_factor(15360)), (7680, 4320), (5120, 2880)]:
        _check(frames, dw, dh)


@pytest.mark.parametrize("sw,sh,dw,dh", [(1, 1, 1, 1), (1, 257, 1, 128), (257, 1, 128, 1), (1, 4096, 1, 1),
                                         (4096, 1, 1, 1), (640, 360, 1, 144), (640, 360, 256, 1), (7, 5, 1, 1),
                                         (4095, 2, 2048, 1), (2, 4095, 1, 2048)])
def test_one_pixel_sides(lib, sw, sh, dw, dh):
    _check(_noise(3, sw, sh, sw * 5 + sh), dw, dh)


def test_scored_height_above_65535_rows(lib):
    """2 x 131 074 at downscale 2 scores 1 x 65 537 rows, 6 x 140 001 at downscale 2 scores 3 x 70 000 (round half
    to even): more rows than one grid dimension launches, so the kernel loops over them."""
    _check(_noise(2, 2, 131074, 1), 1, 65537)
    _check(_noise(2, 6, 140001, 2), 3, 70000)


def _layouts(frames):
    """name -> submit(engine) of `frames` (BGR) from CUDA memory in another layout."""
    n, h, w, _ = frames.shape
    rgb = np.ascontiguousarray(frames[..., ::-1])
    big = np.zeros((n, h + 3, w + 5, 3), dtype=np.uint8)
    big[:, 1:1 + h, 3:3 + w] = frames
    flat = torch.zeros(frames.size + 1, dtype=torch.uint8)
    flat[1:] = torch.from_numpy(frames.reshape(-1))
    flat = flat.cuda()
    one = torch.from_numpy(frames[:1]).cuda()
    return {
        "packed_bgr": lambda e: e.submit(torch.from_numpy(frames).cuda()),
        "packed_rgb": lambda e: e.submit(torch.from_numpy(rgb).cuda(), channel_order="rgb"),
        "nchw_bgr": lambda e: e.submit(torch.from_numpy(np.ascontiguousarray(frames.transpose(0, 3, 1, 2))).cuda()
                                       .permute(0, 2, 3, 1)),
        "nchw_rgb": lambda e: e.submit(torch.from_numpy(np.ascontiguousarray(rgb.transpose(0, 3, 1, 2))).cuda()
                                       .permute(0, 2, 3, 1), channel_order="rgb"),
        "crop_odd_offset": lambda e: e.submit(torch.from_numpy(big).cuda()[:, 1:1 + h, 3:3 + w]),
        "unaligned_base": lambda e: e.submit(torch.as_strided(flat, (n, h, w, 3), (h * w * 3, w * 3, 3, 1), 1)),
    }, one


@pytest.mark.parametrize("sw,sh,dw,dh", [(10241, 4, 5120, 2), (4, 10241, 2, 5120), (131, 97, 50, 37),
                                         (1920, 1080, 256, 144)])
def test_every_layout(lib, sw, sh, dw, dh):
    frames = _noise(3, sw, sh, sw * 7 + sh)
    subs, one = _layouts(frames)
    for name, submit in subs.items():
        _check(frames, dw, dh, submit=submit, tag=name)
    same = np.repeat(frames[:1], 3, axis=0)   # zero frame stride: one frame seen three times
    _check(same, dw, dh, submit=lambda e: e.submit(one.expand(3, sh, sw, 3)), tag="zero_frame_stride")


@pytest.mark.parametrize("batch", [7, 64])
@pytest.mark.parametrize("name", [c["name"] for c in downscale_golden()["cases"]])
def test_downscale_golden_through_scene_manager(lib, name, batch):
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream
    case = next(c for c in downscale_golden()["cases"] if c["name"] == name)
    n, w, h, seed, mn, mx, ns = case["gen"]
    frames = render_frames(ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx).params, w, h)
    assert hashlib.sha256(frames.tobytes()).hexdigest() == case["frames_sha256"]
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=batch)
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case["downscale"]
    if "crop" in case:
        sm.crop = tuple(case["crop"])
    sm.add_detector(ContentDetector(**case["kw"]))
    sm.detect_scenes(ArrayVideoStream(frames, case["fps"]))
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    keys = case["metric_keys"]
    for t in range(n):
        got = stats.get_metrics(FrameTimecode(t, case["fps"]), keys)
        got_hex = [None if v is None else float(v).hex() for v in got]
        want = case["metrics"].get(str(t))
        assert got_hex == (want if want is not None else [None] * len(keys)), (t, got_hex, want)
    buf = io.StringIO()
    stats.save_to_csv(buf)
    assert hashlib.sha256(buf.getvalue().encode()).hexdigest() == case["csv_sha256"]
