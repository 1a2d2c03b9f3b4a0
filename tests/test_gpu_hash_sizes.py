"""HashDetector on the GPU for hashes larger than 16x16 and hash images larger than 64x64: every hash bit against
the reference's cv2 call sequence, the hash_dist scan, batching and halo shards, and the cases recorded from the
reference (tests/golden/hash_sizes_v1.json) through SceneManager, DeviceCuts, GatheredResults and ParameterSweep."""

import hashlib
import io

import numpy as np
import pytest

from oracle import ref_detectors as R
from pyscenedetect_b200.synth import ScenePlan, render_frames
from tests.hash_sizes_util import case_names, check_recorded_dist, get_case, golden, near_median

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


def _frames(gen):
    n, w, h, seed, mn, mx, ns = gen
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    return plan, render_frames(plan.params, w, h)


def _bits(words: np.ndarray, m: int) -> np.ndarray:
    """(words,) uint64 row -> m bools, bit k = word k // 64, bit k % 64."""
    b = np.unpackbits(words.astype("<u8").view(np.uint8), bitorder="little")
    assert not b[m:].any(), "bits past size * size must be 0"
    return b[:m].astype(bool)


# (frame w, h, size, lowpass): the recorded cases' scored sizes, plus 4K at n = 256
SHAPES = [((274, 154), 32, 3), ((640, 360), 17, 1), ((1280, 720), 24, 4), ((640, 360), 64, 2),
          ((480, 270), 256, 1), ((1920, 1080), 100, 10), ((1920, 1080), 30, 36), ((3840, 2160), 32, 8)]


@pytest.mark.parametrize("shape,size,lowpass", SHAPES)
def test_hash_bits_match_cv2(lib, shape, size, lowpass):
    from pyscenedetect_b200._capi import hash_words
    from pyscenedetect_b200.engine import F_HASH, Engine
    w, h = shape
    n_img = size * lowpass
    count = 3 if w * h > 1000000 else 10
    _, scene = _frames((count, w, h, w + size, 1, 3, 30))
    rng = np.random.default_rng(w + size)
    extra = [np.zeros((h, w, 3), np.uint8), rng.integers(0, 256, (h, w, 3), dtype=np.uint8)]
    if n_img & (n_img - 1) == 0:
        extra += [np.full((h, w, 3), 255, np.uint8), np.full((h, w, 3), 37, np.uint8)]
    frames = np.concatenate([scene, np.stack(extra)])
    eng = Engine(w, h, F_HASH, max_batch=8, hash_size=size, hash_lowpass=lowpass)
    eng.submit(frames)
    got = eng.read_hash()
    dist = eng.scan_hash_dist()
    eng.close()
    m = size * size
    assert got.shape == (len(frames), hash_words(size))
    tolerated = [0, 0]   # bits that differ from cv2 within rounding of the median: ScenePlan, other frames
    prev = None
    for i, f in enumerate(frames):
        want = R.hash_frame(f, size, lowpass).ravel()
        bits = _bits(got[i], m)
        diff = bits != want
        if diff.any():
            near, bound = near_median(f, size, lowpass)
            assert not (diff & ~near).any(), (i, int(diff.sum()), int((diff & ~near).sum()), bound)
            tolerated[i >= len(scene)] += int(diff.sum())
        if prev is None:
            assert np.isnan(dist[i])
        else:
            assert dist[i] == np.count_nonzero(bits != prev) / float(m)
        prev = bits
    print(f"{w}x{h} size {size} lowpass {lowpass}: bits within rounding of the median that differ from cv2: "
          f"{tolerated[0]} on {len(scene)} ScenePlan frames, {tolerated[1]} on {len(extra)} black/noise/solid frames")


def test_batching_and_halo_shards_equal_serial(lib):
    from pyscenedetect_b200.engine import F_HASH, Engine
    _, frames = _frames((40, 320, 180, 31, 3, 9, 30))
    outs = []
    for mb in (1, 7, 64):
        eng = Engine(320, 180, F_HASH, max_batch=mb, hash_size=32, hash_lowpass=3)
        for i in range(0, len(frames), mb):
            eng.submit(frames[i:i + mb])
        outs.append((eng.read_hash(), eng.scan_hash_dist()))
        eng.close()
    for hsh, dist in outs[1:]:
        assert np.array_equal(hsh, outs[0][0])
        assert np.array_equal(dist, outs[0][1], equal_nan=True)
    serial_hash, serial_dist = outs[0]
    bounds = [0, 13, 29, 40]
    for a, b in zip(bounds[:-1], bounds[1:]):
        eng = Engine(320, 180, F_HASH, max_batch=16, hash_size=32, hash_lowpass=3)
        if a > 0:
            eng.set_halo(frames[a - 1])
        eng.submit(frames[a:b])
        assert np.array_equal(eng.read_hash(), serial_hash[a:b])
        got = eng.scan_hash_dist()
        eng.close()
        if a == 0:
            assert np.isnan(got[0]) and np.array_equal(got[1:], serial_dist[1:b])
        else:
            assert np.array_equal(got, serial_dist[a:b])


def test_small_sizes_keep_four_words_and_small_frames_raise(lib):
    from pyscenedetect_b200.engine import F_HASH, Engine
    _, frames = _frames((4, 160, 90, 3, 1, 3, 30))
    for size, lowpass in ((8, 2), (16, 4), (1, 1)):
        eng = Engine(160, 90, F_HASH, max_batch=4, hash_size=size, hash_lowpass=lowpass)
        eng.submit(frames)
        assert eng.read_hash().shape == (4, 4)
        eng.close()
    with pytest.raises(ValueError, match="smaller than the 96x96 hash image"):
        Engine(160, 90, F_HASH, hash_size=32, hash_lowpass=3)


def _scored(case):
    w, h = case["gen"][1:3]
    if case.get("auto_downscale"):
        return R.downscaled_size(w, h, R.compute_downscale_factor(max(w, h)))
    return (w, h)


def _scored_frames(case, frames):
    """The frames at the size the detector scores (SceneManager's cv2 INTER_LINEAR downscale)."""
    if not case.get("auto_downscale"):
        return frames
    f = R.compute_downscale_factor(case["gen"][1])
    return np.stack([R.downscale_frame(x, f) for x in frames])


@pytest.mark.parametrize("name", case_names())
def test_recorded_cases_through_scene_manager(lib, name):
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    case = get_case(name)
    _, frames = _frames(case["gen"])
    assert hashlib.sha256(frames.tobytes()).hexdigest() == case["frames_sha256"]
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=16)
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case.get("downscale", 1)
    sm.add_detector(HashDetector(**case["kw"]))
    sm.detect_scenes(ArrayVideoStream(frames, case["fps"]))
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    key = HashDetector(**case["kw"]).get_metrics()[0]
    got = {t: stats.get_metrics(FrameTimecode(t, case["fps"]), [key])[0] for t in range(len(frames))}
    differ = check_recorded_dist({t: float(v) for t, v in got.items() if v is not None}, case,
                                 _scored_frames(case, frames))
    buf = io.StringIO()
    stats.save_to_csv(buf)
    if differ == 0:   # the CSV is byte-identical whenever every metric is
        assert buf.getvalue().splitlines()[:4] == case["csv_head"]
        assert hashlib.sha256(buf.getvalue().encode()).hexdigest() == case["csv_sha256"]
    print(f"{name}: {differ} frames' hash_dist differ from the recording within rounding of the median")


@pytest.mark.parametrize("name", case_names())
def test_recorded_cases_device_cuts_and_gathered(lib, name):
    from pyscenedetect_b200._capi import SUMS_DTYPE
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import F_HASH, Engine
    from pyscenedetect_b200.sharding import GatheredResults
    case = get_case(name)
    _, frames = _frames(case["gen"])
    det = HashDetector(**case["kw"])
    sw, sh = _scored(case)
    eng = Engine(frames.shape[2], frames.shape[1], F_HASH, width=sw, height=sh, max_batch=16, **det.engine_kwargs())
    eng.submit(frames)
    dist = eng.scan_hash_dist()
    check_recorded_dist({t: float(d) for t, d in enumerate(dist) if not np.isnan(d)}, case, _scored_frames(case, frames))
    assert sorted(set(cuts_for_detector(DeviceCuts(eng), det, case["fps"]))) == case["cuts"]
    hashes = eng.read_hash()
    eng.close()
    res = GatheredResults(np.zeros(len(frames), dtype=SUMS_DTYPE), None, sw * sh, hashes=hashes, **det.engine_kwargs())
    assert sorted(set(cuts_for_detector(DeviceCuts(res), det, case["fps"]))) == case["cuts"]
    k = len(frames) // 2
    assert np.array_equal(res.scan_hash_dist(first=k), dist[k:])


def test_parameter_sweep_over_recorded_grid(lib):
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    g = golden()["grid"]
    _, frames = _frames(g["gen"])
    sw = ParameterSweep(HashDetector, [c["kw"] for c in g["cells"]], batch_size=48)
    assert len(sw.groups) == 3
    r = sw.run(ArrayVideoStream(frames, g["fps"]))
    for k, cell in enumerate(g["cells"]):
        assert r.cuts(k) == [b for _a, b in cell["scene_list"]], cell["kw"]
