"""ContentDetector and AdaptiveDetector on the GPU with edge kernel sizes of 65 and above (the separable bit-plane
dilation): every dilated map and edge SAD against cv2.dilate, batching and halo shards, and the cases recorded from
the reference (tests/golden/kernel_sizes_v1.json) through SceneManager, DeviceCuts and ParameterSweep."""

import hashlib
import io
import json
import os

import cv2
import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from pyscenedetect_b200.synth import ScenePlan, render_frames

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kernel_sizes_v1.json")
BIG = (15360, 8640)   # the automatic kernel size is 65 from this frame size on


def golden() -> dict:
    with open(GOLDEN) as f:
        return json.load(f)


def case_names() -> list[str]:
    return [c["name"] for c in golden()["cases"]]


def get_case(name: str) -> dict:
    return next(c for c in golden()["cases"] if c["name"] == name)


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


def _plan(gen):
    n, w, h, seed, mn, mx, ns = gen
    return ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)


def _frames(gen) -> np.ndarray:
    """A recorded case's frames; the 15360x8640 ones are rendered on the device and downloaded."""
    plan = _plan(gen)
    w, h = gen[1], gen[2]
    if (w, h) != BIG:
        return render_frames(plan.params, w, h)
    from pyscenedetect_b200.engine import DeviceBuffer, synth_frames_device
    nbytes = len(plan.params) * w * h * 3
    buf = DeviceBuffer(nbytes)
    synth_frames_device(buf.ptr, plan.params, w, h)
    frames = buf.download(nbytes).reshape(len(plan.params), h, w, 3)
    buf.close()
    return frames


def _check_dilation(w, h, k, frames, sub=4):
    """Sub-batches of `sub` frames (the carry plane holds the predecessor across them): the dilated map of every
    frame equals cv2.dilate(cv2.Canny(V)) and the edge SAD the oracle's."""
    from pyscenedetect_b200.engine import F_EDGES, Engine
    eng = Engine(w, h, F_EDGES, max_batch=sub, edge_kernel_size=k)
    assert eng.edge_kernel_size == k
    kernel = np.ones((k, k), np.uint8)
    prev = None
    for b in range(0, len(frames), sub):
        eng.submit(frames[b:b + sub])
        sums = eng.read_sums(b, min(sub, len(frames) - b))
        for j, f in enumerate(frames[b:b + sub]):
            lum = cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2]
            want = R.detect_edges(lum, kernel)
            assert np.array_equal(eng.debug_plane(3, j), want), (w, h, k, b + j)
            if prev is not None:
                assert int(sums["sad_edges"][j]) == M.sad(want, prev), (w, h, k, b + j)
            prev = want
    eng.close()


def _small_frames(w, h):
    frames = render_frames(ScenePlan(10, seed=6, min_len=3, max_len=5).params, w, h)
    rng = np.random.default_rng(w * h)
    sparse = np.full((h, w, 3), 128, np.uint8)
    ys, xs = rng.integers(0, h, 3), rng.integers(0, w, 3)
    sparse[ys, xs] = 255   # a few isolated edge pixels: every window boundary shows
    extra = np.stack([np.zeros((h, w, 3), np.uint8), sparse, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)])
    return np.concatenate([frames[:5], extra, frames[5:]])


@pytest.mark.parametrize("k", [65, 67, 95, 127, 129, 255, 257, 1023])
@pytest.mark.parametrize("shape", [(200, 90), (131, 97)])
def test_dilated_maps_match_cv2(lib, shape, k):
    w, h = shape
    _check_dilation(w, h, k, _small_frames(w, h))


@pytest.mark.parametrize("k", [65, 255])
def test_dilated_maps_match_cv2_1080p(lib, k):
    frames = render_frames(ScenePlan(6, seed=9, min_len=2, max_len=3).params, 1920, 1080)
    _check_dilation(1920, 1080, k, frames, sub=4)


def test_kernel_above_twice_the_frame_saturates(lib):
    w, h = 131, 97
    k = 2 * max(w, h) + 39   # every output pixel's window covers the whole frame
    frames = _small_frames(w, h)
    _check_dilation(w, h, k, frames)
    from pyscenedetect_b200.engine import F_EDGES, Engine
    eng = Engine(w, h, F_EDGES, max_batch=16, edge_kernel_size=k)
    eng.submit(frames)
    for j in range(len(frames)):
        plane = eng.debug_plane(3, j)
        assert plane.min() == plane.max(), j   # all 0 or all 255
    eng.close()


def test_automatic_size_at_15360x8640_is_65(lib):
    from pyscenedetect_b200.engine import F_EDGES, Engine
    assert R.estimated_kernel_size(*BIG) == 65
    eng = Engine(BIG[0], BIG[1], F_EDGES, max_batch=2)
    assert eng.edge_kernel_size == 65
    eng.close()


def test_batching_and_halo_shards_equal_serial(lib):
    from pyscenedetect_b200.engine import F_EDGES, Engine
    frames = render_frames(ScenePlan(40, seed=31, min_len=3, max_len=9).params, 320, 180)
    outs = []
    for mb in (1, 7, 64):
        eng = Engine(320, 180, F_EDGES, max_batch=mb, edge_kernel_size=129)
        for i in range(0, len(frames), mb):
            eng.submit(frames[i:i + mb])
        outs.append(eng.read_sums())
        eng.close()
    for s in outs[1:]:
        assert np.array_equal(s["sad_edges"], outs[0]["sad_edges"])
    serial = outs[0]
    assert serial["sad_edges"][1:].any()
    bounds = [0, 13, 29, 40]
    for a, b in zip(bounds[:-1], bounds[1:]):
        eng = Engine(320, 180, F_EDGES, max_batch=16, edge_kernel_size=129)
        if a > 0:
            eng.set_halo(frames[a - 1])
        eng.submit(frames[a:b])
        got = eng.read_sums()
        eng.close()
        assert np.array_equal(got, serial[a:b]), (a, b)


def _detector(case):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    kw = dict(case["kw"])
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    return {"content": ContentDetector, "adaptive": AdaptiveDetector}[case["det"]](**kw)


@pytest.mark.parametrize("batch", [7, 64])
@pytest.mark.parametrize("name", case_names())
def test_recorded_cases_through_scene_manager(lib, name, batch):
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    case = get_case(name)
    frames = _frames(case["gen"])
    assert hashlib.sha256(frames.tobytes()).hexdigest() == case["frames_sha256"]
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=batch)
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case.get("downscale", 1)
    sm.add_detector(_detector(case))
    sm.detect_scenes(ArrayVideoStream(frames, case["fps"]))
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    keys = case["metric_keys"]
    for t in range(len(frames)):
        got = stats.get_metrics(FrameTimecode(t, case["fps"]), keys)
        want = case["metrics"].get(str(t))
        got_hex = [None if v is None else float(v).hex() for v in got]
        if want is None:
            assert all(v is None for v in got_hex), (t, got_hex)
        else:
            assert got_hex == want, (t, keys, got_hex, want)
    buf = io.StringIO()
    stats.save_to_csv(buf)
    assert hashlib.sha256(buf.getvalue().encode()).hexdigest() == case["csv_sha256"]


def _scored_frames(case, frames):
    if not case.get("auto_downscale"):
        return frames
    f = R.compute_downscale_factor(case["gen"][1])
    return np.stack([R.downscale_frame(x, f) for x in frames])


@pytest.mark.parametrize("name", [n for n in case_names() if "15360" not in n])
def test_recorded_cases_device_cuts(lib, name):
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import Engine
    case = get_case(name)
    frames = _scored_frames(case, _frames(case["gen"]))
    det = _detector(case)
    h, w = frames.shape[1:3]
    eng = Engine(w, h, det.required_features(), max_batch=16, edge_kernel_size=det.edge_kernel_size_arg())
    assert eng.edge_kernel_size == case["kw"]["kernel_size"]
    eng.submit(frames)
    assert sorted(set(cuts_for_detector(DeviceCuts(eng), det, case["fps"]))) == case["cuts"]
    eng.close()


def test_parameter_sweep_over_recorded_grid(lib):
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    g = golden()["grid"]
    frames = render_frames(_plan(g["gen"]).params, g["gen"][1], g["gen"][2])
    cells = [dict(c["kw"], weights=tuple(c["kw"]["weights"])) for c in g["cells"]]
    sw = ParameterSweep(ContentDetector, cells, batch_size=48)
    assert len(sw.groups) == 3   # one score pass per kernel size
    r = sw.run(ArrayVideoStream(frames, g["fps"]))
    for k, cell in enumerate(g["cells"]):
        assert r.cuts(k) == [b for _a, b in cell["scene_list"]], cell["kw"]
