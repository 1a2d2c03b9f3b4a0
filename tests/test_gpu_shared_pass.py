"""Detectors that disagree on the dilation kernel size or the hash geometry in one SceneManager, one engine and one
sweep: the reference's own SceneManager on such mixes (tests/golden/shared_pass_v1.json, recorded by
tests/golden/make_shared_pass_golden.py), each detector's device automaton over the slots it is attached to, every
slot of a many-slot engine against a one-slot engine on the same frames, the launches that stay shared, and
ParameterSweep.run with one engine for several pixel groups."""

import ctypes as C
import json
import os

import numpy as np
import pytest

from tests.golden_util import case_frames
from tests.test_gpu_parity import _check_stats

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shared_pass_v1.json")
ALL = (1.0, 1.0, 1.0, 1.0)


def _cases() -> list:
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _detector(name, kw):
    from tests.test_gpu_parity import _build
    return _build({"det": name, "kw": kw})


def _frames(n, w, h, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    return render_frames(ScenePlan(n, seed=seed, min_len=6, max_len=20).params, w, h)


@pytest.mark.parametrize("batch", [7, 64])
@pytest.mark.parametrize("name", [c["name"] for c in _cases()])
def test_shared_pass_scene_manager_attaches_views_and_matches_reference(name, batch):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.engine import SlotView
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    case = next(c for c in _cases() if c["name"] == name)
    frames = case_frames(case)
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=batch)
    for det, kw in case["dets"]:
        sm.add_detector(_detector(det, kw))
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case.get("downscale", 1)
    assert sm.detect_scenes(ArrayVideoStream(frames, case["fps"])) == frames.shape[0]
    # more than one kernel size or hash geometry really is in the one engine
    assert any(isinstance(d._engine, SlotView) for d in sm._detector_list)
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    _check_stats(case, stats, frames.shape[0])


@pytest.mark.parametrize("name", [c["name"] for c in _cases()])
def test_device_cuts_read_each_detectors_slots(name):
    """`cuts_for_detector` over the shared engine of a SceneManager runs each detector's automaton over the slots
    the detector is attached to: the cuts of a one-slot engine that scored the same frames for that detector
    alone.  The cases hold non-zero edge slots (the first two) and non-zero hash slots (the last two)."""
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import SlotView
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.sweep import pixel_group_of
    from pyscenedetect_b200.video import ArrayVideoStream
    case = next(c for c in _cases() if c["name"] == name)
    frames, fps = case_frames(case), case["fps"]
    sm = SceneManager(StatsManager())   # the StatsManager turns the edge component on for every content detector
    for det, kw in case["dets"]:
        sm.add_detector(_detector(det, kw))
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case.get("downscale", 1)
    sm.detect_scenes(ArrayVideoStream(frames, fps))
    assert any(isinstance(d._engine, SlotView) for d in sm._detector_list)
    _, (w, h), (sw, sh) = sm._geometry(frames.shape[2], frames.shape[1])
    dc = DeviceCuts(sm._engine)
    for d, (det, kw) in zip(sm._detector_list, case["dets"]):
        alone = pixel_group_of(d).make_engine(w, h, sw, sh)   # d's own kernel size and hash geometry in slot 0
        alone.submit(frames)
        want = cuts_for_detector(DeviceCuts(alone), _detector(det, kw), fps)
        alone.close()
        assert cuts_for_detector(dc, d, fps) == want, (det, kw)


KS = (3, 5, 17, 19, 63)
GEOS = ((8, 2), (16, 2), (8, 3), (64, 2))   # (64, 2): a 128x128 hash image, whose finish runs from global memory


def _edge_sads(holder):
    """stream frames' sad_edges of a holder's edge slot, on the host"""
    from pyscenedetect_b200 import _capi
    p = holder.device_edge_sads()
    if p is None:
        return holder.read_sums()["sad_edges"].copy()
    out = np.zeros(holder.frame_count, dtype=np.uint64)
    holder.sync()
    assert _capi.load().psd_memcpy_d2h(holder.device, out.ctypes.data, p, out.nbytes) == 0
    return out


def _snapshot(edges, hashes):
    """{kernel size: holder}, {geometry: holder} -> every slot's results through the holders' slot-free accessors"""
    res = {}
    for k, e in edges.items():
        val, comps = e.scan_content(ALL)
        res[("edges", k)] = (_edge_sads(e).tobytes(), val.tobytes(), comps.tobytes())
    for g, e in hashes.items():
        res[("hash", g)] = (e.read_hash().tobytes(), e.scan_hash_dist().tobytes())
    return res


def _slot(holder, which):
    from pyscenedetect_b200.engine import SlotView
    return getattr(holder, which) if isinstance(holder, SlotView) else 0


def _feed(eng, frames, dev_buf, halo):
    """halo frame, host submits that do not line up with max_batch, then a device submit of the rest"""
    eng.set_halo(halo)
    eng.submit(frames[:13])
    eng.submit(frames[13:14])
    eng.submit(frames[14:40])
    dev_buf.upload(frames[40:])
    eng.submit_device(dev_buf.ptr, frames.shape[0] - 40)


def test_every_slot_holder_equals_a_one_slot_engine():
    from pyscenedetect_b200.engine import F_EDGES, F_HASH, F_HSV, DeviceBuffer, Engine
    from pyscenedetect_b200.scene_manager import shared_engine
    from pyscenedetect_b200.sweep import PixelGroup
    w, h = 320, 180
    video = _frames(71, w, h, 5)
    second = _frames(30, w, h, 6)
    buf = DeviceBuffer(video.nbytes)
    groups = [PixelGroup(F_HSV | F_EDGES, k, ()) for k in KS] + \
        [PixelGroup(F_HASH, 0, (("hash_lowpass", lp), ("hash_size", s))) for s, lp in GEOS]
    multi, holders = shared_engine(groups, w, h, w, h, max_batch=8)
    edges = dict(zip(KS, holders[:len(KS)]))
    hashes = dict(zip(GEOS, holders[len(KS):]))
    assert [_slot(e, "edge_slot") for e in edges.values()] == list(range(len(KS)))
    assert [_slot(e, "hash_slot") for e in hashes.values()] == list(range(len(GEOS)))
    assert [multi.edge_kernel_size_at(s) for s in range(len(KS))] == list(KS) and multi.edge_kernel_size_at(9) == -1
    _feed(multi, video[1:], buf, video[0])
    got = _snapshot(edges, hashes)
    # the engine's own slot keywords give what the holders give
    for s, k in enumerate(KS):
        assert multi.scan_content(ALL, edge_slot=s)[0].tobytes() == got[("edges", k)][1], k
    for s, g in enumerate(GEOS):
        assert multi.read_hash(hash_slot=s).tobytes() == got[("hash", g)][0], g
        assert multi.scan_hash_dist(hash_slot=s).tobytes() == got[("hash", g)][1], g
    multi.reset()
    multi.submit(second)
    got2 = _snapshot(edges, hashes)
    multi.close()
    for k in KS:
        one = Engine(w, h, F_HSV | F_EDGES, max_batch=8, edge_kernel_size=k)
        _feed(one, video[1:], buf, video[0])
        assert _snapshot({k: one}, {}) == {key: v for key, v in got.items() if key == ("edges", k)}, k
        one.reset()
        one.submit(second)
        assert _snapshot({k: one}, {})[("edges", k)] == got2[("edges", k)], k
        one.close()
    for g in GEOS:
        one = Engine(w, h, F_HASH, max_batch=8, hash_size=g[0], hash_lowpass=g[1])
        _feed(one, video[1:], buf, video[0])
        assert _snapshot({}, {g: one})[("hash", g)] == got[("hash", g)], g
        one.reset()
        one.submit(second)
        assert _snapshot({}, {g: one})[("hash", g)] == got2[("hash", g)], g
        one.close()
    # the slots saw real edges and hashes
    assert all(np.frombuffer(got[("edges", k)][0], np.uint64).any() for k in KS)


def _launches(eng, frames):
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    eng.sync()
    c0 = lib.psd_launch_count()
    eng.submit(frames)
    eng.sync()
    return lib.psd_launch_count() - c0


def test_canny_and_the_gray_pass_run_once_per_batch():
    from pyscenedetect_b200.engine import F_EDGES, F_HASH, F_HSV, Engine
    w, h = 320, 180
    frames = _frames(16, w, h, 7)
    one = Engine(w, h, F_HSV | F_EDGES, max_batch=16, edge_kernel_size=3)
    many = Engine(w, h, F_HSV | F_EDGES, max_batch=16, edge_kernel_size=3)
    for k in KS[1:]:
        many.add_edge_kernel_size(k)
    # per extra slot: its dilation (two passes for k >= 19) and its SAD, nothing else
    extra = sum(3 if k >= 19 else 2 for k in KS[1:])
    for _ in range(2):   # the first batch has no predecessor, the second one does
        assert _launches(many, frames) - _launches(one, frames) == extra
    one.close()
    many.close()
    one = Engine(w, h, F_HASH, max_batch=16)
    many = Engine(w, h, F_HASH, max_batch=16)
    for s, lp in GEOS[1:]:
        many.add_hash_geometry(s, lp)
    # one rows launch (the gray pass) for every geometry, then one finish launch per geometry
    assert _launches(one, frames) == 2
    assert _launches(many, frames) == 1 + len(GEOS)
    one.close()
    many.close()


def test_slots_are_added_before_the_first_frame_only():
    from pyscenedetect_b200.engine import F_EDGES, F_HASH, F_HSV, Engine
    w, h = 160, 90
    frames = _frames(4, w, h, 8)
    eng = Engine(w, h, F_HSV | F_EDGES | F_HASH, max_batch=4, edge_kernel_size=3)
    assert eng.add_edge_kernel_size(0) == 1            # automatic at 160x90: 5
    assert eng.add_edge_kernel_size(5) == 1            # the same effective size
    assert eng.add_edge_kernel_size(3) == 0
    assert eng.add_hash_geometry(8, 2) == 0 and eng.add_hash_geometry(16, 2) == 1
    with pytest.raises(ValueError):
        eng.add_edge_kernel_size(4)
    eng.submit(frames)
    with pytest.raises(RuntimeError):
        eng.add_edge_kernel_size(7)
    with pytest.raises(RuntimeError):
        eng.add_hash_geometry(4, 2)
    eng.reset()
    assert eng.add_edge_kernel_size(7) == 2
    eng.set_halo(frames[0])
    with pytest.raises(RuntimeError):
        eng.add_edge_kernel_size(9)
    eng.close()
    plain = Engine(w, h, F_HSV, max_batch=4)
    with pytest.raises(ValueError):
        plain.add_edge_kernel_size(5)
    with pytest.raises(ValueError):
        plain.add_hash_geometry(16, 2)
    plain.close()


def _scene_manager_pred(det, frames, fps):
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    sm = SceneManager()
    sm.add_detector(det)
    sm.detect_scenes(ArrayVideoStream(frames, fps))
    return [s[1].frame_num for s in sm.get_scene_list()]


def test_sweep_scores_every_pixel_group_with_one_engine(monkeypatch):
    from pyscenedetect_b200 import scene_manager as sm_mod
    from pyscenedetect_b200.detectors import ContentDetector, HashDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream
    built = []

    class CountingEngine(sm_mod.Engine):
        def __init__(self, *a, **kw):
            built.append(kw)
            super().__init__(*a, **kw)

    monkeypatch.setattr(sm_mod, "Engine", CountingEngine)
    frames = render_frames(ScenePlan(240, seed=12, noise_shift=30, min_len=15, max_len=60).params, 320, 180)
    for cls, grid in (
            (ContentDetector, [dict(weights=ALL, kernel_size=k, threshold=t, min_scene_len=m)
                               for k in (3, 5) for t in (20.0, 30.0) for m in (0, 10)] + [dict(threshold=20.0)]),
            (HashDetector, [dict(size=s, threshold=t, min_scene_len=m) for s in (8, 16) for t in (0.2, 0.35)
                            for m in (0, 10)])):
        sw = ParameterSweep(cls, grid, batch_size=50)
        assert len(sw.groups) == (3 if cls is ContentDetector else 2)
        built.clear()
        r = sw.run(ArrayVideoStream(frames, 30.0))
        assert len(built) == 1
        for k, kw in enumerate(grid):
            assert r.cuts(k) == _scene_manager_pred(cls(**kw), frames, 30.0), kw
