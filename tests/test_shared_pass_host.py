"""SceneManager's engine slots without a GPU: which kernel sizes and hash geometries the one engine is configured
and extended with, in which order, and which slot every detector is attached to.  The engine is the oracle-backed
stand-in of tests/fake_engine.py with slot bookkeeping on top."""

from ctypes import c_double as C_double
from ctypes import c_int32 as C_int32

import numpy as np
import pytest

from oracle import ref_detectors as R
from pyscenedetect_b200.engine import Engine, SlotView
from tests.fake_engine import OracleEngine

ALL = (1.0, 1.0, 1.0, 1.0)


class SlotEngine(OracleEngine):
    """The engine's slot contract: `add_*` returns the slot that already holds the effective kernel size or the
    geometry, else appends one."""
    made: list = []

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.config = (kw.get("edge_kernel_size", 0), kw.get("hash_size"), kw.get("hash_lowpass"))
        self._edge_sizes = [self._effective(self.config[0])]
        self._geometries = [(self.hash_size, self.hash_lowpass)]
        self.added_edges, self.added_hashes, self.scans = [], [], []
        SlotEngine.made.append(self)

    def _effective(self, k):
        return k or R.estimated_kernel_size(self.width, self.height)

    def add_edge_kernel_size(self, k):
        assert self.frame_count == 0
        k = self._effective(k)
        if k not in self._edge_sizes:
            self._edge_sizes.append(k)
            self.added_edges.append(k)
        return self._edge_sizes.index(k)

    def add_hash_geometry(self, size, lowpass):
        assert self.frame_count == 0
        if (size, lowpass) not in self._geometries:
            self._geometries.append((size, lowpass))
            self.added_hashes.append((size, lowpass))
        return self._geometries.index((size, lowpass))

    view = Engine.view

    def scan_content(self, weights, first=0, n=None, edge_slot=0):
        self.scans.append(("content", edge_slot))
        return super().scan_content(weights, first, n)

    def scan_hash_dist(self, first=0, n=None, hash_slot=0):
        self.scans.append(("hash", hash_slot))
        return super().scan_hash_dist(first, n)


def _slots(d):
    """(edge slot, hash slot) of the holder a detector is attached to: a view, or the engine itself for 0 / 0"""
    (eng,) = SlotEngine.made
    if d._engine is eng:
        return 0, 0
    assert isinstance(d._engine, SlotView) and d._engine._engine is eng
    return d._engine.edge_slot, d._engine.hash_slot


@pytest.fixture
def patched(monkeypatch):
    from pyscenedetect_b200 import scene_manager as sm_mod
    from pyscenedetect_b200.detectors import _base as base_mod
    monkeypatch.setattr(base_mod, "Engine", SlotEngine)
    monkeypatch.setattr(sm_mod, "Engine", SlotEngine)
    SlotEngine.made = []
    return SlotEngine


def _run(dets, w=640, h=360, stats=True, n=6):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = render_frames(ScenePlan(n, seed=3, min_len=2, max_len=4).params, w, h)
    sm = SceneManager(StatsManager() if stats else None, batch_size=4)
    for d in dets:
        sm.add_detector(d)
    sm.detect_scenes(ArrayVideoStream(frames, 30.0))
    return sm


def test_engine_deduplicates_automatic_and_explicit_kernel_sizes(patched):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    # 640x360 is auto-downscaled to 256x144, where the automatic kernel size is 5
    dets = [ContentDetector(kernel_size=5), AdaptiveDetector(), ContentDetector(weights=ALL, kernel_size=7),
            AdaptiveDetector(kernel_size=7), ContentDetector(kernel_size=3)]
    _run(dets)
    (eng,) = patched.made
    assert eng.config[0] == 5                 # the first edge detector's argument configures slot 0
    assert eng.added_edges == [7, 3]          # then every other effective size, in detector order
    assert [_slots(d)[0] for d in dets] == [0, 0, 1, 1, 2]
    assert {s for kind, s in eng.scans if kind == "content"} == {0, 1, 2}


def test_automatic_first_then_its_explicit_twin_shares_slot_0(patched):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    dets = [AdaptiveDetector(), ContentDetector(kernel_size=5), ContentDetector(kernel_size=9)]
    _run(dets)
    (eng,) = patched.made
    assert eng.config[0] == 0 and eng.added_edges == [9]
    assert [_slots(d)[0] for d in dets] == [0, 0, 1]


def test_edge_free_detectors_take_no_edge_slot(patched):
    from pyscenedetect_b200.detectors import ContentDetector
    # without a StatsManager a ContentDetector with edge weight 0 has no edge component: its kernel size is moot
    dets = [ContentDetector(kernel_size=9), ContentDetector(weights=ALL, kernel_size=3),
            ContentDetector(weights=ALL, kernel_size=5)]
    _run(dets, stats=False)
    (eng,) = patched.made
    assert eng.config[0] == 3 and eng.added_edges == [5]
    assert [_slots(d)[0] for d in dets] == [0, 0, 1]


def test_hash_geometry_slots_in_detector_order(patched):
    from pyscenedetect_b200.detectors import HashDetector, HistogramDetector
    dets = [HashDetector(size=16), HistogramDetector(), HashDetector(), HashDetector(size=8, lowpass=3),
            HashDetector(size=16, threshold=0.2)]
    _run(dets)
    (eng,) = patched.made
    assert eng.config[1:] == (16, 2)
    assert eng.added_hashes == [(8, 2), (8, 3)]
    assert [_slots(d)[1] for d in dets] == [0, 0, 1, 2, 0]
    assert {s for kind, s in eng.scans if kind == "hash"} == {0, 1, 2}


def test_one_size_one_geometry_adds_no_slot(patched):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector, HashDetector
    dets = [ContentDetector(kernel_size=5), AdaptiveDetector(kernel_size=5), HashDetector(size=8)]
    _run(dets)
    (eng,) = patched.made
    assert eng.added_edges == [] and eng.added_hashes == []
    assert all(d._engine is eng for d in dets)   # slot 0 everywhere: the engine itself, no view


def test_c_abi_slot_calls_reject_null_engines():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    slot = C_int32()
    assert lib.psd_engine_add_edge_kernel_size(None, 5, slot) == _capi.PSD_ERR_INVALID
    assert lib.psd_engine_add_hash_geometry(None, 8, 2, slot) == _capi.PSD_ERR_INVALID
    assert lib.psd_engine_edge_kernel_size_at(None, 0) == -1
    sums = np.zeros(1, dtype=_capi.SUMS_DTYPE)
    w = (C_double * 4)(1.0, 1.0, 1.0, 1.0)
    assert lib.psd_scan_content_edges(sums.ctypes.data, None, 1, 0, w, 4.0, None, None, None) == _capi.PSD_ERR_INVALID
