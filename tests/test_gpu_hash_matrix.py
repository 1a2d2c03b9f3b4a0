"""The hash pass on the GPU against its stage twin (tests/hash_twin.py), bit for bit and with no tolerance: the row
buffer, the normalised image, the float32 low band and the hash words of every geometry of the matrix
(tests/hash_matrix_cases.py) through psd_test_hash_stages, then the production path (Engine with F_HASH and its hash
slots: shared-memory finish where the working set fits, host and device frames, sub-batches) against the twin's
words and hash_dist, and the frame sizes the rows kernel refused before its block height was capped by the frame
width through Engine, SceneManager and ParameterSweep.  The last test fails if the runs missed a branch that
tests/hash_plan_twin.py names."""

import numpy as np
import pytest

from oracle import intmath as M
from oracle import ref_detectors as R
from tests import hash_plan_twin as P
from tests import hash_twin as T
from tests.hash_matrix_cases import (CASES, SUB_BATCH, SUB_BATCH_FRAMES, SUB_BATCH_MAX_BATCH, WIDE_FRAMES, frame,
                                     frames)

pytestmark = pytest.mark.gpu

REACHED = set()   # branches of every launch_hash call made below, by the plan twin


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


_TWIN = {}


def twin(f: np.ndarray, size: int, lowpass: int) -> T.Stages:
    key = (f.shape, f.tobytes().__hash__(), size, lowpass)
    if key not in _TWIN:
        _TWIN[key] = T.stages(f, size, lowpass)
    return _TWIN[key]


def _device_frames(fr: np.ndarray, offset: int):
    from pyscenedetect_b200.engine import DeviceBuffer
    buf = DeviceBuffer(fr.nbytes + offset + 16)
    buf.upload(fr, offset)
    return buf, buf.ptr + offset


def _stages_on_device(lib, fr, geos, offset=0, with_images=True):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200._capi import hash_words
    nf, H, W = fr.shape[:3]
    buf, ptr = _device_frames(fr, offset)
    g = np.array(geos, np.int32).reshape(-1, 2)
    ns = [s * lp for s, lp in geos]
    rowbuf = np.zeros(sum(nf * H * n for n in ns), np.float32)
    words = np.zeros(sum(nf * hash_words(s) for s, _ in geos), np.uint64)
    image = np.zeros(sum(nf * n * n for n in ns), np.float64) if with_images else None
    low = np.zeros(sum(nf * s * s for s, _ in geos), np.float32) if with_images else None
    try:
        _capi.check(lib.psd_test_hash_stages(0, ptr, nf, W, H, W * H * 3, g.ctypes.data, len(geos), rowbuf.ctypes.data,
                                             words.ctypes.data, image.ctypes.data if with_images else None,
                                             low.ctypes.data if with_images else None), "psd_test_hash_stages")
    finally:
        buf.close()
    out, ro, wo, io, lo = [], 0, 0, 0, 0
    for (s, lp), n in zip(geos, ns):
        hw = hash_words(s)
        out.append((rowbuf[ro:ro + nf * H * n].reshape(nf, H, n), words[wo:wo + nf * hw].reshape(nf, hw),
                    image[io:io + nf * n * n].reshape(nf, n, n) if with_images else None,
                    low[lo:lo + nf * s * s].reshape(nf, s, s) if with_images else None))
        ro, wo, io, lo = ro + nf * H * n, wo + nf * hw, io + nf * n * n, lo + nf * s * s
    return out


def _same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _check_stages(case_name, fr, geos, got):
    for (s, lp), (rowbuf, words, image, low) in zip(geos, got):
        for i, f in enumerate(fr):
            tw = twin(f, s, lp)
            where = (case_name, (s, lp), i)
            assert _same_bits(rowbuf[i], tw.rowbuf), where
            if image is not None:
                assert _same_bits(image[i], tw.x), where
                assert _same_bits(low[i], tw.low), where
            assert np.array_equal(words[i], tw.words), where


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_every_stage_matches_twin(lib, case):
    fr = frames(case)
    got = _stages_on_device(lib, fr, case.geos)
    REACHED.update(P.branches([P.plan(case.W, case.H, s, lp, len(fr), force_global=True) for s, lp in case.geos],
                              len(fr)))
    _check_stages(case.name, fr, case.geos, got)


def test_unaligned_device_base_takes_the_byte_gray_path(lib):
    case = CASES[4]   # W % 16 == 0: only the base address keeps the kernel off the 16-pixel path
    fr = np.concatenate([frames(case), frames(case)[:1]])
    got = _stages_on_device(lib, fr, case.geos, offset=1)
    REACHED.update(P.branches([P.plan(case.W, case.H, s, lp, len(fr), force_global=True) for s, lp in case.geos],
                              len(fr), aligned=False))
    _check_stages(case.name + "_unaligned", fr, case.geos, got)


def _engine(W, H, geos, max_batch):
    from pyscenedetect_b200.engine import F_HASH, Engine
    eng = Engine(W, H, F_HASH, max_batch=max_batch, hash_size=geos[0][0], hash_lowpass=geos[0][1])
    for s, lp in geos[1:]:
        eng.add_hash_geometry(s, lp)
    return eng


def _check_engine(eng, fr, geos, where):
    for slot, (s, lp) in enumerate(geos):
        got = eng.read_hash(hash_slot=slot)
        dist = eng.scan_hash_dist(hash_slot=slot)
        prev = None
        for i, f in enumerate(fr):
            tw = twin(f, s, lp)
            assert np.array_equal(got[i], tw.words), (where, (s, lp), i)
            if prev is None:
                assert np.isnan(dist[i])
            else:
                assert dist[i] == np.count_nonzero(tw.bits != prev) / float(s * s), (where, (s, lp), i)
            prev = tw.bits


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_engine_words_and_dist_match_twin(lib, case):
    fr = frames(case)
    eng = _engine(case.W, case.H, case.geos, 64)
    try:
        eng.submit(fr)
        _check_engine(eng, fr, case.geos, case.name)
    finally:
        eng.close()
    REACHED.update(P.branches([P.plan(case.W, case.H, s, lp, 64) for s, lp in case.geos], len(fr)))


@pytest.mark.parametrize("source", ["host", "device_aligned", "device_unaligned"])
def test_engine_frame_sources(lib, source):
    case = CASES[3]
    fr = frames(case)
    eng = _engine(case.W, case.H, case.geos, 4)
    try:
        if source == "host":
            eng.submit(fr)
        else:
            buf, ptr = _device_frames(fr, 0 if source == "device_aligned" else 1)
            eng.submit_device(ptr, len(fr))
            eng.sync()
            buf.close()
        _check_engine(eng, fr, case.geos, source)
    finally:
        eng.close()


def test_engine_sub_batches(lib):
    distinct = frames(SUB_BATCH)   # cycled: frame 24, the first of the second sub-batch, is not frame 0
    fr = np.stack([distinct[i % len(distinct)] for i in range(SUB_BATCH_FRAMES)])
    eng = _engine(SUB_BATCH.W, SUB_BATCH.H, SUB_BATCH.geos, SUB_BATCH_MAX_BATCH)
    try:
        eng.submit(fr)
        _check_engine(eng, fr, SUB_BATCH.geos, SUB_BATCH.name)
    finally:
        eng.close()
    plans = [P.plan(SUB_BATCH.W, SUB_BATCH.H, s, lp, SUB_BATCH_MAX_BATCH) for s, lp in SUB_BATCH.geos]
    assert len(P.launch(plans, SUB_BATCH_FRAMES).sub_batches) == 2
    REACHED.update(P.branches(plans, SUB_BATCH_FRAMES))


def _wide_frames(W, H):
    return np.stack([frame("plan", W, H, 1), frame("hgrad", W, H, 2), frame("noise", W, H, 3)])


@pytest.mark.parametrize("wh,geos", WIDE_FRAMES, ids=[f"{w}x{h}" for (w, h), _ in WIDE_FRAMES])
def test_wide_frames_run(lib, wh, geos):
    W, H = wh
    fr = _wide_frames(W, H)
    eng = _engine(W, H, list(geos), 16)
    try:
        eng.submit(fr)
        _check_engine(eng, fr, list(geos), f"{W}x{H}")
    finally:
        eng.close()
    REACHED.update(P.branches([P.plan(W, H, s, lp, 16) for s, lp in geos], len(fr)))


def _sweep_frames():
    return np.stack([frame(k, 1920, 1080, 40 + i) for i, k in
                     enumerate(("plan", "plan", "hgrad", "hgrad", "noise", "vgrad", "vgrad", "plan"))])


def _expected(monkeypatch, fr, size, fps, threshold):
    """RefHashDetector's cuts and metrics with the twin's bits in place of cv2's hash."""
    monkeypatch.setattr(R, "hash_frame", lambda f, s, lp: twin(f, s, lp).bits.reshape(s, s))
    det = R.RefHashDetector(threshold=threshold, size=size, lowpass=1, min_scene_len=1, fps=fps, with_stats=True)
    cuts = R.run_detector(det, fr)
    return cuts, {t: v[det.metric_key] for t, v in det.metrics.items()}


def test_scene_manager_small_hashes_full_size(lib, monkeypatch):
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    fr, fps = _sweep_frames(), 30.0
    stats = StatsManager()
    sm = SceneManager(stats, batch_size=8)
    sm.auto_downscale = False
    sm.downscale = 1
    dets = [HashDetector(threshold=0.3, size=s, lowpass=1, min_scene_len=1) for s in range(1, 17)]
    for d in dets:
        sm.add_detector(d)
    sm.detect_scenes(ArrayVideoStream(fr, fps))
    want_cuts = set()
    for s, d in zip(range(1, 17), dets):
        cuts, metrics = _expected(monkeypatch, fr, s, fps, 0.3)
        want_cuts |= set(cuts)
        key = d.get_metrics()[0]
        for t, v in metrics.items():
            assert stats.get_metrics(FrameTimecode(t, fps), [key])[0] == v, (s, t)
    assert [c.frame_num for c in sm.get_cut_list()] == sorted(want_cuts)


def test_parameter_sweep_small_hashes_full_size(lib, monkeypatch):
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.scene_manager import shared_engine
    from pyscenedetect_b200.sweep import ParameterSweep
    fr, fps = _sweep_frames(), 30.0
    grid = [{"threshold": 0.3, "size": s, "lowpass": 1, "min_scene_len": 1} for s in range(1, 17)]
    sw = ParameterSweep(HashDetector, grid, batch_size=8)
    engine, holders = shared_engine(sw.groups, 1920, 1080, 1920, 1080, max_batch=8)
    try:
        engine.submit(fr)
        r = sw.run_scored(holders, fps)
        for k, cell in enumerate(grid):
            cuts, _ = _expected(monkeypatch, fr, cell["size"], fps, 0.3)
            assert r.cuts(k) == (cuts + [len(fr)] if cuts else []), cell   # scene ends: the cuts, then end_frame
    finally:
        engine.close()
    REACHED.update(P.branches([P.plan(1920, 1080, s, 1, 8) for s in range(1, 17)], len(fr)))


def test_twin_area_is_cv2_on_the_matrix_frames():
    """The comparisons above are exact against the twin; the twin's area image is cv2's on the same frames."""
    import cv2
    for case in CASES[2:5]:
        for f in frames(case):
            g = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
            for s, lp in case.geos:
                n = s * lp
                assert np.array_equal(twin(f, s, lp).area, cv2.resize(g, (n, n), interpolation=cv2.INTER_AREA))
                assert np.array_equal(twin(f, s, lp).area, M.resize_area(g, n))


def test_matrix_reached_every_branch():
    missing = P.REQUIRED - REACHED
    assert not missing, sorted(missing)
