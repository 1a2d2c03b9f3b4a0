"""`detect_clips(windows=...)` on the GPU (clips.py, psd_clip_cuts_steps):

* psd_clip_cuts_steps over the recorded metric arrays of the adversarial sequences equals psd_clip_cuts_step run clip
  by clip with each clip's step, and with every step equal it is bit-identical to psd_clip_cuts_step over all clips;
* 48 numpy (pageable and page-locked) and CUDA clips (BGR, RGB and an NCHW permutation, with and without
  `read_batch`) of several sizes, rates and lengths, each with its own crop, duration / end_time and frame_skip,
  equal a fresh SceneManager per clip in frame count, cuts, both scene lists, start, end and where each stream stands
  afterwards; with `stats=True` their CSVs are byte-equal;
* clips cropped to one size share an engine, and a pass makes one cut-automaton call whatever its mix of steps;
* the changed kernels use no stack frame or local memory."""

from __future__ import annotations

import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from tests import clip_steps_twin, clip_window_cases
from tests.test_gpu_clip_windows import (_ReadOnlyStream, _TwinMemory, _detectors, _got, _lists, _per_clip, _render,
                                         _upload)

pytestmark = pytest.mark.gpu

BATCH = 16
SIZES = [(160, 90), (200, 96), (192, 108), (320, 180)]
RATES = [25, Fraction(30000, 1001), 24, 60]
SOURCES = ["host", "pinned", "cuda", "read_only"]
# (0, 6, 159, 83) crops the first three sizes to 160x78; (20, 0, 275, 143) gives the 320x180 clips a 256-wide crop,
# which scores at 255 wide; (4, 4, 400, 400) ends outside every frame
CROPS = [None, (0, 6, 159, 83), (20, 0, 275, 143), (7, 5, 120, 70), (150, 80, 3, 2), (4, 4, 400, 400)]
SPANS = [("duration", 40), ("duration", 1.3), ("duration", "2.5s"), ("end_time", 90), ("end_time", 3.0),
         ("end_time", "00:00:02.200")]


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


# -- 1. the per-clip step entry on adversarial metric sequences -------------------------------------------------------
def _run(lib, cells, k, offsets, first, mf, step, end, steps=None):
    """(offsets, cuts) of psd_clip_cuts_step (steps None) or psd_clip_cuts_steps over the clip table `offsets`."""
    import ctypes as C
    from pyscenedetect_b200.engine import DeviceBuffer
    c = len(first)
    bufs = [_upload(np.asarray(offsets, np.int64)), _upload(np.asarray(first, np.int64)),
            _upload(np.asarray(mf, np.int64))]
    ebuf = _upload(np.asarray(end, np.int64)) if end is not None else None
    cap = 1 << 20
    cuts, obuf = DeviceBuffer(cap * 8), DeviceBuffer((k * c + 1) * 8)
    try:
        args = [cells, k, bufs[0].ptr, bufs[1].ptr, c, bufs[2].ptr, cuts.ptr, cap, obuf.ptr]
        if steps is None:
            rc = lib.psd_clip_cuts_step(*args, step, ebuf.ptr if ebuf else None, None)
        else:
            rc = lib.psd_clip_cuts_steps(*args, (C.c_int64 * c)(*steps), ebuf.ptr if ebuf else None, None)
        assert rc == 0, lib.psd_last_error()
        offs = obuf.download((k * c + 1) * 8).view(np.int64)
        total = int(offs[-1])
        assert total <= cap
        return offs.tobytes(), cuts.download(total * 8).tobytes()
    finally:
        for b in bufs + [cuts, obuf] + ([ebuf] if ebuf else []):
            b.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_steps_entry_on_adversarial_sequences(lib, seed):
    rng = np.random.default_rng(seed)
    for kind, _w, sizes, metric, metric2, params in clip_window_cases.groups():
        mbuf = _upload(metric)
        m2 = _upload(metric2) if metric2 is not None else None
        c = len(sizes)
        cells, k, mf = clip_window_cases.cells_and_min_frames(kind, params, mbuf.ptr, m2.ptr if m2 else None, c,
                                                              seed=seed)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        try:
            # every step equal: psd_clip_cuts_step's bytes
            for step in (1, 3):
                first, end = clip_window_cases.first_and_end(sizes, step, seed=20 + seed)
                for e in (None, end):
                    want = _run(lib, cells, k, off, first, mf, step, e)
                    assert _run(lib, cells, k, off, first, mf, None, e, [step] * c) == want, (kind, step)
            # mixed steps: clip j's lists are psd_clip_cuts_step's over clip j alone with its step
            steps = [int(s) for s in rng.integers(1, 6, c)]
            first, end = clip_window_cases.first_and_end(sizes, 6, seed=30 + seed)
            for e in (None, end):
                got = _lists(*_run(lib, cells, k, off, first, mf, None, e, steps))
                for j in range(c):
                    one = _lists(*_run(lib, cells, k, off[j:j + 2], first[j:j + 1], mf.reshape(k, c)[:, j],
                                       steps[j], e[j:j + 1] if e is not None else None))
                    assert [got[i * c + j] for i in range(k)] == one, (kind, j, steps[j])
                twin_cells = (type(cells[0]) * k)(*cells)
                with _TwinMemory(metric, metric2, twin_cells):
                    assert got == clip_steps_twin.clip_cut_lists_steps(twin_cells, k, off, first, c, mf, steps, e)
                assert any(got), kind
        finally:
            mbuf.close()
            if m2:
                m2.close()


def test_steps_entry_rejects_bad_steps(lib):
    import ctypes as C
    from pyscenedetect_b200 import _capi
    cells = (_capi.PsdSweepCell * 1)()
    cells[0].kind, cells[0].metric = _capi.SWEEP_CONTENT, 4096
    for bad in (0, -1):
        steps = (C.c_int64 * 3)(1, bad, 2)
        assert lib.psd_clip_cuts_steps(cells, 1, 4096, 4096, 3, 4096, 4096, 16, 4096, steps, None, None) \
            == _capi.PSD_ERR_INVALID
        assert f"psd_clip_cuts_steps: frame_step[1] is {bad}, must be >= 1".encode() in lib.psd_last_error()
    assert lib.psd_clip_cuts_steps(cells, 1, 4096, 4096, 3, 4096, 4096, 16, 4096, None, None, None) \
        == _capi.PSD_ERR_INVALID
    assert b"psd_clip_cuts_steps: no frame_step array" in lib.psd_last_error()


# -- 2. detect_clips(windows=) against one SceneManager per clip ---------------------------------------------------------
_PINNED = []  # page-locked copies stay alive for the module


def _clip_set(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        w, h = SIZES[int(rng.integers(len(SIZES)))]
        length = int(rng.choice([0, 1, 2, 17, 45, 90, 150, 240]))
        out.append((_render(length, w, h, seed=seed + 7 * i), RATES[i % len(RATES)], SOURCES[i % len(SOURCES)]))
    return out


def _streams(clips):
    """Every clip as its source says: numpy pageable or page-locked, or CUDA in BGR, RGB or an NCHW permutation, read
    with read_batch or with read() only."""
    import torch
    from pyscenedetect_b200.engine import PinnedBuffer
    from pyscenedetect_b200.video import ArrayVideoStream
    out = []
    for i, (f, fps, source) in enumerate(clips):
        if source == "host":
            out.append(ArrayVideoStream(f, fps))
        elif source == "pinned":
            p = PinnedBuffer(max(1, f.nbytes))
            _PINNED.append(p)
            a = p.array[:f.nbytes].reshape(f.shape)
            a[...] = f
            out.append(ArrayVideoStream(a, fps, pinned=True))
        else:
            layout = (i // len(SOURCES)) % 3
            if layout == 0:
                t, order = torch.from_numpy(f).cuda(), "bgr"
            elif layout == 1:
                t, order = torch.from_numpy(np.ascontiguousarray(f[..., ::-1])).cuda(), "rgb"
            else:
                nchw = np.ascontiguousarray(f[..., ::-1].transpose(0, 3, 1, 2))
                t, order = torch.from_numpy(nchw).cuda().permute(0, 2, 3, 1), "rgb"
            cls = _ReadOnlyStream if source == "read_only" else ArrayVideoStream
            out.append(cls(t, fps, channel_order=order))
    return out


def _windows(n, seed, stats=False):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        if rng.random() < 0.1:
            out.append(None)
            continue
        w = {}
        if rng.random() < 0.75:
            w["crop"] = CROPS[int(rng.integers(len(CROPS)))]
        if not stats and rng.random() < 0.7:
            w["frame_skip"] = int(rng.integers(0, 4))
        if rng.random() < 0.7:
            key, value = SPANS[int(rng.integers(len(SPANS)))]
            w[key] = value
        out.append(w)
    return out


def _compare(clips, dets_fn, windows, stats=False):
    from pyscenedetect_b200.clips import detect_clips
    streams = _streams(clips)
    results = detect_clips(streams, dets_fn(), batch_size=BATCH, stats=stats, windows=windows)
    for j, (r, video, w) in enumerate(zip(results, _streams(clips), windows)):
        assert _got(r, stats) == _per_clip(dets_fn, video, w or {}, stats), (j, w, clips[j][2])
        assert streams[j].frame_number == video.frame_number, (j, w)
    return results


@pytest.mark.parametrize("name", ["content", "adaptive", "threshold", "histogram", "hash", "mix"])
def test_windows_equal_scene_manager_per_clip(lib, name):
    clips = _clip_set(48, seed=3)
    results = _compare(clips, lambda: _detectors(name), _windows(len(clips), seed=len(name)))
    if name != "threshold":
        assert any(r.cut_frames for r in results)


def test_stats_with_crops_and_durations(lib):
    clips = _clip_set(40, seed=8)
    windows = _windows(len(clips), seed=4, stats=True)
    results = _compare(clips, lambda: _detectors("mix"), windows, stats=True)
    assert all(r.stats_csv.startswith(b"Frame Number,Timecode,") for r in results)


def test_one_engine_per_cropped_size_and_one_cut_call_per_pass(lib, monkeypatch):
    import torch
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200 import scene_manager
    from pyscenedetect_b200.video import ArrayVideoStream
    made = []

    class Counted(scene_manager.Engine):
        def __init__(self, src_width, src_height, *a, **kw):
            made.append((src_width, src_height))
            super().__init__(src_width, src_height, *a, **kw)

    calls = []

    def counted(name, fn):
        def call(*a):
            calls.append(name)
            return fn(*a)
        return call

    monkeypatch.setattr(scene_manager, "Engine", Counted)
    for name in ("psd_clip_cuts", "psd_clip_cuts_step", "psd_clip_cuts_steps"):
        monkeypatch.setattr(lib, name, counted(name, getattr(lib, name)))
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 4.0)  # no retry of the cut buffer
    # letterboxed 1920x1080 and 1920x800 sources, both cropped to 1920x800, on the GPU: one engine, one pass
    tall = torch.from_numpy(_render(40, 1920, 1080, seed=1)).cuda()
    wide = torch.from_numpy(_render(40, 1920, 800, seed=2)).cuda()
    streams = [ArrayVideoStream(tall[i * 10:(i + 1) * 10], 25) if i % 2 else
               ArrayVideoStream(wide[i * 10:(i + 1) * 10], 24) for i in range(4)]
    windows = [{"crop": (0, 0, 1919, 799)}, {"crop": (0, 140, 1919, 939), "frame_skip": 1},
               {"crop": (0, 0, 1919, 799), "end_time": 0.2}, {"crop": (0, 140, 1919, 939), "frame_skip": 2,
                                                              "duration": 8}]
    results = clips_mod.detect_clips(streams, _detectors("mix"), batch_size=BATCH, windows=windows)
    assert made == [(1920, 800)] and calls == ["psd_clip_cuts_steps"]
    for j, (r, w) in enumerate(zip(results, windows)):
        video = ArrayVideoStream(streams[j]._frames, streams[j].frame_rate)
        assert _got(r) == _per_clip(lambda: _detectors("mix"), video, w), j


# -- 3. the changed kernels ---------------------------------------------------------------------------------------------
def test_cut_kernels_use_no_stack_or_local_memory():
    from pyscenedetect_b200 import _capi
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([tool, "-res-usage", _capi.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    found = re.findall(r"Function (\S*psd_clip_cuts_kernel\S*):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert len(found) == 2, out[:2000]
    for fn, stack, local in found:
        assert stack == "0" and local == "0", f"{fn} uses a stack frame or local memory"
