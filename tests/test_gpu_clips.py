"""Many clips in one engine pass on the GPU (pyscenedetect_b200/clips.py, clip_kernels.cu):

* after the scans and psd_clip_fill, every clip's slice of every metric array equals, byte for byte, the array a
  one-clip engine scans from that clip alone - for host frames, aligned and unaligned device frames, an RGB / NCHW
  layout and auto-downscaled frames;
* `detect_clips` equals one `SceneManager` per clip (cut lists, both scene lists, frame counts);
* every golden case of the reference, as the middle clip of a pass, gives its recorded cuts and scene list;
* the automaton and fix-up launches of a pass do not depend on its number of clips;
* a tiny first cut buffer (the retry) and a lowered per-pass bound (the drain) change nothing."""

from __future__ import annotations

import json
import os
from fractions import Fraction

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
BATCH = 16
LENGTHS = [0, 1, 2, 3, 4, 5, 10, 11, BATCH - 1, BATCH, BATCH + 1, 300]  # 2w and 2w + 1 for w = 1, 2, 5
ALL = (1.0, 1.0, 1.0, 1.0)
HSV = (1.0, 1.0, 1.0, 0.0)


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


def _render(n, w, h, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    if n == 0:
        return np.zeros((0, h, w, 3), np.uint8)
    return render_frames(ScenePlan(n, seed=seed, min_len=2, max_len=12 if n < 100 else 60).params, w, h)


def _source(frames, kind):
    """(frames in the given form, channel order): host numpy, or CUDA (torch) aligned, unaligned, NCHW RGB."""
    import torch
    if kind == "host":
        return frames, "bgr"
    if kind == "aligned":
        return torch.from_numpy(frames).cuda(), "bgr"
    n, h, w, _ = frames.shape
    if kind == "unaligned":
        fb = h * w * 3
        buf = torch.zeros(n * fb + 16, dtype=torch.uint8, device="cuda")
        buf[1:1 + n * fb] = torch.from_numpy(frames.reshape(-1)).cuda()
        return torch.as_strided(buf, (n, h, w, 3), (fb, w * 3, 3, 1), 1), "bgr"
    rgb = np.ascontiguousarray(frames[..., ::-1].transpose(0, 3, 1, 2))
    return torch.from_numpy(rgb).cuda().permute(0, 2, 3, 1), "rgb"


# -- 1. metric arrays ------------------------------------------------------------------------------------------------
FEATURES = 1 | 2 | 4 | 8 | 16


def _engine(w, h, sw, sh):
    from pyscenedetect_b200.engine import Engine
    e = Engine(w, h, FEATURES, width=sw, height=sh, max_batch=BATCH, edge_kernel_size=3)
    assert e.add_edge_kernel_size(7) == 1 and e.add_hash_geometry(16, 2) == 1
    return e


# (edge slot, hash slot, metric key) of every array checked; the adaptive ratios read the content_val of their slot
KEYS = ([(0, 0, ("content_val", HSV)), (0, 0, ("content_val", ALL)), (1, 0, ("content_val", ALL))]
        + [(0, 0, ("adaptive_ratio", HSV, w, 15.0)) for w in (1, 2, 5)]
        + [(1, 0, ("adaptive_ratio", ALL, 2, 5.0)), (0, 0, ("average_rgb",))]
        + [(0, 0, ("hist_correl", b)) for b in (256, 128, 7)]
        + [(0, 0, ("hash_dist",)), (0, 1, ("hash_dist",))])


def _arrays(lib, engine, clips=None) -> list[bytes]:
    """Every array of KEYS over what `engine` holds, as bytes; `clips`: (table buffer, clip count) of the pass."""
    from pyscenedetect_b200.device_cuts import scan_metric
    from pyscenedetect_b200.engine import DeviceBuffer
    n = engine.frame_count
    bufs, out = {}, []
    table = (clips[0].ptr, clips[1]) if clips else None
    for edge, hsh, key in KEYS:
        holder = engine.view(edge, hsh)
        buf = bufs[(edge, hsh) + key] = DeviceBuffer(max(8, n * 8))
        val = bufs[(edge, hsh, "content_val", key[1])].ptr if key[0] == "adaptive_ratio" else None
        scan_metric(lib, holder, key, buf.ptr, val, clips=table)
    engine.sync()
    for edge, hsh, key in KEYS:
        out.append(bufs[(edge, hsh) + key].download(n * 8).tobytes())
    for b in bufs.values():
        b.close()
    return out


def _submit(engine, frames, order, host_batches):
    if host_batches:
        for a in range(0, frames.shape[0], BATCH):
            engine.submit(frames[a:a + BATCH])
    elif frames.shape[0]:
        engine.submit(frames, channel_order=order)


@pytest.mark.parametrize("kind", ["host", "aligned", "unaligned", "nchw_rgb", "downscaled"])
def test_fixed_up_metric_arrays_equal_one_clip_engines(lib, kind):
    from pyscenedetect_b200.engine import DeviceBuffer
    from pyscenedetect_b200.scene_manager import SceneManager
    w, h = (640, 360) if kind == "downscaled" else (160, 90)
    _, _, (sw, sh) = SceneManager()._geometry(w, h)
    assert (sw, sh) == ((256, 144) if kind == "downscaled" else (w, h))
    clips = [_render(n, w, h, seed=7 * i + 3) for i, n in enumerate(LENGTHS)]
    src_kind = "host" if kind == "downscaled" else kind
    host = src_kind == "host"
    multi = _engine(w, h, sw, sh)
    if host:  # batches of BATCH frames across the clip boundaries
        _submit(multi, np.concatenate(clips), "bgr", True)
    else:     # a view of each clip of one device array, as detect_clips submits them
        allf, order = _source(np.concatenate(clips), src_kind)
        o = 0
        for c in clips:
            if len(c):
                multi.submit(allf[o:o + len(c)], channel_order=order)
            o += len(c)
    offsets = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    table = DeviceBuffer(offsets.nbytes)
    table.upload(offsets)
    got = _arrays(lib, multi, (table, len(clips)))
    multi.close()
    table.close()
    for i, c in enumerate(clips):
        if not len(c):
            continue
        one = _engine(w, h, sw, sh)
        f, order = _source(c, src_kind)
        _submit(one, f, order, host)
        want = _arrays(lib, one)
        one.close()
        b, e = int(offsets[i]) * 8, int(offsets[i + 1]) * 8
        for (edge, hsh, key), g, ww in zip(KEYS, got, want):
            assert g[b:e] == ww, (kind, len(c), edge, hsh, key)


# -- 2. end to end ---------------------------------------------------------------------------------------------------
def _detectors(name):
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    return {
        "content": lambda: [ContentDetector(threshold=20.0, min_scene_len=0.2)],
        "adaptive": lambda: [AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=0.12)],
        "threshold": lambda: [ThresholdDetector(threshold=40, min_scene_len=2, add_final_scene=True)],
        "histogram": lambda: [HistogramDetector(threshold=0.1, min_scene_len=0.1)],
        "hash": lambda: [HashDetector(threshold=0.3, min_scene_len=3)],
        "mix": lambda: [ContentDetector(threshold=20.0, min_scene_len=0.2),
                        ContentDetector(weights=ContentDetector.Components(*ALL), kernel_size=7, threshold=25.0),
                        AdaptiveDetector(adaptive_threshold=2.0, min_scene_len=4, window_width=3),
                        HistogramDetector(threshold=0.1, bins=64), HashDetector(threshold=0.3, min_scene_len=0.3),
                        HashDetector(size=16, threshold=0.25), ThresholdDetector(threshold=40, min_scene_len=0.1)],
    }[name]()


def _clip_set(kind):
    """(frames, fps) of clips of mixed sizes, lengths and rates, empty ones included."""
    sizes = [(160, 90), (96, 64), (640, 360)]
    rates = [25, Fraction(30000, 1001), 24, 30]
    out = []
    for i, n in enumerate(LENGTHS + [0, 37, 120]):
        w, h = sizes[i % 3]
        if n >= 100:
            w, h = 160, 90
        out.append((_render(n, w, h, seed=13 * i + 2), rates[i % 4]))
    return out


def _streams(clips, kind):
    from pyscenedetect_b200.video import ArrayVideoStream
    streams = []
    for f, fps in clips:
        if kind == "host":
            streams.append(ArrayVideoStream(f, fps))
        else:
            t, order = _source(f, "aligned" if len(f) % 2 else "nchw_rgb")
            streams.append(ArrayVideoStream(t, fps, channel_order=order))
    return streams


def _expect(clips, kind, name):
    from pyscenedetect_b200.scene_manager import SceneManager
    out = []
    for stream in _streams(clips, kind):
        sm = SceneManager(batch_size=BATCH)
        for d in _detectors(name):
            sm.add_detector(d)
        n = sm.detect_scenes(stream)
        out.append((n, [c.frame_num for c in sm.get_cut_list()],
                    [[(a.frame_num, b.frame_num) for a, b in sm.get_scene_list(start_in_scene=s)] for s in (0, 1)]))
    return out


def _got(results):
    return [(r.frames, r.cut_frames, [[(a.frame_num, b.frame_num) for a, b in r.scene_list(start_in_scene=s)]
                                      for s in (0, 1)]) for r in results]


@pytest.mark.parametrize("kind", ["host", "cuda"])
@pytest.mark.parametrize("name", ["content", "adaptive", "threshold", "histogram", "hash", "mix"])
def test_detect_clips_equals_scene_manager_per_clip(lib, name, kind):
    from pyscenedetect_b200.clips import detect_clips
    clips = _clip_set(kind)
    dets = _detectors(name)
    results = detect_clips(_streams(clips, kind), dets, batch_size=BATCH)
    assert all(d._engine is None for d in dets)
    want = _expect(clips, kind, name)
    assert _got(results) == want
    assert any(w[1] for w in want)


# -- 3. goldens as the middle clip of a pass ---------------------------------------------------------------------------
def _golden_cases():
    out = []
    for f in ("golden_v1", "golden_v2", "multi_detector_v1", "kernel_sizes_v1", "shared_pass_v1"):
        with open(os.path.join(HERE, "golden", f + ".json")) as fh:
            out += [(f, c) for c in json.load(fh)["cases"]]
    return out


@pytest.mark.parametrize("which", [f"{f}:{c['name']}" for f, c in _golden_cases()])
def test_golden_case_as_the_middle_clip(lib, which):
    import hashlib
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.golden_util import case_frames
    from tests.test_gpu_kernel_sizes import _frames as kernel_frames
    from tests.test_gpu_parity import _build
    f, case = next((f, c) for f, c in _golden_cases() if f"{f}:{c['name']}" == which)
    frames = kernel_frames(case["gen"]) if f == "kernel_sizes_v1" else case_frames(case)
    assert hashlib.sha256(frames.tobytes()).hexdigest() == case["frames_sha256"]
    dets = [_build({"det": d, "kw": kw}) for d, kw in case["dets"]] if "dets" in case else [_build(case)]
    auto = case.get("mode", "scene_manager") == "scene_manager" and bool(case.get("auto_downscale"))
    downscale = 1 if auto else case.get("downscale", 1)
    big = frames.shape[2] > 4096
    batch, before, after = (2, 1, 1) if big else (7, 5, 4)  # the case's first and last frames lie inside batches
    rev = frames[::-1]
    clips = [rev[:before], frames, rev[-after:]]
    results = detect_clips([ArrayVideoStream(c, case["fps"]) for c in clips], dets, auto_downscale=auto,
                           downscale=downscale, batch_size=batch)
    r = results[1]
    assert r.frames == frames.shape[0]
    assert r.cut_frames == case["cuts"]
    if case.get("scene_list") is not None:
        assert [[a.frame_num, b.frame_num] for a, b in r.scene_list()] == case["scene_list"]


# -- 4. launches per pass --------------------------------------------------------------------------------------------
def test_pass_launches_do_not_depend_on_the_clip_count(lib, monkeypatch):
    import torch
    from pyscenedetect_b200 import clips as clips_mod
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = torch.from_numpy(_render(2000, 64, 36, seed=4)).cuda()
    counts = []
    finish = clips_mod._Pass.finish

    def spy(self, engine, holders, done):
        before = lib.psd_launch_count()
        finish(self, engine, holders, done)
        counts.append(lib.psd_launch_count() - before)

    monkeypatch.setattr(clips_mod._Pass, "finish", spy)
    for n_clips in (1, 1000):
        k = 2000 // n_clips
        streams = [ArrayVideoStream(frames[i * k:(i + 1) * k], 25) for i in range(n_clips)]
        clips_mod.detect_clips(streams, _detectors("mix"), batch_size=64)
    # scans + fix-ups (one each per metric array, none for average_rgb) + the three psd_clip_cuts launches
    assert counts[0] == counts[1] > 0, counts


# -- 5. the retry and the drain ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["host", "cuda"])
def test_tiny_cut_buffer_and_lowered_pass_bound_change_nothing(lib, monkeypatch, kind):
    from pyscenedetect_b200 import clips as clips_mod
    clips = _clip_set(kind)
    want = _got(clips_mod.detect_clips(_streams(clips, kind), _detectors("mix"), batch_size=BATCH))
    passes = []
    finish = clips_mod._Pass.finish

    def spy(self, engine, holders, done):
        passes.append(engine.frame_count)
        finish(self, engine, holders, done)

    monkeypatch.setattr(clips_mod._Pass, "finish", spy)
    monkeypatch.setattr(clips_mod, "FIRST_CUTS_PER_FRAME", 0)
    monkeypatch.setattr(clips_mod, "MAX_PASS_FRAMES", 20)
    assert _got(clips_mod.detect_clips(_streams(clips, kind), _detectors("mix"), batch_size=BATCH)) == want
    assert len(passes) > 4 and max(passes) == 300  # the 300-frame clip is held whole
