"""GPU tests of the stage from integer sums to cut list: the trailing scans (psd_scan_*), the single-cell cut
automata (`DeviceCuts`) and the batched sweep cells (`ParameterSweep.run_scored`), against what PySceneDetect
0.7.1 computed from the same scripted integer results (tests/automata_inputs.py, recorded in
tests/golden/automata_v1.json.gz).  The scripted results are uploaded into `sharding.GatheredResults`, so no
pixels and no Engine are involved.  The device FlashFilter is also compared with the reference FlashFilter's
own output in tests/golden/reference_compat.json.gz."""

import gzip
import json
import math
import os
import random
import zlib

import numpy as np
import pytest

from tests import automata_inputs as A
from tests import sweep_model

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SPECS = A.sequences()
TOLS = (0, 2)


@pytest.fixture(scope="module")
def lib():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    return lib


def _spec(name):
    return next(s for s in SPECS if s["name"] == name)


def _results(inp):
    from pyscenedetect_b200.sharding import GatheredResults
    return GatheredResults(inp.sums, inp.yhist, inp.n_pixels, hashes=inp.hashes, hash_size=inp.hash_size,
                           hash_lowpass=2)


def _hex(arr):
    return [None if math.isnan(v) else float(v).hex() for v in arr]


def _names(*dets):
    return [s["name"] for s in SPECS if s["det"] in dets]


@pytest.mark.parametrize("name", _names("content", "adaptive", "threshold", "histogram", "hash"))
def test_scans_match_reference(lib, name):
    """content_val, components, adaptive_ratio, average_rgb and hash_dist bit for bit (NaN exactly where the
    reference records nothing); hist_diff within 1e-9 and exactly 1.0 where the reference's is; scans that
    start at frame k > 0 (the sharded tail's prev_hist / prev_hash) equal the slice of the whole scan."""
    spec = _spec(name)
    rec, inp = A.recorded(spec)
    res = _results(inp)
    n, det, m = spec["n"], spec["det"], rec["metrics"]
    starts = sorted({k for k in (1, n // 2, n - 1) if 0 < k < n})
    if det in ("content", "adaptive"):
        for w in spec["weights"]:
            val, comps = res.scan_content(w)
            assert _hex(val) == m[A.metric_key("content_val", w)], w
            for c, key in enumerate(("delta_hue", "delta_sat", "delta_lum", "delta_edges")):
                want = m[A.metric_key(key)]
                assert want[:1] == [None] * min(1, n) and (n == 0 or comps[0, c] == 0.0)
                assert _hex(comps[1:, c]) == want[1:], key
            for key, want in m.items():
                if key.startswith("adaptive_ratio|" + repr(list(w)) + "|"):
                    _, _, win, mcv = key.split("|")
                    assert _hex(res.scan_adaptive(val, int(win), float(mcv))) == want, key
    elif det == "threshold":
        assert _hex(res.scan_average()) == m[A.metric_key("average_rgb")]
    elif det == "hash":
        got = res.scan_hash_dist()
        assert _hex(got) == m[A.metric_key("hash_dist")]
        for k in starts:
            assert res.scan_hash_dist(first=k).tobytes() == got[k:].tobytes(), k
    else:
        for key, want in m.items():
            bins = int(key.split("|")[1])
            got = res.scan_hist_correl(bins)
            assert len(got) == len(want) == n, bins
            if n == 0:
                continue
            assert want[0] is None and math.isnan(got[0]), bins
            ref = np.array([float.fromhex(x) for x in want[1:]])
            assert np.all(np.abs(got[1:] - ref) <= 1e-9), (bins, np.max(np.abs(got[1:] - ref)))
            assert np.array_equal(got[1:] == 1.0, ref == 1.0), bins
            for k in starts:
                assert res.scan_hist_correl(bins, first=k).tobytes() == got[k:].tobytes(), (bins, k)


def _device_cuts(dc, spec, kw):
    fps, first = spec["fps"], spec["first_frame"]
    det = spec["det"]
    if det == "content":
        return dc.content(weights=tuple(kw["weights"]), threshold=kw["threshold"], min_scene_len=kw["min_scene_len"],
                          suppress=kw["filter_mode"] == "SUPPRESS", fps=fps, first_frame=first)
    if det == "adaptive":
        return dc.adaptive(weights=tuple(kw["weights"]), adaptive_threshold=kw["adaptive_threshold"],
                           min_scene_len=kw["min_scene_len"], window_width=kw["window_width"],
                           min_content_val=kw["min_content_val"], fps=fps, first_frame=first)
    if det == "threshold":
        return dc.threshold(threshold=kw["threshold"], min_scene_len=kw["min_scene_len"], fade_bias=kw["fade_bias"],
                            add_final_scene=kw["add_final_scene"], ceiling=kw["method"] == "CEILING", fps=fps,
                            first_frame=first)
    if det == "histogram":
        return dc.histogram(threshold=kw["threshold"], bins=kw["bins"], min_scene_len=kw["min_scene_len"], fps=fps,
                            first_frame=first)
    return dc.hash(threshold=kw["threshold"], min_scene_len=kw["min_scene_len"], fps=fps, first_frame=first)


def _increasing(spec, kw) -> bool:
    """Every automaton emits strictly increasing frames except the threshold one with |fade_bias| > 1."""
    return spec["det"] != "threshold" or abs(kw["fade_bias"]) <= 1.0


@pytest.mark.parametrize("name", _names("content", "adaptive", "threshold", "histogram", "hash"))
def test_single_cell_automata_match_reference(lib, name):
    """`DeviceCuts` gives the reference's cut list for every recorded parameter set (which include every
    min_scene_len form, so flash_filter_frames / min_len_frames are pinned too)."""
    from pyscenedetect_b200.device_cuts import DeviceCuts
    spec = _spec(name)
    rec, inp = A.recorded(spec)
    dc = DeviceCuts(_results(inp))
    for run in rec["runs"]:
        got = _device_cuts(dc, spec, run["kw"])
        if _increasing(spec, run["kw"]):
            assert got == run["cuts"], run["kw"]
        else:
            assert sorted(set(got)) == run["cuts"], run["kw"]


def _detector_kw(spec, kw):
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import ContentDetector, ThresholdDetector
    kw = dict(kw)
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    if "filter_mode" in kw:
        kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
    if "method" in kw:
        kw["method"] = ThresholdDetector.Method[kw["method"]]
    if spec["det"] == "hash":
        kw.update(size=spec["size"], lowpass=2)
    return kw


def _cls(det):
    from pyscenedetect_b200 import detectors as D
    return {"content": D.ContentDetector, "adaptive": D.AdaptiveDetector, "threshold": D.ThresholdDetector,
            "histogram": D.HistogramDetector, "hash": D.HashDetector}[det]


@pytest.mark.parametrize("name", _names("content", "adaptive", "threshold", "histogram", "hash"))
def test_sweep_cells_match_reference(lib, name):
    """One ParameterSweep per sequence over all of its recorded parameter sets: every cell's predicted list
    and its counts against a small ground truth."""
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    spec = _spec(name)
    rec, inp = A.recorded(spec)
    first, n = spec["first_frame"], spec["n"]
    end = first + n
    runs = rec["runs"]
    assert runs
    if n == 0:  # a sweep evaluates scored frames: an empty sequence is refused, not swept to nothing
        sw = ParameterSweep(_cls(spec["det"]), [_detector_kw(spec, r["kw"]) for r in runs])
        with pytest.raises(ValueError, match="non-zero number of frames"):
            sw.run_scored([_results(inp)] * len(sw.groups), spec["fps"], first_frame=first)
        return
    gt = GroundTruth(sorted(set(runs[0]["cuts"][::2] + [c + 1 for c in runs[-1]["cuts"][1::3]] + [first + n // 2])),
                     [(first + n // 4, first + n // 4 + 3)])
    sw = ParameterSweep(_cls(spec["det"]), [_detector_kw(spec, r["kw"]) for r in runs], tolerances=TOLS)
    res = _results(inp)
    r = sw.run_scored([res] * len(sw.groups), spec["fps"], gt, first_frame=first)
    for k, run in enumerate(runs):
        pred = sweep_model.predicted_list(run["cuts"], end)
        assert r.cuts(k) == pred, run["kw"]
        if _increasing(spec, run["kw"]):
            assert r.raw_count(k) == len(run["cuts"]), run["kw"]
        else:
            assert r.raw_count(k) >= len(run["cuts"]), run["kw"]
        for t in TOLS:
            want_h, want_f = sweep_model.score(pred, gt.hard_cuts, gt.fades, t)
            assert (*r.hard(k, t), int(r.hard_offset(k, t)[0]), r.hard_offset(k, t)[1]) == want_h, (run["kw"], t)
            assert r.fades(k) == want_f, run["kw"]


@pytest.fixture(scope="module")
def compat():
    with gzip.open(os.path.join(HERE, "golden", "reference_compat.json.gz"), "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("mode", ["MERGE", "SUPPRESS"])
@pytest.mark.parametrize("length", [15, 0, 1, 40, 0.5, "0.6s", "00:00:00.700", "20"])
def test_flash_filter_matches_reference(lib, compat, mode, length):
    """The `above` sequences of test_compat_vs_reference.test_flash_filter_sequences (same seeds), through
    psd_cuts_flash_filter and through a ContentDetector sweep cell, against the reference FlashFilter."""
    from pyscenedetect_b200._capi import SUMS_DTYPE
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.device_cuts import flash_filter_frames
    from pyscenedetect_b200.engine import DeviceBuffer
    from pyscenedetect_b200.sharding import GatheredResults
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(zlib.crc32(f"{mode}|{length}".encode()) & 0xFFFF)
    n, cap = 600, 1024
    for fps, want in zip((30.0, 24000 / 1001), compat["flash_filter"][f"{mode}|{length}"]):
        p = rng.choice([0.05, 0.2, 0.5])
        above = np.array([rng.random() < p for _ in range(n)], dtype=np.uint8)
        expect = [c for t in range(n) for c in want["cuts"].get(str(t), [])]
        flags, cuts, count = DeviceBuffer(n), DeviceBuffer(cap * 8), DeviceBuffer(8)
        flags.upload(above)
        rc = lib.psd_cuts_flash_filter(flags.ptr, n, 0, flash_filter_frames(length, fps), int(mode == "SUPPRESS"),
                                       cuts.ptr, count.ptr, cap, None)
        assert rc == 0, lib.psd_last_error()
        m = int(count.download(4).view(np.int32)[0])
        assert cuts.download(m * 8).view(np.int64).tolist() == expect, fps
        # content_val = sad_lum exactly (P = 1, luma only): 40 where above (a tie with the threshold), 39 elsewhere.
        # Frame 0 is scored too (has_prev = 1), so that the first draw reaches the automaton as well.
        sums = np.zeros(n, dtype=SUMS_DTYPE)
        sums["has_prev"] = 1
        sums["sad_lum"] = 39 + above.astype(np.uint64)
        sw = ParameterSweep(ContentDetector, [dict(luma_only=True, threshold=40.0, min_scene_len=length,
                                                   filter_mode=FlashFilter.Mode[mode])])
        r = sw.run_scored([GatheredResults(sums, None, 1)], fps)
        assert r.cuts(0) == sweep_model.predicted_list(expect, n) and r.raw_count(0) == len(expect), fps


def test_device_cuts_capacity_raises(lib):
    """More cuts than `max_cuts` raise instead of returning a truncated list."""
    from pyscenedetect_b200.device_cuts import DeviceCuts
    best = None
    for spec in SPECS:
        if spec["det"] != "content":
            continue
        for run in A.recording()[spec["name"]]["runs"]:
            if best is None or len(run["cuts"]) > len(best[1]["cuts"]):
                best = (spec, run)
    spec, run = best
    _, inp = A.recorded(spec)
    m = len(run["cuts"])
    assert m >= 20
    res = _results(inp)
    assert _device_cuts(DeviceCuts(res, max_cuts=m), spec, run["kw"]) == run["cuts"]
    with pytest.raises(RuntimeError, match="exceed the device cut buffer"):
        _device_cuts(DeviceCuts(res, max_cuts=m - 1), spec, run["kw"])
