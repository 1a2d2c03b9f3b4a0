"""GPU tests of the sweep over detector sets (`ParameterSweep(detector_sets=...)`: every distinct detector's automaton
once per setting and clip, then psd_clip_union merges them into every set's cut list before psd_clip_eval(_tables)):

* psd_clip_union equals its twin (tests/sweep_sets_twin.py) on made-up tables: empty, identical, interleaved and
  unsorted member lists, repeated members, a set at the member bound, and the overflow index;
* every case of tests/golden/multi_detector_v1.json, as a set, gives the reference SceneManager's recorded cut list
  followed by its end frame;
* the five classes' grids and 64 Adaptive x Threshold combinations (plus mixes of hash sizes, histogram bins and edge
  kernel sizes) under two settings, over 40 pageable, page-locked and CUDA (BGR, RGB, NCHW) clips, equal one
  `detect_clips` per (setting, set) scored on the host, and the one-detector sets equal per-class sweeps."""

from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from tests import sweep_model, sweep_sets_twin
from tests.test_gpu_sweep_clips import TOLS, _clip_set, _cls, _counts, _random_grid, _totals
from tests.test_gpu_sweep_settings import _open, _sources

pytestmark = pytest.mark.gpu

SETTINGS = [{}, {"frame_skip": 1}]
KINDS = ["content", "adaptive", "threshold", "histogram", "hash"]


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


# -- 1. the entry --------------------------------------------------------------------------------------------------------
def _union_case(rng, n_lists, n_clips):
    """(list, clip) cut lists, list-major: empty, shared, interleaved, unsorted with repeats."""
    lists = []
    for t in range(n_lists * n_clips):
        shape = t % 5
        if shape == 0:
            lists.append([])
        elif shape == 1:
            lists.append(list(range(3, 40, 4)))                       # the same in many lists
        elif shape == 2:
            lists.append(sorted(rng.sample(range(200), rng.randint(1, 30))))
        elif shape == 3:
            lists.append(list(range(t % 7, 300, 7)))                  # interleaves with its neighbours
        else:
            lists.append([rng.randrange(60) for _ in range(rng.randint(1, 25))])  # unsorted, repeats
    return lists


def test_union_entry_equals_the_twin(lib):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200._capi import check
    from pyscenedetect_b200.engine import DeviceBuffer
    rng = random.Random(3)
    n_lists, n_clips, bound = 20, 7, _capi.SWEEP_MAX_MEMBERS
    lists = _union_case(rng, n_lists, n_clips)
    cells = [[i] for i in range(n_lists)] + [[i, i] for i in range(0, n_lists, 3)] + \
        [rng.sample(range(n_lists), rng.randint(2, 6)) for _ in range(40)] + [list(range(bound)), list(range(4, 20))]
    assert max(len(c) for c in cells) == bound
    offs = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    flat = np.array([x for x in lists for x in x], np.int64)
    co = (C.c_int32 * (len(cells) + 1))(*np.concatenate([[0], np.cumsum([len(c) for c in cells])]).tolist())
    cl = (C.c_int32 * int(co[len(cells)]))(*[i for c in cells for i in c])
    m = len(cells) * n_clips
    for max_cuts in (64, 20):
        cuts, obuf = DeviceBuffer(flat.nbytes), DeviceBuffer(offs.nbytes)
        cuts.upload(flat)
        obuf.upload(offs)
        out_o, over, unique = DeviceBuffer(8 * (m + 1)), DeviceBuffer(8), DeviceBuffer(4 * n_lists * n_clips)
        check(lib.psd_clip_union(cuts.ptr, obuf.ptr, n_lists, n_clips, len(flat), max_cuts, co, cl, len(cells),
                                 unique.ptr, None, 0, out_o.ptr, over.ptr, None), "psd_clip_union")
        total = int(out_o.download(8, offset=8 * m).view(np.int64)[0])
        out = DeviceBuffer(max(8, 8 * total))
        check(lib.psd_clip_union(cuts.ptr, obuf.ptr, n_lists, n_clips, len(flat), max_cuts, co, cl, len(cells),
                                 unique.ptr, out.ptr, total, out_o.ptr, over.ptr, None), "psd_clip_union")
        got_o = out_o.download(8 * (m + 1)).view(np.int64)
        got = out.download(8 * total).view(np.int64)
        # the twin on the same lists
        long = [t for t, x in enumerate(lists) if len(x) > max_cuts]
        kept = [[] if t in long else sorted(set(x)) for t, x in enumerate(lists)]
        want = sweep_sets_twin.union_lists(kept, n_clips, list(co), list(cl), len(cells))
        assert [got[got_o[t]:got_o[t + 1]].tolist() for t in range(m)] == want
        assert int(over.download(8).view(np.int64)[0]) == (long[0] if long else -1)
        # the member lists are sorted and unique in place
        data = cuts.download(flat.nbytes).view(np.int64)
        for t, x in enumerate(lists):
            if t not in long:
                assert data[offs[t]:offs[t] + len(set(x))].tolist() == sorted(set(x))
        for b in (cuts, obuf, out_o, over, unique, out):
            b.close()
    assert any(want) and any(len(x) != len(set(x)) or x != sorted(x) for x in lists)


# -- 2. the reference's SceneManager with several detectors ---------------------------------------------------------------
def test_multi_detector_cases_as_sets(lib):
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.golden_util import case_frames
    from tests.test_gpu_multi_detector import _cases, _detector
    for case in _cases():
        frames = case_frames(case)
        setting = {"auto_downscale": bool(case.get("auto_downscale"))}
        if not setting["auto_downscale"]:
            setting["downscale"] = case.get("downscale", 1)
        dets = [_detector(det, kw) for det, kw in case["dets"]]
        for d in dets:
            d.stats_manager = None
        sw = ParameterSweep(detector_sets=[dets] + [[d] for d in dets], tolerances=TOLS, settings=[setting])
        r = sw.run_clips([ArrayVideoStream(frames, case["fps"])])
        want = case["cuts"] + [frames.shape[0]] if case["cuts"] else []
        assert r.cuts(0, 0) == want, case["name"]
        singles = set()
        for k in range(1, len(dets) + 1):
            singles |= set(r.cuts(k, 0)[:-1])
        assert sorted(singles) == case["cuts"], case["name"]


# -- 3. a dataset -----------------------------------------------------------------------------------------------------------
def _sets(rng):
    """The five classes' grids (8 cells each) as one-detector sets, 64 Adaptive x Threshold combinations, and mixes of
    hash geometries, histogram bins and edge kernel sizes."""
    from pyscenedetect_b200.detectors import ContentDetector, HashDetector, HistogramDetector
    grids = {det: _random_grid(det, 8 if det != "adaptive" else 16, rng) for det in KINDS}
    grids["threshold"] = grids["threshold"][:4]
    singles = [_cls(det)(**p) for det in KINDS for p in grids[det]]
    ad = [d for d in singles if type(d).__name__ == "AdaptiveDetector"]
    th = [d for d in singles if type(d).__name__ == "ThresholdDetector"]
    cross = [[a, t] for a in ad for t in th]
    assert len(cross) == 64
    edges = ContentDetector(threshold=20.0, weights=ContentDetector.Components(1.0, 1.0, 1.0, 1.0), kernel_size=5)
    mixes = [[HashDetector(size=16, lowpass=2, threshold=0.3), HistogramDetector(bins=128, threshold=0.05)],
             [HashDetector(size=8, lowpass=3, threshold=0.25), HashDetector(size=12, lowpass=2, threshold=0.3), edges],
             [edges, ContentDetector(threshold=15.0), singles[0], ad[0], th[0], th[0]]]
    return grids, singles, cross + mixes


def test_sets_over_a_dataset_equal_detect_clips(lib):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.sweep import ParameterSweep
    rng = random.Random(11)
    clips = _sources(_clip_set(7))
    gts = [gt for _, _, gt, _ in clips]
    grids, singles, combos = _sets(rng)
    sets = singles + combos
    keep = []
    sw = ParameterSweep(detector_sets=sets, tolerances=TOLS, settings=SETTINGS)
    r = sw.run_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], gts)
    assert len(r) == len(SETTINGS) * len(sets)
    n = len(sets)
    for s, st in enumerate(SETTINGS):
        for k, dets in enumerate(sets):
            dets = dets if isinstance(dets, list) else [dets]
            res = detect_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], dets, **st)
            for j, cr in enumerate(res):
                end = cr.end.frame_num + 1
                assert r.end_frame(j, setting=s) == end
                preds = sweep_model.predicted_list(cr.cut_frames, end)
                assert r.cuts(s * n + k, j) == preds, (s, k, j)
                gt = gts[j]
                for t in TOLS:
                    h, f = sweep_model.score(preds, gt.hard_cuts, gt.fades, t)
                    assert r.hard(s * n + k, j, t) == h[:3] and r.hard_offset(s * n + k, j, t) == (float(h[3]), h[4])
                assert r.fades(s * n + k, j) == f
    assert any(r.cuts(len(singles) + i, j) for i in range(64) for j in range(len(clips)))
    # one-detector sets: the per-class sweeps, count for count
    k = 0
    for det in KINDS:
        one = ParameterSweep(_cls(det), grids[det], tolerances=TOLS, settings=SETTINGS)
        got = one.run_clips([_open(f, fps, src, keep) for f, fps, _, src in clips], gts)
        g_n = len(grids[det])
        for s in range(len(SETTINGS)):
            for g in range(g_n):
                for j in range(len(clips)):
                    a, b = _counts(r, s * n + k + g, j), _counts(got, s * g_n + g, j)
                    assert a[0] == b[0] and a[2:] == b[2:], (det, s, g, j)
        tot = _totals(one)[0]
        mine = [(t.hard, t.hard_offset, t.fades) for t in sw.totals()]
        assert [mine[s * n + k + g] for s in range(len(SETTINGS)) for g in range(g_n)] == tot
        k += g_n
    for b in keep:
        b.close()


def test_member_overflow_names_the_detector(lib):
    from pyscenedetect_b200.detectors import ContentDetector, HistogramDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.test_gpu_sweep_clips import _render
    frames, _ = _render(120, 96, 54, seed=4)
    sw = ParameterSweep(detector_sets=[[ContentDetector(threshold=1.0, min_scene_len=0),
                                        HistogramDetector(threshold=0.01)]], max_cuts_per_cell=2, settings=SETTINGS)
    with pytest.raises(RuntimeError, match=r"detector (Content|Histogram)Detector\(.*\) of setting 0 \(\{\}\) found "
                                           r"\d+ cuts in clip 0, more than max_cuts_per_cell=2"):
        sw.run_clips([ArrayVideoStream(frames, 25)], [GroundTruth([])])
    assert sw.videos == 0
