"""Host side of the parameter sweep (no GPU): the scorer model against the reference evaluator's recorded
results, the planner, the cell arguments against what `cuts_for_detector` passes to psd_cuts_*, and the
argument checks."""

import ctypes as C
import json
import os

import pytest

from tests import sweep_model

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "sweep_v1.json")) as f:
        return json.load(f)


def _check(preds, hard, fades, want):
    for tol, w in want.items():
        got_hard, got_fades = sweep_model.score(preds, hard, [tuple(f) for f in fades], int(tol))
        assert list(got_hard) == w["hard"], (tol, got_hard, w)
        assert list(got_fades) == w["fades"], (tol, got_fades, w)


def test_model_equals_reference_evaluator(golden):
    """The distance-outer walk the kernel implements equals evaluator.py's sort-based greedy matching."""
    assert len(golden["evaluator"]) >= 50
    for case in golden["evaluator"]:
        _check(case["preds"], case["hard"], case["fades"], case["want"])


def test_model_on_reference_scene_lists(golden):
    for g in golden["grids"]:
        for cell in g["cells"]:
            _check(cell["pred"], g["true_cuts"], g["fades"], cell["want"])
            if cell["pred"]:
                assert sweep_model.predicted_list(cell["pred"][:-1][::-1], cell["pred"][-1]) == cell["pred"]


def test_golden_covers_every_detector(golden):
    dets = {g["det"] for g in golden["grids"]}
    assert dets == {"content", "adaptive", "threshold", "histogram", "hash"}
    for g in golden["grids"]:
        assert 8 <= len(g["cells"]) <= 20
        assert any(c["pred"] for c in g["cells"]), g["det"]


def _grid(det):
    from pyscenedetect_b200.compat import FlashFilter
    from pyscenedetect_b200.detectors import ContentDetector, ThresholdDetector
    out = []
    for c in det["cells"]:
        kw = dict(c["kw"])
        if "weights" in kw:
            kw["weights"] = ContentDetector.Components(*kw["weights"])
        if "filter_mode" in kw:
            kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
        if "method" in kw:
            kw["method"] = ThresholdDetector.Method[kw["method"]]
        out.append(kw)
    return out


def _cls(name):
    from pyscenedetect_b200 import detectors as D
    return {"content": D.ContentDetector, "adaptive": D.AdaptiveDetector, "threshold": D.ThresholdDetector,
            "histogram": D.HistogramDetector, "hash": D.HashDetector}[name]


def test_planner_groups_keys_and_order():
    from pyscenedetect_b200._capi import F_EDGES, F_HASH, F_HSV
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector, HashDetector
    from pyscenedetect_b200.sweep import ParameterSweep
    grid = [dict(threshold=t, weights=w, kernel_size=k) for k in (None, 3, 5)
            for w in ((1, 1, 1, 0), (1, 1, 1, 1)) for t in (20.0, 30.0)]
    sw = ParameterSweep(ContentDetector, grid)
    # kernel_size only splits cells that use the edge component
    assert [(g.features, g.edge_kernel_size) for g in sw.groups] == [(F_HSV, 0), (F_HSV | F_EDGES, 0),
                                                                     (F_HSV | F_EDGES, 3), (F_HSV | F_EDGES, 5)]
    assert len(sw.metric_keys) == 4
    assert [sw.cells[k].metric for k in sw.order] == sorted((c.metric for c in sw.cells),
                                                            key=sw.metric_keys.index)
    assert sorted(sw.order) == list(range(len(grid))) and all(sw.order[sw.slot_of[k]] == k for k in range(len(grid)))

    h = ParameterSweep(HashDetector, [dict(size=s, threshold=t) for t in (0.3, 0.4) for s in (8, 16)])
    assert [(g.features, dict(g.engine_kwargs)["hash_size"]) for g in h.groups] == [(F_HASH, 8), (F_HASH, 16)]
    assert h.order == [0, 2, 1, 3]  # cells of one metric array are adjacent, grid order within it

    a = ParameterSweep(AdaptiveDetector, [dict(window_width=w, adaptive_threshold=t) for t in (2.0, 3.0)
                                          for w in (2, 3)] + [dict(luma_only=True)])
    assert len(a.groups) == 1
    kinds = [k[0] for k in a.metric_keys]
    assert kinds.count("content_val") == 2 and kinds.count("adaptive_ratio") == 3
    for c in a.cells:  # content_val is scanned before the ratio that reads it
        assert a.metric_keys.index(c.metric2) < a.metric_keys.index(c.metric)
    # warp ordering: the 32 cells of a warp read one array unless a key's run ends inside the warp
    big = ParameterSweep(ContentDetector, [dict(threshold=float(t), luma_only=bool(t % 2)) for t in range(128)])
    runs = [big.cells[k].metric for k in big.order]
    assert runs[:64] == [runs[0]] * 64 and runs[64:] == [runs[64]] * 64


class _Buf:
    def __init__(self, nbytes=8, device=0):
        self.ptr = 4096
        self.nbytes = nbytes


class _Rec:
    def __init__(self):
        self.calls = {}

    def __getattr__(self, name):
        def f(*args):
            self.calls[name] = args
            return 0
        return f


class _Eng:
    frame_count, n_pixels, hash_size, device, compute_stream = 100, 64, 8, 0, None

    def device_results(self):
        return 1, 2

    def device_hash(self):
        return 3

    def device_edge_sads(self):
        return None


@pytest.mark.parametrize("det", ["content", "adaptive", "threshold", "histogram", "hash"])
def test_cell_arguments_equal_device_cuts_launches(golden, monkeypatch, det):
    from pyscenedetect_b200 import device_cuts
    from pyscenedetect_b200.sweep import ParameterSweep
    monkeypatch.setattr(device_cuts, "DeviceBuffer", _Buf)
    g = next(x for x in golden["grids"] if x["det"] == det)
    grid = _grid(g)
    grid += [dict(grid[0], min_scene_len=m) for m in (0.5, "0.4s", "12", 1)]
    sw = ParameterSweep(_cls(det), grid)
    for fps in (30.0, 24000 / 1001, 25):
        for k, kw in enumerate(grid):
            rec = _Rec()
            dc = device_cuts.DeviceCuts.__new__(device_cuts.DeviceCuts)
            dc._e, dc._lib, dc._dev, dc._cap, dc._stream = _Eng(), rec, 0, 16, None
            dc._cuts = dc._count = _Buf()
            dc._fetch = lambda: []
            device_cuts.cuts_for_detector(dc, _cls(det)(**kw), fps, first_frame=0)
            c, calls = sw.cells[k], rec.calls
            mf = c.min_frames(fps)
            if det == "content":
                assert list(calls["psd_scan_content_edges"][4]) == [float(x) for x in c.metric[2]]
                assert calls["psd_scan_compare"][2] == c.threshold
                assert calls["psd_cuts_flash_filter"][3:5] == (mf, c.mode)
            elif det == "adaptive":
                assert list(calls["psd_scan_content_edges"][4]) == [float(x) for x in c.metric2[2]]
                assert calls["psd_scan_adaptive"][2:4] == (c.window, c.min_content_val) == c.metric[3:5]
                assert calls["psd_cuts_adaptive"][4:8] == (c.window, c.threshold, c.min_content_val, mf)
            elif det == "histogram":
                assert calls["psd_scan_hist_correl"][2] == c.metric[2]
                assert calls["psd_cuts_histogram"][3:5] == (c.threshold, mf)
            elif det == "hash":
                # the engine of the cell's pixel group hashes at the detector's size
                assert dict(sw.groups[c.metric[1]].engine_kwargs)["hash_size"] == kw.get("size", 8)
                assert calls["psd_cuts_hash"][3:5] == (c.threshold, mf)
            else:
                assert calls["psd_cuts_threshold"][3:8] == (c.threshold, c.mode, c.fade_bias, mf, c.add_final_scene)


def test_validation_errors():
    from pyscenedetect_b200.detectors import ContentDetector, HistogramDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    with pytest.raises(ValueError):
        GroundTruth(hard_cuts=[5, 5, 9])
    with pytest.raises(ValueError):
        GroundTruth(hard_cuts=[9, 5])
    assert GroundTruth([1, 2], fades=[(9, 4), (1, 3)]).fades == [(9, 4), (1, 3)]  # kept as given
    with pytest.raises(ValueError):
        ParameterSweep(ContentDetector, [])
    for tols in ((), (-1,), (1, 1), tuple(range(9))):
        with pytest.raises(ValueError):
            ParameterSweep(ContentDetector, [{}], tolerances=tols)
    with pytest.raises(ValueError):
        ParameterSweep(ContentDetector, [{}], max_cuts_per_cell=0)
    with pytest.raises(ValueError):  # the constructor's own validation
        ParameterSweep(ContentDetector, [dict(kernel_size=4)])
    with pytest.raises(ValueError):
        ParameterSweep(HistogramDetector, [dict(bins=300)])
    with pytest.raises(TypeError):
        ParameterSweep(ContentDetector, [dict(no_such_argument=1)])
    with pytest.raises(TypeError):
        ParameterSweep(object, [{}])
    sw = ParameterSweep(ContentDetector, [{}])
    with pytest.raises(ValueError):
        sw.run_scored([], 30.0)


def test_c_abi_rejects_bad_arguments_without_a_device():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    cells = (_capi.PsdSweepCell * 1)()
    cells[0].kind, cells[0].metric = 7, 4096
    assert lib.psd_sweep_cuts(cells, 1, 10, 0, 4096, 4096, 4, None) == _capi.PSD_ERR_INVALID
    assert b"unknown kind" in lib.psd_last_error()
    cells[0].kind, cells[0].window = _capi.SWEEP_ADAPTIVE, 0
    assert lib.psd_sweep_cuts(cells, 1, 10, 0, 4096, 4096, 4, None) == _capi.PSD_ERR_INVALID
    cells[0].kind, cells[0].mode = _capi.SWEEP_HASH, 1
    assert lib.psd_sweep_cuts(cells, 1, 10, 0, 4096, 4096, 4, None) == _capi.PSD_ERR_INVALID
    cells[0].kind, cells[0].mode, cells[0].metric = _capi.SWEEP_CONTENT, 0, None
    assert lib.psd_sweep_cuts(cells, 1, 10, 0, 4096, 4096, 4, None) == _capi.PSD_ERR_INVALID
    tols = (C.c_int32 * 9)(*range(9))
    args = [4096, 4096, 1, 4, 10, 4096, 1, None, 0]
    outs = [4096, 4096, 4096, None]
    assert lib.psd_sweep_eval(*args, tols, 9, 4096, 1 << 20, *outs) == _capi.PSD_ERR_INVALID
    assert lib.psd_sweep_eval(*args, tols, 0, 4096, 1 << 20, *outs) == _capi.PSD_ERR_INVALID
    neg = (C.c_int32 * 1)(-1)
    assert lib.psd_sweep_eval(*args, neg, 1, 4096, 1 << 20, *outs) == _capi.PSD_ERR_INVALID
    one = (C.c_int32 * 1)(1)
    assert lib.psd_sweep_eval(*args, one, 1, 4096, 4, *outs) == _capi.PSD_ERR_INVALID  # workspace too small
    assert b"workspace" in lib.psd_last_error()
