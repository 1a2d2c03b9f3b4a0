"""The oracle's detectors (oracle/ref_detectors.py, which bench.py's parity check trusts) against PySceneDetect
0.7.1 on the scripted sequences of tests/automata_inputs.py: every per-frame metric bit for bit and every
parameter set's cut list, as recorded in tests/golden/automata_v1.json.gz by make_automata_golden.py.

The oracle is driven through the same two overrides the recording used: its `mean_pixel_distance` returns
the scripted SAD / pixel count of the current frame's component and its `hash_frame` the scripted bits;
ThresholdDetector and HistogramDetector get real frames built from the scripted byte sum and Y histogram."""

import ast
import collections

import numpy as np
import pytest

from oracle import ref_detectors as R
from tests import automata_inputs as A

SPECS = A.sequences()


def test_recording_covers_every_sequence():
    rec = A.recording()
    assert sorted(rec) == sorted(s["name"] for s in SPECS)
    for det in ("content", "adaptive", "threshold", "histogram", "hash"):
        mine = [rec[s["name"]] for s in SPECS if s["det"] == det]
        assert len(mine) >= 30 and sum(len(r["runs"]) for r in mine) >= 500, det
        assert sum(len(run["cuts"]) for r in mine for run in r["runs"]) > 1000, det


_PENDING: collections.deque = collections.deque()


def _scripted_distance(left, right):
    return _PENDING.popleft()


class _Scripted:
    """Routes the oracle's pixel-distance and hash steps to the scripted inputs while a test runs.  The
    oracle's histogram of each (frame, bins) is computed once, by its own `calculate_histogram` on the real
    gray frame, and reused by every parameter set (a 7680x4320 frame is 100 MB)."""

    def __init__(self, monkeypatch, spec, inp):
        self.spec, self.inp = spec, inp
        self._hists: dict = {}
        self._calc = R.calculate_histogram
        monkeypatch.setattr(R, "mean_pixel_distance", _scripted_distance)
        monkeypatch.setattr(R, "hash_frame", self._hash)
        monkeypatch.setattr(R, "calculate_histogram", self._histogram)

    def _hash(self, frame_img, hash_size, factor):
        assert hash_size == self.inp.hash_size
        return A.hash_bits(self.inp.hashes[A.frame_index(frame_img)], hash_size)

    def _histogram(self, frame_img, bins=256, normalize=True):
        key = (A.frame_index(frame_img), bins, normalize)
        if key not in self._hists:
            frame = A.gray_frame(self.inp.yhist[key[0]], self.spec["shape"])
            self._hists[key] = self._calc(frame, bins=bins, normalize=normalize)
        return self._hists[key].copy()


def make_oracle(spec, kw):
    det, fps = spec["det"], spec["fps"]
    if det == "content":
        return R.RefContentDetector(threshold=kw["threshold"], min_scene_len=kw["min_scene_len"],
                                    weights=tuple(kw["weights"]), fps=fps, with_stats=True,
                                    filter_mode=R.RefFlashFilter.SUPPRESS if kw["filter_mode"] == "SUPPRESS"
                                    else R.RefFlashFilter.MERGE)
    if det == "adaptive":
        return R.RefAdaptiveDetector(adaptive_threshold=kw["adaptive_threshold"], min_scene_len=kw["min_scene_len"],
                                     window_width=kw["window_width"], min_content_val=kw["min_content_val"],
                                     weights=tuple(kw["weights"]), fps=fps, with_stats=True)
    if det == "threshold":
        return R.RefThresholdDetector(threshold=kw["threshold"], min_scene_len=kw["min_scene_len"],
                                      fade_bias=kw["fade_bias"], add_final_scene=kw["add_final_scene"],
                                      method=R.RefThresholdDetector.CEILING if kw["method"] == "CEILING"
                                      else R.RefThresholdDetector.FLOOR, fps=fps, with_stats=True)
    if det == "histogram":
        return R.RefHistogramDetector(threshold=kw["threshold"], bins=kw["bins"], min_scene_len=kw["min_scene_len"],
                                      fps=fps, with_stats=True)
    return R.RefHashDetector(threshold=kw["threshold"], size=spec["size"], lowpass=2,
                             min_scene_len=kw["min_scene_len"], fps=fps, with_stats=True)


def run_oracle(spec, inp, kw, frames):
    """-> (sorted unique cuts, per-frame scores (content / adaptive), the detector)."""
    det = make_oracle(spec, kw)
    first, n = spec["first_frame"], spec["n"]
    cuts, scores = [], []
    for i in range(n):
        _PENDING.clear()
        if spec["det"] in ("content", "adaptive") and i > 0:
            _PENDING.extend(A.components(inp, i))
        cuts += det.process_frame(first + i, frames(i))
        assert not _PENDING
        if spec["det"] in ("content", "adaptive"):
            scores.append(det._frame_score)
    if n:
        cuts += det.post_process(first + n - 1)
    return sorted(set(cuts)), scores, det


def _frames(spec, inp):
    if spec["det"] == "histogram":
        return A.index_frame  # the real frame is built by _Scripted._histogram, once per (frame, bins)
    cache = [A.frame_source(spec, inp, i) for i in range(spec["n"])]
    return cache.__getitem__


def _hex(vals):
    return [None if v is None else float(v).hex() for v in vals]


def oracle_metric(spec, inp, key, frames):
    """The oracle's per-frame values of one recorded metric key."""
    name, *params = key.split("|")
    params = [ast.literal_eval(p) for p in params]
    first, n = spec["first_frame"], spec["n"]
    at = lambda det, k: [det.metrics.get(first + i, {}).get(k) for i in range(n)]  # noqa: E731
    if name == "content_val" or name.startswith("delta_"):
        w = params[0] if params else spec["weights"][0]
        kw = (dict(weights=w, threshold=255.0, min_scene_len=0, filter_mode="MERGE") if spec["det"] == "content" else
              dict(weights=w, window_width=2, min_content_val=15.0, adaptive_threshold=3.0, min_scene_len=0))
        _, scores, det = run_oracle(spec, inp, kw, frames)
        return scores if name == "content_val" else at(det, name)
    if name == "adaptive_ratio":
        w, win, mcv = params
        det = run_oracle(spec, inp, dict(weights=w, window_width=win, min_content_val=mcv, adaptive_threshold=3.0,
                                         min_scene_len=0), frames)[2]
        return at(det, det.ratio_key)
    if name == "average_rgb":
        return at(run_oracle(spec, inp, dict(threshold=spec["T"], min_scene_len=0, fade_bias=0.0,
                                             add_final_scene=False, method="FLOOR"), frames)[2], name)
    if name == "hist_diff":
        det = run_oracle(spec, inp, dict(threshold=0.0, bins=params[0], min_scene_len=0), frames)[2]
        return at(det, det.metric_key)
    det = run_oracle(spec, inp, dict(threshold=1.0, min_scene_len=0), frames)[2]
    return at(det, det.metric_key)


@pytest.mark.parametrize("name", [s["name"] for s in SPECS])
def test_oracle_matches_reference(monkeypatch, name):
    spec = next(s for s in SPECS if s["name"] == name)
    rec, inp = A.recorded(spec)
    _Scripted(monkeypatch, spec, inp)
    frames = _frames(spec, inp)
    for key, want in rec["metrics"].items():
        assert _hex(oracle_metric(spec, inp, key, frames)) == want, key
    for run in rec["runs"]:
        got, _, _ = run_oracle(spec, inp, run["kw"], frames)
        assert got == run["cuts"], run["kw"]


def test_scripted_inputs_are_engine_results():
    """What every sequence holds could come out of the engine's score pass."""
    for spec in SPECS:
        inp = A.build(spec)
        s, P = inp.sums, inp.n_pixels
        assert s.shape[0] == spec["n"]
        assert np.array_equal(s["has_prev"], (np.arange(spec["n"]) > 0).astype(np.uint64)), spec["name"]
        assert (s["sad_hue"] <= 179 * P).all() and (s["sad_sat"] <= 255 * P).all(), spec["name"]
        assert (s["sad_lum"] <= 255 * P).all() and (s["bgr_sum"] <= 765 * P).all(), spec["name"]
        assert (s["sad_edges"] <= 255 * P).all(), spec["name"]
        if spec["det"] in ("content", "adaptive") and not all(w[3] > 0 for w in spec["weights"]):
            assert not s["sad_edges"].any(), spec["name"]
        if inp.yhist is not None:
            assert (inp.yhist.astype(np.int64).sum(axis=1) == P).all(), spec["name"]
        if inp.hashes is not None:
            nb = inp.hash_size ** 2
            for w in range(A.HASH_WORDS):
                lo = 64 * w
                valid = 0 if nb <= lo else (~np.uint64(0) if nb >= lo + 64 else (np.uint64(1) << np.uint64(nb - lo)) - np.uint64(1))
                assert not (inp.hashes[:, w] & ~np.uint64(valid)).any(), spec["name"]
