#!/usr/bin/env python
"""Generate tests/golden/automata_v1.json.gz: what the real PySceneDetect 0.7.1 (imported from the source checkout
given as the first argument) computes from the scripted integer results of tests/automata_inputs.py - per-frame
metrics as `float.hex` strings and the cut list of every parameter set.

    python tests/golden/make_automata_golden.py <path of a PySceneDetect 0.7.1 source checkout>

The reference computes everything it can from the inputs itself.  ThresholdDetector gets real frames whose byte
sum is the scripted one and HistogramDetector real gray frames with the scripted Y histogram.  ContentDetector
and AdaptiveDetector get 1x1 frames and a `_mean_pixel_distance` that returns the scripted SAD / pixel count of
the current frame's component; HashDetector gets a `hash_frame` that returns the scripted bits.  Weighting,
FlashFilter, rolling window, ratio, fades, calcHist / normalize / compareHist, Hamming distance and every cut rule
are the reference's own.  Parameter sets are chosen from the reference's own metric values (exact ties and their
floating-point neighbours).  The output is deterministic: running the script twice gives the same bytes.
"""

from __future__ import annotations

import collections
import gzip
import itertools
import json
import math
import os
import random
import sys
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.abspath(sys.argv[1]))
sys.path.insert(0, ROOT)  # ahead of the reference, which has a `tests` package of its own

import numpy as np  # noqa: E402
import scenedetect  # noqa: E402
from scenedetect.common import FrameTimecode  # noqa: E402
from scenedetect.detector import FlashFilter  # noqa: E402
from scenedetect.detectors import (  # noqa: E402
    AdaptiveDetector,
    ContentDetector,
    HashDetector,
    HistogramDetector,
    ThresholdDetector,
)
from scenedetect.detectors import content_detector as _content_mod  # noqa: E402
from scenedetect.stats_manager import StatsManager  # noqa: E402

from tests import automata_inputs as A  # noqa: E402

# the current frame's four scripted components, consumed in the order ContentDetector asks for them
_PENDING: collections.deque = collections.deque()
_HASH_INPUT: dict = {}


def _scripted_distance(left, right):
    return _PENDING.popleft()


def _scripted_hash(frame_img, hash_size, factor):
    inp = _HASH_INPUT["inp"]
    assert hash_size == inp.hash_size
    return A.hash_bits(inp.hashes[A.frame_index(frame_img)], hash_size)


_content_mod._mean_pixel_distance = _scripted_distance
HashDetector.hash_frame = staticmethod(_scripted_hash)


def make_detector(det: str, kw: dict, spec: dict):
    kw = dict(kw)
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    if "filter_mode" in kw:
        kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
    if "method" in kw:
        kw["method"] = ThresholdDetector.Method[kw["method"]]
    if det == "hash":
        kw.update(size=spec["size"], lowpass=2)
    cls = {"content": ContentDetector, "adaptive": AdaptiveDetector, "threshold": ThresholdDetector,
           "histogram": HistogramDetector, "hash": HashDetector}[det]
    return cls(**kw)


def run(spec, inp, kw):
    """One reference detector over the sequence: (sorted unique cuts, {stats key: [value or None]}, scores)."""
    det = make_detector(spec["det"], kw, spec)
    sm = StatsManager()
    det.stats_manager = sm
    sm.register_metrics(det.get_metrics())
    fps, first, n = spec["fps"], spec["first_frame"], spec["n"]
    _HASH_INPUT["inp"] = inp
    cuts, scores = [], []
    for i in range(n):
        _PENDING.clear()
        if spec["det"] in ("content", "adaptive") and i > 0:
            _PENDING.extend(A.components(inp, i))
        cuts += det.process_frame(FrameTimecode(first + i, fps), A.frame_source(spec, inp, i))
        assert not _PENDING, "ContentDetector asked for fewer components than scripted"
        if spec["det"] in ("content", "adaptive"):
            scores.append(det._frame_score)
    if n:
        cuts += det.post_process(FrameTimecode(first + n - 1, fps))
    keys = det.get_metrics()
    stats = {k: [] for k in keys}
    for i in range(n):
        vals = sm.get_metrics(FrameTimecode(first + i, fps), keys)
        for k, v in zip(keys, vals):
            stats[k].append(v)
    return sorted({c.frame_num for c in cuts}), stats, scores


def hexes(vals):
    return [None if v is None else float(v).hex() for v in vals]


def msl_forms(det: str, m: int) -> list:
    if det in ("content", "adaptive"):
        return [0, 1, m, 0.5, "0.6s", "00:00:00.700", "20"]
    return [0, 1, 3, 0.25, "0.3s", "00:00:00.200", "4"]


def neighbours(v: float) -> list[float]:
    return [math.nextafter(v, -math.inf), v, math.nextafter(v, math.inf)]


def hist_bound_ok(bound: float, corr: list[float]) -> bool:
    """Cut decisions at `bound` are exact on the device: every correlation lies more than 1e-9 away from it,
    except exact 1.0 against a bound of 1.0 (identical or degenerate histograms, exact on both sides)."""
    return all((c == 1.0 and bound == 1.0) or abs(c - bound) > 1e-9 for c in corr)


def record(spec) -> dict:
    rng = random.Random(zlib.crc32(("params|" + spec["name"]).encode()))
    inp = A.build(spec)
    det, n = spec["det"], spec["n"]
    assert inp.sums.shape[0] == n
    metrics: dict = {}
    runs: list[dict] = []
    forms = msl_forms(det, spec.get("m", 3))

    def put(key, vals):
        h = hexes(vals)
        assert metrics.setdefault(key, h) == h, key

    if det in ("content", "adaptive"):
        vals_of = {}
        for w in spec["weights"]:
            _, stats, scores = run(spec, inp, dict(weights=w, threshold=255.0, min_scene_len=0) if det == "content"
                                   else dict(weights=w, min_scene_len=0))
            put(A.metric_key("content_val", w), scores)
            for c in ("delta_hue", "delta_sat", "delta_lum", "delta_edges"):
                put(A.metric_key(c), stats[c])
            vals_of[tuple(w)] = scores
    if det == "content":
        grid = []
        for w in spec["weights"]:
            above = sorted({v for v in vals_of[tuple(w)][1:] if v >= 20.0})
            picks = sorted(set(rng.sample(above, min(2, len(above))) + above[:1])) if above else \
                vals_of[tuple(w)][-1:]
            thresholds = sorted({t for v in picks for t in neighbours(v)} | {27.0})
            for t in thresholds:
                grid += [dict(weights=w, threshold=t, min_scene_len=spec["m"], filter_mode=mode)
                         for mode in ("MERGE", "SUPPRESS")]
            rest = list(itertools.product(thresholds, forms, ("MERGE", "SUPPRESS")))
            grid += [dict(weights=w, threshold=t, min_scene_len=f, filter_mode=mode)
                     for t, f, mode in rng.sample(rest, min(10, len(rest)))]
    elif det == "adaptive":
        grid = []
        for w in spec["weights"]:
            nz = sorted({v for v in vals_of[tuple(w)] if v > 0.0})
            v = rng.choice(nz) if nz else 15.0
            for win in (1, 2, 5):
                for mcv in sorted({15.0, v, math.nextafter(v, math.inf)}):
                    _, stats, _ = run(spec, inp, dict(weights=w, window_width=win, min_content_val=mcv,
                                                      adaptive_threshold=3.0, min_scene_len=0))
                    ratio = next(x for k, x in stats.items() if k.startswith("adaptive_ratio"))
                    put(A.metric_key("adaptive_ratio", w, win, mcv), ratio)
                    finite = sorted({r for r in ratio if r is not None and r > 0.0})
                    thr = sorted(set(rng.sample(finite, min(2, len(finite)))) | {3.0, 255.0})
                    for t in thr:
                        grid.append(dict(weights=w, window_width=win, min_content_val=mcv, adaptive_threshold=t,
                                         min_scene_len=forms[len(grid) % len(forms)]))
    elif det == "threshold":
        _, stats, _ = run(spec, inp, dict(threshold=spec["T"]))
        put(A.metric_key("average_rgb"), stats["average_rgb"])
        T = spec["T"]
        grid = [dict(threshold=T, method=meth, fade_bias=b, add_final_scene=afs, min_scene_len=forms[k % len(forms)])
                for k, (meth, b, afs) in enumerate(itertools.product(("FLOOR", "CEILING"), A.FADE_BIASES,
                                                                     (False, True)))]
        rest = list(itertools.product(sorted({max(0, T - 1), T + 1}), ("FLOOR", "CEILING"), A.FADE_BIASES,
                                      (False, True), forms))
        grid += [dict(threshold=t, method=meth, fade_bias=b, add_final_scene=afs, min_scene_len=f)
                 for t, meth, b, afs, f in rng.sample(rest, 16)]
    elif det == "histogram":
        grid = []
        for bins in ((1, 2, 128, 256) if spec.get("uhd8k") else A.HIST_BINS):
            _, stats, _ = run(spec, inp, dict(bins=bins, threshold=0.0))
            corr = stats[f"hist_diff [bins={bins}]"]
            put(A.metric_key("hist_diff", bins), corr)
            c = sorted({x for x in corr if x is not None})
            cands = [(a + b) / 2.0 for a, b in zip(c, c[1:]) if b - a > 4e-9]
            thresholds = [0.0] + [1.0 - x for x in rng.sample(cands, min(2, len(cands)))]
            for t in thresholds:
                if hist_bound_ok(max(0.0, min(1.0, 1.0 - t)), c):
                    grid.append(dict(bins=bins, threshold=t, min_scene_len=forms[len(grid) % len(forms)]))
    else:
        _, stats, _ = run(spec, inp, dict(threshold=1.0))
        dist = next(iter(stats.values()))
        put(A.metric_key("hash_dist"), dist)
        seen = sorted({d for d in dist if d is not None and d > 0.0})
        picks = rng.sample(seen, min(3, len(seen)))
        thresholds = sorted({0.35} | set(picks) | set(neighbours(picks[0]) if picks else []))
        grid = [dict(threshold=t, min_scene_len=f) for t in thresholds for f in rng.sample(forms, 3)]
    for kw in grid:
        try:
            cuts, _, _ = run(spec, inp, kw)
        except ValueError:  # fade_bias < -1 can put a cut before frame 0, which a FrameTimecode cannot hold
            assert det == "threshold" and kw["fade_bias"] < -1.0, kw
            continue
        runs.append(dict(kw=kw, cuts=cuts))
    return dict(spec=spec, sha256=inp.sha256(), metrics=metrics, runs=runs)


def main():
    seqs = [record(s) for s in A.sequences()]
    doc = {"reference_version": scenedetect.__version__, "sequences": seqs}
    path = os.path.join(HERE, "automata_v1.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps(doc, separators=(",", ":"), sort_keys=True).encode())
    for det in ("content", "adaptive", "threshold", "histogram", "hash"):
        mine = [s for s in seqs if s["spec"]["det"] == det]
        print(det, len(mine), "sequences", sum(len(s["runs"]) for s in mine), "parameter sets",
              sum(len(r["cuts"]) for s in mine for r in s["runs"]), "cuts")
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
