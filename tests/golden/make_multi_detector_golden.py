#!/usr/bin/env python
"""Generate tests/golden/multi_detector_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout
given as the first argument): several detectors in one reference `SceneManager`.

Run `python tests/golden/make_multi_detector_golden.py <reference checkout>`.  Each case stores the cut list and the
scene list; with a `StatsManager`, also the per-frame metrics (`float.hex`) and the CSV's sha256.  In this package
the detectors of one SceneManager share one fused score pass, whose feature mask is the union of what they need,
so together the cases run masks 5, 6, 11, 13 and 15 and a hash launch next to the fused pass:

* Content + Threshold, with stats: a ContentDetector with a StatsManager computes edges (mask 11);
* Content + Histogram, without stats, at 133x99 (P mod 16 = 15; mask 5);
* Threshold + Histogram, with stats (mask 6);
* Adaptive (edges) + Histogram + Threshold + Hash, with stats, 640x360 auto-downscaled (mask 15 + the hash);
* Content (edges) + Adaptive with the same kernel_size + Histogram, with stats: both write `content_val` (mask 13).
"""

from __future__ import annotations

import hashlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import SyntheticStream, build_detector, hexify  # noqa: E402  (puts the checkout on sys.path)

import scenedetect  # noqa: E402
from scenedetect.common import FrameTimecode  # noqa: E402
from scenedetect.scene_manager import SceneManager  # noqa: E402
from scenedetect.stats_manager import StatsManager  # noqa: E402

from pyscenedetect_b200.synth import ScenePlan, render_frames  # noqa: E402

ALL = (1.0, 1.0, 1.0, 1.0)

# name, gen(n, w, h, seed, min_len, max_len, noise_shift), detectors [(name, kwargs)], stats, scaling
CASES = [
    dict(name="content_threshold_stats", gen=(200, 160, 90, 51, 15, 50, 30),
         dets=[("content", {}), ("threshold", dict(threshold=20))], stats=True, downscale=1),
    dict(name="content_histogram_133x99", gen=(180, 133, 99, 52, 15, 50, 30),
         dets=[("content", dict(threshold=25.0)), ("histogram", dict(bins=64, threshold=0.1))], stats=False,
         downscale=1),
    dict(name="threshold_histogram_stats", gen=(200, 160, 90, 53, 15, 50, 30),
         dets=[("threshold", dict(threshold=30, add_final_scene=True)), ("histogram", {})], stats=True, downscale=1),
    dict(name="adaptive_hist_threshold_hash_360p", gen=(150, 640, 360, 54, 15, 50, 30),
         dets=[("adaptive", dict(window_width=3, weights=ALL)), ("histogram", dict(bins=256, threshold=0.05)),
               ("threshold", {}), ("hash", {})], stats=True, auto_downscale=True),
    dict(name="content_adaptive_shared_kernel", gen=(180, 192, 108, 55, 15, 50, 30),
         dets=[("content", dict(weights=ALL, kernel_size=5, threshold=30.0)),
               ("adaptive", dict(weights=ALL, kernel_size=5)), ("histogram", dict(bins=128))], stats=True,
         downscale=1),
]


def run_case(case: dict) -> dict:
    n, w, h, seed, mn, mx, ns = case["gen"]
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    frames = render_frames(plan.params, w, h)
    fps = 30.0
    out = dict(case, fps=fps)
    out["frames_sha256"] = hashlib.sha256(frames.tobytes()).hexdigest()
    out["true_cuts"] = plan.cut_frames
    stats = StatsManager() if case["stats"] else None
    sm = SceneManager(stats)
    for name, kw in case["dets"]:
        sm.add_detector(build_detector(name, kw))
    if case.get("auto_downscale"):
        sm.auto_downscale = True
    else:
        sm.auto_downscale = False
        sm.downscale = case.get("downscale", 1)
    sm.detect_scenes(SyntheticStream(frames, fps), show_progress=False)
    out["cuts"] = [c.frame_num for c in sm.get_cut_list()]
    out["scene_list"] = [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]
    if stats is not None:
        keys = sorted(stats.metric_keys)
        rows = {}
        for t in range(n):
            vals = stats.get_metrics(FrameTimecode(t, fps), keys)
            if any(v is not None for v in vals):
                rows[str(t)] = [hexify(v) for v in vals]
        out["metric_keys"] = keys
        out["metrics"] = rows
        buf = io.StringIO()
        stats.save_to_csv(buf)
        out["csv_sha256"] = hashlib.sha256(buf.getvalue().encode()).hexdigest()
        out["csv_head"] = buf.getvalue().splitlines()[:4]
    return out


def main():
    cases = []
    for c in CASES:
        out = run_case(c)
        print(out["name"], "cuts", out["cuts"], "true", out["true_cuts"])
        cases.append(out)
    golden = {"reference_version": scenedetect.__version__, "cases": cases}
    path = os.path.join(HERE, "multi_detector_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
