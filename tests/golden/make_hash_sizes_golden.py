#!/usr/bin/env python
"""Generate tests/golden/hash_sizes_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout
given as the first argument) - HashDetector at sizes above 16 and hash images above 64x64.

Run `python tests/golden/make_hash_sizes_golden.py <reference checkout>`.  Two parts:

* `cases`: one ScenePlan video per (size, lowpass) through the reference's own `SceneManager` with a
  `StatsManager`: per-frame hash_dist as `float.hex`, the cut list, the scene list and the CSV's sha256
  (make_golden.run_case, the recipe of golden_v1/v2).
* `grid`: the scene list of each cell of a small size x threshold x min_scene_len grid, one reference
  `SceneManager` per cell, as make_sweep_golden.py records its grids.
"""

from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import SyntheticStream, build_detector, run_case  # noqa: E402  (puts the checkout on sys.path)

import scenedetect  # noqa: E402
from scenedetect.scene_manager import SceneManager  # noqa: E402

from pyscenedetect_b200.synth import ScenePlan, render_frames  # noqa: E402

# name, gen(n, w, h, seed, min_len, max_len, noise_shift), HashDetector kwargs, SceneManager scaling
CASES = [
    # the CLI help's example: 1080p auto-downscaled to 274x154, n = 96 (non-integer area scales)
    dict(name="hash_32_3_1080p_auto", gen=(40, 1920, 1080, 21, 6, 14, 30), kw=dict(size=32, lowpass=3),
         auto_downscale=True),
    # n = 17: odd, no folding; 289 bits = 5 words
    dict(name="hash_17_1_360p", gen=(90, 640, 360, 22, 10, 30, 30), kw=dict(size=17, lowpass=1, threshold=0.3),
         downscale=1),
    dict(name="hash_24_4_720p", gen=(60, 1280, 720, 23, 8, 20, 30), kw=dict(size=24, lowpass=4), downscale=1),
    # n = 128
    dict(name="hash_64_2_360p", gen=(90, 640, 360, 24, 10, 30, 30), kw=dict(size=64, lowpass=2, threshold=0.3),
         downscale=1),
    # m = 65 536 low-band values, 1 024 words
    dict(name="hash_256_1_270p", gen=(60, 480, 270, 25, 8, 20, 30), kw=dict(size=256, lowpass=1, threshold=0.3),
         downscale=1),
    # n = 1 000
    dict(name="hash_100_10_1080p", gen=(24, 1920, 1080, 26, 4, 10, 30), kw=dict(size=100, lowpass=10),
         downscale=1),
    # n = 1 080 = H: an identity vertical scale
    dict(name="hash_30_36_1080p", gen=(24, 1920, 1080, 27, 4, 10, 30), kw=dict(size=30, lowpass=36),
         downscale=1),
]

GRID = dict(gen=(200, 320, 180, 28, 15, 50, 30), fps=30.0,
            cells=[dict(size=s, threshold=t, min_scene_len=m) for s in (8, 16, 32) for t in (0.2, 0.3, 0.4)
                   for m in (0, 15)])


def grid_cells():
    n, w, h, seed, mn, mx, ns = GRID["gen"]
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    frames = render_frames(plan.params, w, h)
    out = []
    for kw in GRID["cells"]:
        sm = SceneManager()
        sm.auto_downscale = False
        sm.add_detector(build_detector("hash", kw))
        sm.detect_scenes(SyntheticStream(frames, GRID["fps"]), show_progress=False)
        scenes = [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]
        out.append(dict(kw=kw, scene_list=scenes))
        print("grid", kw, scenes)
    return dict(GRID, true_cuts=plan.cut_frames, cells=out)


def main():
    cases = []
    for c in CASES:
        case = dict(c, det="hash", mode="scene_manager", stats=True, fps=30.0)
        out = run_case(case)
        print(out["name"], "cuts", out["cuts"], "true", out["true_cuts"])
        cases.append(out)
    golden = {"reference_version": scenedetect.__version__, "cases": cases, "grid": grid_cells()}
    path = os.path.join(HERE, "hash_sizes_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
