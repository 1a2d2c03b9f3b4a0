#!/usr/bin/env python
"""Generate tests/golden/kernel_sizes_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout
given as the first argument) - ContentDetector and AdaptiveDetector with edge kernel sizes of 65 and above.

Run `python tests/golden/make_kernel_sizes_golden.py <reference checkout>`.  Two parts:

* `cases`: one ScenePlan video per (detector, frame size, kernel_size) through the reference's own `SceneManager`
  with a `StatsManager`: per-frame metrics as `float.hex`, the cut list, the scene list and the CSV's sha256
  (make_golden.run_case, the recipe of golden_v1/v2).
* `grid`: the scene list of each cell of a small kernel_size x threshold grid, one reference `SceneManager` per
  cell, as make_sweep_golden.py records its grids.
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

ALL = (1.0, 1.0, 1.0, 1.0)
EDGES = (0.0, 0.0, 0.0, 1.0)

# name, detector, gen(n, w, h, seed, min_len, max_len, noise_shift), kwargs, SceneManager scaling
CASES = [
    dict(name="content_k65_360p", det="content", gen=(60, 640, 360, 41, 8, 20, 30),
         kw=dict(kernel_size=65, weights=ALL, threshold=30.0), downscale=1),
    dict(name="content_k101_720p_edges", det="content", gen=(40, 1280, 720, 42, 6, 14, 30),
         kw=dict(kernel_size=101, weights=EDGES, threshold=20.0), downscale=1),
    dict(name="adaptive_k129_360p", det="adaptive", gen=(60, 640, 360, 43, 8, 20, 30),
         kw=dict(kernel_size=129, weights=ALL), downscale=1),
    # k > H
    dict(name="content_k255_180p", det="content", gen=(90, 320, 180, 44, 10, 30, 30),
         kw=dict(kernel_size=255, weights=ALL, threshold=30.0), downscale=1),
    # k > 2W - 1: every pixel's window covers the whole frame
    dict(name="content_k641_180p", det="content", gen=(90, 320, 180, 45, 10, 30, 30),
         kw=dict(kernel_size=641, weights=ALL, threshold=30.0), downscale=1),
    dict(name="content_k65_1080p_auto", det="content", gen=(24, 1920, 1080, 46, 4, 10, 30),
         kw=dict(kernel_size=65, weights=ALL, threshold=30.0), auto_downscale=True),
    # the automatic size 4 + round(sqrt(W H) / 192), made odd, is 65 here
    dict(name="content_auto_15360x8640", det="content", gen=(4, 15360, 8640, 47, 1, 2, 30),
         kw=dict(weights=ALL, threshold=30.0, min_scene_len=1), downscale=1),
]

GRID = dict(det="content", gen=(200, 320, 180, 48, 15, 50, 30), fps=30.0,
            cells=[dict(kernel_size=k, threshold=t, weights=ALL) for k in (5, 65, 129) for t in (20.0, 30.0, 40.0)])


def grid_cells():
    n, w, h, seed, mn, mx, ns = GRID["gen"]
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    frames = render_frames(plan.params, w, h)
    out = []
    for kw in GRID["cells"]:
        sm = SceneManager()
        sm.auto_downscale = False
        sm.add_detector(build_detector(GRID["det"], kw))
        sm.detect_scenes(SyntheticStream(frames, GRID["fps"]), show_progress=False)
        scenes = [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]
        out.append(dict(kw=kw, scene_list=scenes))
        print("grid", kw, scenes)
    return dict(GRID, true_cuts=plan.cut_frames, cells=out)


def main():
    cases = []
    for c in CASES:
        case = dict(c, mode="scene_manager", stats=True, fps=30.0)
        out = run_case(case)
        print(out["name"], "cuts", out["cuts"], "true", out["true_cuts"])
        cases.append(out)
    golden = {"reference_version": scenedetect.__version__, "cases": cases, "grid": grid_cells()}
    path = os.path.join(HERE, "kernel_sizes_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
