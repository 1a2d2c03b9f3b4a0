#!/usr/bin/env python
"""Generate tests/golden/sweep_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout
given as the first argument, including its benchmark/ directory) - the data the sweep tests compare with.

Run `python tests/golden/make_sweep_golden.py <reference checkout>`.  Two parts:

* `evaluator`: benchmark/evaluator.py `score_video` at tolerances 0, 1 and 5 for seeded random and
  adversarial (predictions, ground truth) cases: ties at equal distance on both sides of a prediction,
  runs of predictions closer together than the tolerance, predictions inside fade intervals (two in one
  interval), overlapping and repeated intervals, empty predictions or ground truth.  Every prediction list
  has the shape benchmark/sweep.py:169 records (strictly increasing cuts, then the end position).
* `grids`: per-cell predicted lists (`[scene[1].frame_num for scene in sm.get_scene_list()]`,
  benchmark/sweep.py:169) of the reference SceneManager with default settings, for a small grid of every
  detector over the synthetic sequences golden_v1.json uses, plus `score_video` of each list against the
  sequence's true cuts and one fade interval.
"""

from __future__ import annotations

import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, HERE)
sys.path.insert(0, REF)

from make_golden import SyntheticStream, build_detector  # noqa: E402  (puts the checkout on sys.path)

import scenedetect  # noqa: E402
from benchmark.evaluator import EventInterval, GroundTruth, score_video  # noqa: E402
from scenedetect.scene_manager import SceneManager  # noqa: E402

from pyscenedetect_b200.synth import ScenePlan, render_frames  # noqa: E402

TOLERANCES = (0, 1, 5)


def ref_score(preds, hard, fades):
    gt = GroundTruth(hard_cuts=list(hard), fades=[EventInterval(a, b) for a, b in fades])
    out = {}
    for tol in TOLERANCES:
        v = score_video(list(preds), gt, tol, 0.0)
        out[str(tol)] = {"hard": [v.hard_cuts.matched, v.hard_cuts.false_positives, v.hard_cuts.missed,
                                  int(v.hard_offset[0]), v.hard_offset[1]],
                         "fades": [v.fades.matched, v.fades.false_positives, v.fades.missed]}
    return out


ADVERSARIAL = [
    # name, predictions, hard cuts, fades
    ("tie_both_sides", [12, 100], [10, 14], []),
    ("tie_chain", [11, 13, 200], [10, 12, 14], []),
    ("run_closer_than_tol", [20, 21, 22, 23, 24, 300], [21, 25], []),
    ("two_in_one_fade", [31, 35, 50, 400], [50], [(30, 40)]),
    ("overlapping_fades", [16, 25, 31, 100], [31], [(10, 20), (15, 30), (15, 30)]),
    ("fade_consumes_exact_hit", [10, 50], [10, 50], [(8, 12)]),
    ("repeated_interval", [6, 7, 100], [6], [(5, 8), (5, 8)]),
    ("end_inside_fade", [3, 9], [3], [(8, 20)]),
    ("empty_predictions", [], [5, 10], [(1, 3)]),
    ("empty_ground_truth", [5, 9, 20], [], []),
    ("all_empty", [], [], []),
    ("one_cut", [6, 7], [5, 6, 7, 8], []),
    ("dense_both", list(range(0, 40, 2)) + [41], list(range(1, 40, 3)), [(18, 19)]),
]


def evaluator_cases():
    cases = []
    for name, preds, hard, fades in ADVERSARIAL:
        cases.append(dict(name=name, preds=preds, hard=hard, fades=[list(f) for f in fades],
                          want=ref_score(preds, hard, fades)))
    rng = random.Random(20261015)
    for i in range(40):
        span = rng.choice([30, 100, 400])
        preds = sorted(rng.sample(range(span), rng.randint(0, min(40, span // 2))))
        if preds:
            preds.append(preds[-1] + rng.randint(1, 10))  # the end position
        hard = sorted(rng.sample(range(span), rng.randint(0, min(40, span // 2))))
        fades = []
        for _ in range(rng.randint(0, 4)):
            a = rng.randrange(span)
            fades.append([a, a + rng.randint(0, 12)])
        cases.append(dict(name=f"random_{i}", preds=preds, hard=hard, fades=fades,
                          want=ref_score(preds, hard, [tuple(f) for f in fades])))
    return cases


GRIDS = [
    dict(det="content", gen=(260, 160, 90, 0, 20, 70, 30), fps=30.0, fades=[[100, 110]],
         cells=[dict(threshold=t, min_scene_len=m) for t in (15.0, 27.0, 40.0) for m in (0, 15, 30)]
         + [dict(threshold=27.0, min_scene_len=m, filter_mode="SUPPRESS") for m in (15, 30)]
         + [dict(weights=(1.0, 1.0, 1.0, 1.0), kernel_size=k, threshold=30.0) for k in (3, 5)]
         + [dict(luma_only=True, threshold=15.0)]),
    dict(det="adaptive", gen=(260, 160, 90, 0, 20, 70, 30), fps=30.0, fades=[[100, 110]],
         cells=[dict(adaptive_threshold=t, window_width=w, min_scene_len=m)
                for t in (2.0, 3.0) for w in (2, 3) for m in (0, 15)]
         + [dict(min_content_val=8.0, window_width=w) for w in (2, 4)]
         + [dict(luma_only=True, adaptive_threshold=2.0), dict(weights=(1.0, 1.0, 1.0, 1.0), kernel_size=3)]),
    dict(det="threshold", gen=(300, 160, 90, 7, 20, 70, 30), fps=30.0, fades=[[60, 80]],
         cells=[dict(threshold=t, add_final_scene=a, min_scene_len=5) for t in (20, 60, 140) for a in (False, True)]
         + [dict(threshold=t, method="CEILING", add_final_scene=a, min_scene_len=5)
            for t in (100, 140) for a in (False, True)]
         + [dict(threshold=140, fade_bias=b, min_scene_len=5) for b in (-0.5, 0.5)]),
    dict(det="histogram", gen=(260, 160, 90, 10, 20, 70, 30), fps=30.0, fades=[[100, 110]],
         cells=[dict(threshold=t, bins=b, min_scene_len=m) for t in (0.05, 0.1, 0.2) for b in (128, 256)
                for m in (0, 15)]),
    dict(det="hash", gen=(260, 160, 90, 0, 20, 70, 30), fps=30.0, fades=[[100, 110]],
         cells=[dict(threshold=t, size=s, min_scene_len=m) for t in (0.25, 0.35) for s in (8, 16) for m in (0, 15)]
         + [dict(threshold=0.45, size=s) for s in (8, 16)]),
]


def grid_cases():
    out = []
    for g in GRIDS:
        n, w, h, seed, mn, mx, ns = g["gen"]
        plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
        frames = render_frames(plan.params, w, h)
        cells = []
        for kw in g["cells"]:
            sm = SceneManager()
            sm.add_detector(build_detector(g["det"], kw))
            sm.detect_scenes(SyntheticStream(frames, g["fps"]), show_progress=False)
            pred = [scene[1].frame_num for scene in sm.get_scene_list()]
            cells.append(dict(kw=kw, pred=pred, want=ref_score(pred, plan.cut_frames, [tuple(f) for f in g["fades"]])))
            print(g["det"], kw, pred)
        out.append(dict(det=g["det"], gen=list(g["gen"]), fps=g["fps"], true_cuts=plan.cut_frames,
                        fades=g["fades"], cells=cells))
    return out


def main():
    golden = {"reference_version": scenedetect.__version__, "tolerances": list(TOLERANCES),
              "evaluator": evaluator_cases(), "grids": grid_cases()}
    path = os.path.join(HERE, "sweep_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
