#!/usr/bin/env python
"""Generate tests/golden/shared_pass_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout
given as the first argument): detectors that disagree on the dilation kernel size or the hash geometry in one
reference `SceneManager`.

Run `python tests/golden/make_shared_pass_golden.py <reference checkout>`.  The cases are stored exactly as
make_multi_detector_golden.py stores its own (cut list, scene list, per-frame metrics as `float.hex`, the CSV's
sha256), all with a `StatsManager`, which turns the edge component on for every Content/Adaptive detector.  In this
package the detectors of one SceneManager share one engine that holds each distinct kernel size and hash geometry
as a slot:

* 640x360 auto-downscaled to 256x144 (automatic kernel size 5): kernel sizes 5, automatic and 7, two slots;
* 640x360 at full size: kernel size 19 (separable dilation) and 5 (register dilation) in one engine;
* 640x360 auto-downscaled: hashes (8, 2), (16, 2) and (8, 3) next to a HistogramDetector;
* 133x99: kernel sizes 3 and 5 and hashes (8, 2) and (16, 3).
"""

from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_multi_detector_golden import run_case  # noqa: E402  (puts the checkout on sys.path)

import scenedetect  # noqa: E402

ALL = (1.0, 1.0, 1.0, 1.0)

# name, gen(n, w, h, seed, min_len, max_len, noise_shift), detectors [(name, kwargs)], stats, scaling
CASES = [
    dict(name="kernel_sizes_auto_dedup_360p", gen=(120, 640, 360, 61, 15, 50, 30),
         dets=[("content", dict(kernel_size=5)), ("adaptive", {}),
               ("content", dict(weights=ALL, kernel_size=7, threshold=30.0))], stats=True, auto_downscale=True),
    dict(name="kernel_sizes_separable_and_register_360p", gen=(100, 640, 360, 62, 15, 50, 30),
         dets=[("content", dict(kernel_size=19, weights=ALL)), ("adaptive", dict(kernel_size=5))], stats=True,
         downscale=1),
    dict(name="hash_geometries_histogram_360p", gen=(120, 640, 360, 63, 15, 50, 30),
         dets=[("hash", dict(size=8)), ("hash", dict(size=16, threshold=0.3)), ("hash", dict(size=8, lowpass=3)),
               ("histogram", {})], stats=True, auto_downscale=True),
    dict(name="kernel_sizes_and_hashes_133x99", gen=(150, 133, 99, 64, 15, 50, 30),
         dets=[("content", dict(kernel_size=3, weights=ALL)), ("adaptive", dict(kernel_size=5, window_width=3)),
               ("hash", dict(size=8)), ("hash", dict(size=16, lowpass=3, threshold=0.3))], stats=True, downscale=1),
]


def main():
    cases = []
    for c in CASES:
        out = run_case(c)
        print(out["name"], "cuts", out["cuts"], "true", out["true_cuts"])
        cases.append(out)
    golden = {"reference_version": scenedetect.__version__, "cases": cases}
    path = os.path.join(HERE, "shared_pass_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
