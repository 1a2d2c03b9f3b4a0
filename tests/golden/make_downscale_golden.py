#!/usr/bin/env python
"""Generate tests/golden/downscale_v1.json by running the REAL reference (a PySceneDetect 0.7.1 source checkout given
as the first argument) at the frame sizes where cv2.resize's INTER_LINEAR scale, 1 / (dst / src), and src / dst give
different coefficients.

Run `python tests/golden/make_downscale_golden.py <reference checkout>`.  Each case is a ScenePlan video a few rows
high (so the recording stays small) through the reference's own `SceneManager` with a ContentDetector and a
`StatsManager`: per-frame metrics as `float.hex`, the cut list, the scene list and the CSV's sha256, as
make_golden.run_case records them, plus a crop where the case has one.  The sizes:

* 10241x4, 12287x6, 4x10241 (tall) and 15360x8 at downscale 2, 14335x14 at downscale 7: the scored side is 5120,
  6144, 5120, 7680 and 2048 (15360 -> 7680 has equal coefficients under both scales);
* a 10300x6 frame cropped to 10241x4 at downscale 2;
* 7680x4320 and the odd 1001x563 under auto-downscale (256x144 and 256x144).
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

KW = dict(min_scene_len=5)

# gen = (n, w, h, seed, min_len, max_len, noise_shift); crop as SceneManager.crop takes it (inclusive corners)
CASES = [
    dict(name="ds2_10241x4", gen=(40, 10241, 4, 61, 5, 12, 26), downscale=2),
    dict(name="ds2_12287x6", gen=(40, 12287, 6, 62, 5, 12, 26), downscale=2),
    dict(name="ds7_14335x14", gen=(40, 14335, 14, 63, 5, 12, 26), downscale=7),
    dict(name="ds2_4x10241", gen=(40, 4, 10241, 64, 5, 12, 26), downscale=2),
    dict(name="ds2_15360x8", gen=(40, 15360, 8, 65, 5, 12, 26), downscale=2),
    dict(name="crop_ds2_10241x4", gen=(40, 10300, 6, 66, 5, 12, 26), downscale=2, crop=(30, 1, 10270, 4)),
    dict(name="auto_7680x4320", gen=(4, 7680, 4320, 67, 1, 2, 26), auto_downscale=True),
    dict(name="auto_1001x563", gen=(40, 1001, 563, 68, 5, 12, 26), auto_downscale=True),
]


def run(case: dict) -> dict:
    n, w, h, seed, mn, mx, ns = case["gen"]
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    frames = render_frames(plan.params, w, h)
    fps = 30.0
    out = dict(case, det="content", kw=KW, fps=fps)
    out["frames_sha256"] = hashlib.sha256(frames.tobytes()).hexdigest()
    out["true_cuts"] = plan.cut_frames
    stats = StatsManager()
    sm = SceneManager(stats)
    sm.add_detector(build_detector("content", KW))
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case["downscale"]
    if "crop" in case:
        sm.crop = tuple(case["crop"])
    sm.detect_scenes(SyntheticStream(frames, fps), show_progress=False)
    out["cuts"] = [c.frame_num for c in sm.get_cut_list()]
    out["scene_list"] = [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]
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
    return out


def main():
    cases = []
    for c in CASES:
        out = run(c)
        print(out["name"], "cuts", out["cuts"], "true", out["true_cuts"])
        cases.append(out)
    golden = {"reference_version": scenedetect.__version__, "cases": cases}
    path = os.path.join(HERE, "downscale_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
