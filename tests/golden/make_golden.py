#!/usr/bin/env python
"""Generate tests/golden/golden_v1.json by running the REAL reference (imported from
a PySceneDetect 0.7.1 source checkout given as the first argument) on seeded synthetic sequences.

Run `python tests/golden/make_golden.py <reference checkout>`; the tests do not need the reference,
which is why the outputs are committed.  Metric values are stored as
`float.hex()` strings so they round-trip bit for bit.  Cases that go through the
reference's own `SceneManager.detect_scenes` (decode thread, cv2.resize downscale,
StatsManager CSV) use a synthetic `VideoStream`.
"""

from __future__ import annotations

import hashlib
import io
import json
import os
import sys
from fractions import Fraction

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.abspath(sys.argv[1]))  # a PySceneDetect 0.7.1 source checkout

import cv2  # noqa: E402
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
from scenedetect.scene_manager import SceneManager  # noqa: E402
from scenedetect.stats_manager import StatsManager  # noqa: E402
from scenedetect.video_stream import VideoStream  # noqa: E402

from pyscenedetect_b200.synth import ScenePlan, render_frames  # noqa: E402


class SyntheticStream(VideoStream):
    """Minimal forward-only VideoStream over an in-memory frame array."""

    BACKEND_NAME = "synthetic"

    def __init__(self, frames: np.ndarray, fps=30.0):
        self._frames = frames
        self._fps = Fraction(fps).limit_denominator(1000000)
        self._n = 0

    path = property(lambda self: "synthetic")
    name = property(lambda self: "synthetic")
    is_seekable = property(lambda self: False)
    frame_rate = property(lambda self: self._fps)
    duration = property(lambda self: FrameTimecode(len(self._frames), self._fps))
    frame_size = property(lambda self: (self._frames.shape[2], self._frames.shape[1]))
    aspect_ratio = property(lambda self: 1.0)
    frame_number = property(lambda self: self._n)

    @property
    def position(self):
        return FrameTimecode(max(0, self._n - 1), self._fps)

    @property
    def position_ms(self):
        return 0.0 if self._n == 0 else 1000.0 * (self._n - 1) / float(self._fps)

    def read(self, decode: bool = True):
        if self._n >= len(self._frames):
            return False
        frame = self._frames[self._n]
        self._n += 1
        return frame if decode else True

    def reset(self):
        self._n = 0

    def seek(self, target):
        raise NotImplementedError


DETECTORS = {
    "content": ContentDetector,
    "adaptive": AdaptiveDetector,
    "threshold": ThresholdDetector,
    "histogram": HistogramDetector,
    "hash": HashDetector,
}


def build_detector(name: str, kwargs: dict):
    kw = dict(kwargs)
    if "weights" in kw:
        kw["weights"] = ContentDetector.Components(*kw["weights"])
    if "filter_mode" in kw:
        kw["filter_mode"] = FlashFilter.Mode[kw["filter_mode"]]
    if "method" in kw:
        kw["method"] = ThresholdDetector.Method[kw["method"]]
    return DETECTORS[name](**kw)


def hexify(v):
    if v is None:
        return None
    return float(v).hex()


CASES = [
    # name, gen(n,w,h,seed,min_len,max_len,noise_shift), detector, kwargs, mode, fps
    dict(name="cfg1_threshold_360p", gen=(300, 640, 360, 1, 20, 70, 30), det="threshold", kw={},
         mode="direct", stats=True, fps=30.0),
    dict(name="threshold_ceiling_final", gen=(300, 160, 90, 7, 20, 70, 30), det="threshold",
         kw=dict(threshold=140, method="CEILING", add_final_scene=True, fade_bias=0.5,
                 min_scene_len=5), mode="direct", stats=True, fps=30.0),
    dict(name="threshold_bias_neg", gen=(300, 160, 90, 4, 20, 70, 30), det="threshold",
         kw=dict(threshold=20, fade_bias=-0.7, min_scene_len="0.4s", add_final_scene=True),
         mode="direct", stats=False, fps=25.0),
    dict(name="content_default_stats", gen=(260, 160, 90, 0, 20, 70, 30), det="content", kw={},
         mode="direct", stats=True, fps=30.0),
    dict(name="content_default_nostats", gen=(260, 160, 90, 0, 20, 70, 30), det="content", kw={},
         mode="direct", stats=False, fps=30.0),
    dict(name="content_suppress", gen=(260, 160, 90, 1, 20, 60, 29), det="content",
         kw=dict(filter_mode="SUPPRESS", min_scene_len=25), mode="direct", stats=False, fps=30.0),
    dict(name="content_merge_long", gen=(300, 160, 90, 2, 20, 40, 29), det="content",
         kw=dict(min_scene_len=30, threshold=20.0), mode="direct", stats=False, fps=30.0),
    dict(name="content_edges_w", gen=(200, 192, 108, 4, 20, 60, 30), det="content",
         kw=dict(weights=(1.0, 1.0, 1.0, 1.0), threshold=30.0), mode="direct", stats=True, fps=30.0),
    dict(name="content_edges_k3", gen=(120, 96, 64, 6, 20, 50, 30), det="content",
         kw=dict(weights=(0.5, 0.25, 1.0, 2.0), kernel_size=3), mode="direct", stats=True,
         fps=30.0),
    # width not a multiple of 32 / 16 / 4: the bit-packed dilation has padding bits in every row's last
    # word, and the fused pass scores an aligned copy and sends the last pixels of each frame to its tail kernel
    dict(name="content_edges_odd_size", gen=(140, 131, 97, 12, 20, 50, 30), det="content",
         kw=dict(weights=(1.0, 1.0, 1.0, 1.0), threshold=28.0), mode="direct", stats=True, fps=30.0),
    dict(name="content_luma_only", gen=(200, 160, 90, 7, 20, 60, 30), det="content",
         kw=dict(luma_only=True, threshold=15.0, min_scene_len=0.5), mode="direct", stats=True,
         fps=24000 / 1001),
    dict(name="adaptive_w2", gen=(260, 160, 90, 0, 20, 70, 30), det="adaptive", kw={},
         mode="direct", stats=True, fps=30.0),
    dict(name="adaptive_w5_edges", gen=(220, 160, 90, 8, 20, 60, 30), det="adaptive",
         kw=dict(window_width=5, weights=(1.0, 1.0, 1.0, 1.0)), mode="direct", stats=True,
         fps=30.0),
    dict(name="adaptive_lum_w3", gen=(220, 128, 72, 9, 20, 60, 29), det="adaptive",
         kw=dict(window_width=3, luma_only=True, adaptive_threshold=2.0, min_content_val=8.0,
                 min_scene_len="10"), mode="direct", stats=True, fps=30.0),
    dict(name="hist_128", gen=(260, 160, 90, 0, 20, 70, 30), det="histogram", kw={},
         mode="direct", stats=True, fps=30.0),
    dict(name="hist_256", gen=(260, 160, 90, 10, 20, 70, 30), det="histogram",
         kw=dict(bins=256, threshold=0.05), mode="direct", stats=True, fps=30.0),
    dict(name="hist_256_minlen_edge", gen=(260, 160, 90, 10, 20, 70, 30), det="histogram",
         kw=dict(bins=256, threshold=0.05, min_scene_len=22), mode="direct", stats=True, fps=30.0),
    dict(name="hist_100", gen=(200, 100, 60, 11, 20, 70, 29), det="histogram",
         kw=dict(bins=100, threshold=0.1, min_scene_len=0), mode="direct", stats=True, fps=30.0),
    # Through the reference SceneManager: auto-downscale (640x360 -> 256x144) + CSV.
    dict(name="sm_content_downscale", gen=(220, 640, 360, 12, 20, 70, 30), det="content", kw={},
         mode="scene_manager", stats=True, fps=30.0, auto_downscale=True),
    dict(name="sm_adaptive_downscale", gen=(220, 640, 360, 12, 20, 70, 30), det="adaptive",
         kw=dict(window_width=3), mode="scene_manager", stats=True, fps=30.0,
         auto_downscale=True),
    dict(name="sm_hist_downscale3", gen=(200, 480, 270, 13, 20, 70, 30), det="histogram",
         kw=dict(bins=256), mode="scene_manager", stats=True, fps=30.0, downscale=3),
    dict(name="sm_threshold_full", gen=(260, 320, 180, 14, 20, 70, 30), det="threshold", kw={},
         mode="scene_manager", stats=True, fps=30.0, downscale=1),
]


# Second fixture file (golden_v2.json): HashDetector (SURVEY §8 N4) and a histogram-through-SceneManager case
# whose cut list is not empty (golden_v1's sm_hist_downscale3 has none).
CASES_V2 = [
    # 160x90 -> 16x16: non-integer area scale (10 x 5.625): OpenCV's float-accumulating INTER_AREA path
    dict(name="hash_default", gen=(260, 160, 90, 0, 20, 70, 30), det="hash", kw={}, mode="direct", stats=True, fps=30.0),
    # 256x144 -> 16x16: integer scale (16 x 9): the integer-sum path; lower threshold, float min_scene_len
    dict(name="hash_int_scale", gen=(220, 256, 144, 5, 20, 60, 30), det="hash",
         kw=dict(threshold=0.25, min_scene_len=0.4), mode="direct", stats=True, fps=25.0),
    # size 16, lowpass 4 -> 64x64 DCT, 256-bit hash; 320x176 -> 64: scale 5 x 2.75
    dict(name="hash_16_4", gen=(200, 320, 176, 6, 20, 60, 30), det="hash",
         kw=dict(size=16, lowpass=4, threshold=0.3), mode="direct", stats=True, fps=30.0),
    dict(name="hash_4_2_odd", gen=(160, 131, 97, 12, 20, 50, 30), det="hash",
         kw=dict(size=4, lowpass=2, threshold=0.3, min_scene_len=10), mode="direct", stats=False, fps=30.0),
    # through the reference SceneManager: 640x360 auto-downscaled to 256x144 first
    dict(name="sm_hash_downscale", gen=(220, 640, 360, 12, 20, 70, 30), det="hash", kw={},
         mode="scene_manager", stats=True, fps=30.0, auto_downscale=True),
    dict(name="sm_hist_downscale2_cuts", gen=(260, 320, 180, 10, 20, 70, 30), det="histogram",
         kw=dict(bins=256, threshold=0.05), mode="scene_manager", stats=True, fps=30.0, downscale=2),
]


def run_case(case: dict) -> dict:
    n, w, h, seed, mn, mx, ns = case["gen"]
    plan = ScenePlan(n, seed=seed, noise_shift=ns, min_len=mn, max_len=mx)
    frames = render_frames(plan.params, w, h)
    det = build_detector(case["det"], case["kw"])
    fps = case["fps"]
    out = dict(case)
    out["frames_sha256"] = hashlib.sha256(frames.tobytes()).hexdigest()
    out["true_cuts"] = plan.cut_frames
    stats = StatsManager() if case["stats"] else None
    if case["mode"] == "direct":
        det.stats_manager = stats
        if stats is not None:
            stats.register_metrics(det.get_metrics())
        cuts = []
        for i in range(n):
            cuts += det.process_frame(FrameTimecode(i, fps), frames[i])
        cuts += det.post_process(FrameTimecode(n - 1, fps))
        cut_frames = sorted({c.frame_num for c in cuts})
        scene_list = None
    else:
        sm = SceneManager(stats)
        sm.add_detector(det)
        if case.get("auto_downscale"):
            sm.auto_downscale = True
        else:
            sm.auto_downscale = False
            sm.downscale = case.get("downscale", 1)
        stream = SyntheticStream(frames, fps)
        sm.detect_scenes(stream, show_progress=False)
        cut_frames = [c.frame_num for c in sm.get_cut_list()]
        scene_list = [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]
    out["cuts"] = cut_frames
    out["scene_list"] = scene_list
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
    golden = {
        "reference_version": scenedetect.__version__,
        "cv2": cv2.__version__,
        "numpy": np.__version__,
        "cases": [run_case(c) for c in CASES],
    }
    path = os.path.join(HERE, "golden_v1.json")
    with open(path, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
    for c in golden["cases"]:
        print(c["name"], "cuts", c["cuts"], "true", c["true_cuts"])
    print("wrote", path, os.path.getsize(path), "bytes")
    golden2 = dict(golden, cases=[run_case(c) for c in CASES_V2])
    path = os.path.join(HERE, "golden_v2.json")
    with open(path, "w") as f:
        json.dump(golden2, f, indent=0, sort_keys=True)
    for c in golden2["cases"]:
        print(c["name"], "cuts", c["cuts"], "true", c["true_cuts"])
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
