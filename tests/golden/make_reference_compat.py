#!/usr/bin/env python
"""Generate tests/golden/reference_compat.json.gz: what the reference (PySceneDetect 0.7.1) returns for the
inputs of tests/test_compat_vs_reference.py and tests/test_reference_scene_manager.py, so that those tests
compare this package against the reference without needing it installed.

    python tests/golden/make_reference_compat.py <path of a PySceneDetect 0.7.1 source checkout>
"""

from __future__ import annotations

import gzip
import io
import json
import os
import random
import sys
import zlib
from fractions import Fraction

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.abspath(sys.argv[1]))
sys.path.insert(0, ROOT)  # ahead of the reference, which has a `tests` package of its own

import numpy as np  # noqa: E402
import scenedetect  # noqa: E402
from scenedetect.common import FrameTimecode  # noqa: E402
from scenedetect.detector import FlashFilter  # noqa: E402
from scenedetect.detectors import ContentDetector  # noqa: E402
from scenedetect.scene_manager import SceneManager  # noqa: E402
from scenedetect.stats_manager import StatsManager  # noqa: E402
from scenedetect.video_stream import VideoStream  # noqa: E402

from tests.golden_util import case_frames, get_case  # noqa: E402

FPS = [30.0, 25.0, 24000 / 1001, 29.97, 60.0]
OTHERS = [15, 0.5, 0.6, "0.6s", "00:00:01.250", "12", 1.0 / 3.0]
FLASH_MODES = ["MERGE", "SUPPRESS"]
FLASH_LENGTHS = [15, 0, 1, 40, 0.5, "0.6s", "00:00:00.700", "20"]
SM_SETTINGS = [dict(), dict(end_time=100), dict(end_time=3.5), dict(end_time="00:00:05.100"), dict(duration=77),
               dict(duration=2.0), dict(duration="3s"), dict(end_time=0), dict(duration=0), dict(frame_skip=1),
               dict(frame_skip=3, end_time=120), dict(crop=[143, 10, 16, 81]), dict(crop=[0, 0, 40, 30], auto=True),
               dict(crop=[100, 50, 400, 300]), dict(start=40, duration=60), dict(start=40, end_time=90)]


def flash_seed(mode, length) -> int:
    return zlib.crc32(f"{mode}|{length}".encode()) & 0xFFFF


def compare_bits(a, b) -> int:
    """(a - b) >= o and a < o for each of OTHERS, then a == b and a >= b, as bits 0, 1, ... of an int."""
    bits = [(a - b) >= o for o in OTHERS] + [a < o for o in OTHERS] + [a == b, a >= b]
    return sum(int(v) << i for i, v in enumerate(bits))


def frame_timecodes():
    out = {}
    for fps in FPS:
        rng = random.Random(1)
        rows = []
        for _ in range(300):
            a, b = rng.randrange(0, 200000), rng.randrange(0, 200000)
            ra, rb = FrameTimecode(a, fps), FrameTimecode(b, fps)
            rows.append([ra.frame_num, ra.get_timecode(), ra.seconds, (ra - rb).frame_num, (ra + 7).frame_num,
                         compare_bits(ra, rb), hash(ra)])
        out[repr(fps)] = {"frame_rate": str(FrameTimecode(0, fps).frame_rate), "rows": rows,
                          "str_of_timecode": str(FrameTimecode("00:01:02.500", fps)),
                          "frame_of_1.5s": FrameTimecode(1.5, fps).frame_num}
    return out


def flash_filters():
    out = {}
    for mode in FLASH_MODES:
        for length in FLASH_LENGTHS:
            rng = random.Random(flash_seed(mode, length))
            runs = []
            for fps in (30.0, 24000 / 1001):
                f = FlashFilter(FlashFilter.Mode[mode], length)
                max_behind = f.max_behind
                p = rng.choice([0.05, 0.2, 0.5])
                cuts = {}
                for t in range(600):
                    got = [c.frame_num for c in f.filter(FrameTimecode(t, fps), rng.random() < p)]
                    if got:
                        cuts[str(t)] = got
                runs.append({"max_behind": max_behind, "cuts": cuts})
            out[f"{mode}|{length}"] = runs
    return out


def stats_manager():
    sm = StatsManager()
    keys = ["content_val", "delta_hue", "adaptive_ratio (w=2)"]
    sm.register_metrics(keys)
    rng = random.Random(3)
    for t in range(1, 80):
        row = {"content_val": np.float64(rng.random() * 50), "delta_hue": np.float64(rng.random())}
        if t % 3:
            row["adaptive_ratio (w=2)"] = rng.random() * 4
        sm.set_metrics(FrameTimecode(t, 30.0), row)
    buf = io.StringIO()
    sm.save_to_csv(buf)
    return {"keys": keys, "metrics_at_3": sm.get_metrics(FrameTimecode(3, 30.0), keys), "csv": buf.getvalue()}


class SyntheticStream(VideoStream):
    BACKEND_NAME = "synthetic"

    def __init__(self, frames, fps=30.0):
        self._frames, self._n = frames, 0
        self._fps = Fraction(fps).limit_denominator(1000000)

    path = property(lambda self: "synthetic")
    name = property(lambda self: "synthetic")
    is_seekable = property(lambda self: False)
    frame_rate = property(lambda self: self._fps)
    duration = property(lambda self: FrameTimecode(len(self._frames), self._fps))
    frame_size = property(lambda self: (self._frames.shape[2], self._frames.shape[1]))
    aspect_ratio = property(lambda self: 1.0)
    frame_number = property(lambda self: self._n)
    position = property(lambda self: FrameTimecode(max(0, self._n - 1), self._fps))
    position_ms = property(lambda self: 0.0 if self._n == 0 else 1000.0 * (self._n - 1) / float(self._fps))

    def read(self, decode=True):
        if self._n >= len(self._frames):
            return False
        self._n += 1
        return self._frames[self._n - 1] if decode else True

    def reset(self):
        self._n = 0

    def seek(self, target):
        raise NotImplementedError


def scene_manager_settings():
    """The reference SceneManager + ContentDetector() on golden case content_default_nostats."""
    frames = case_frames(get_case("content_default_nostats"))
    out = []
    for st in SM_SETTINGS:
        sm, stream = SceneManager(), SyntheticStream(frames, 30.0)
        sm.add_detector(ContentDetector())
        sm.auto_downscale = bool(st.get("auto", False))
        if "crop" in st:
            sm.crop = tuple(st["crop"])
        for _ in range(st.get("start", 0)):
            stream.read(decode=False)
        kw = {k: v for k, v in st.items() if k in ("end_time", "duration", "frame_skip")}
        n = sm.detect_scenes(stream, **kw)
        out.append({"settings": st, "frames": n, "cuts": [c.frame_num for c in sm.get_cut_list()],
                    "scenes": [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()]})
    return out


def main():
    doc = {"reference_version": scenedetect.__version__, "others": OTHERS,
           "frame_timecode": frame_timecodes(), "flash_filter": flash_filters(),
           "stats_manager": stats_manager(), "scene_manager_settings": scene_manager_settings()}
    with gzip.GzipFile(os.path.join(HERE, "reference_compat.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(doc, separators=(",", ":")).encode())


if __name__ == "__main__":
    main()
