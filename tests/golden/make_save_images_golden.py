#!/usr/bin/env python
"""Generate tests/golden/save_images_v1.json by running the REAL reference save_images (scenedetect/output/image.py
of a PySceneDetect source checkout given as the first argument) in both `threading` modes.

Run `python tests/golden/make_save_images_golden.py <reference checkout>`.  Each case is a scene list over a seekable
numpy stream of `frames` frames at `fps` that logs the frame index each read returns; recorded per case and mode:
the returned dict, the frames read (in order), the names of the files written, and whether "Could not generate all
output images." was logged.  The image bytes are cv2.imencode's and are not recorded (the GPU test checks them).
"""

from __future__ import annotations

import json
import logging
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, frames, fps, scene bounds (frame numbers), num_images, frame_margin
    dict(name="default_30", frames=120, fps=30, bounds=[0, 30, 31, 75, 120], num_images=3, frame_margin=1),
    dict(name="one_frame_scenes", frames=12, fps=24, bounds=[0, 1, 2, 3, 10, 12], num_images=3, frame_margin=1),
    dict(name="one_image", frames=90, fps=24, bounds=[0, 17, 50, 90], num_images=1, frame_margin=1),
    dict(name="two_images_margin0", frames=90, fps=60, bounds=[0, 17, 50, 90], num_images=2, frame_margin=0),
    dict(name="twelve_images_ntsc", frames=300, fps="30000/1001", bounds=[0, 100, 101, 260, 300], num_images=12,
         frame_margin=1),
    dict(name="margin_str_secs", frames=200, fps="30000/1001", bounds=[0, 40, 120, 200], num_images=3,
         frame_margin="0.1s"),
    dict(name="margin_float", frames=200, fps=60, bounds=[0, 40, 120, 200], num_images=3, frame_margin=0.5),
    dict(name="past_the_end", frames=50, fps=30, bounds=[0, 20, 60], num_images=3, frame_margin=0),
    dict(name="past_the_end_twelve", frames=40, fps=24, bounds=[0, 10, 50, 55], num_images=12, frame_margin=1),
]


def main(argv):
    sys.path.insert(0, os.path.abspath(argv[1]))
    from fractions import Fraction

    from scenedetect.common import FrameTimecode
    from scenedetect.output.image import save_images

    class LoggingStream:
        """seekable numpy stream (the VideoStream members save_images uses) that logs the frame each read returns"""

        def __init__(self, frames, fps):
            self.frames, self.frame_rate, self.pos, self.reads = frames, fps, 0, []
            self.name, self.aspect_ratio = "clip", 1.0

        def reset(self):
            self.pos = 0

        def seek(self, target):
            self.pos = FrameTimecode(target, self.frame_rate).frame_num

        def read(self, decode=True):
            if self.pos >= len(self.frames):
                return False
            self.reads.append(self.pos)
            self.pos += 1
            return self.frames[self.pos - 1]

    class Errors(logging.Handler):
        def __init__(self):
            super().__init__()
            self.messages = []

        def emit(self, record):
            if record.levelno >= logging.ERROR:
                self.messages.append(record.getMessage())

    out = {"cases": []}
    for case in CASES:
        fps = Fraction(case["fps"]) if isinstance(case["fps"], str) else float(case["fps"])
        frames = np.zeros((case["frames"], 16, 16, 3), np.uint8)
        frames[:, 0, 0, 0] = np.arange(case["frames"]) % 256
        b = case["bounds"]
        scenes = [(FrameTimecode(s, fps), FrameTimecode(e, fps)) for s, e in zip(b, b[1:])]
        rec = dict(case)
        for threading in (True, False):
            stream = LoggingStream(frames, fps)
            handler = Errors()
            logging.getLogger("pyscenedetect").addHandler(handler)
            with tempfile.TemporaryDirectory() as tmp:
                got = save_images(scenes, stream, num_images=case["num_images"], frame_margin=case["frame_margin"],
                                  output_dir=tmp, threading=threading)
                written = sorted(os.listdir(tmp))
            logging.getLogger("pyscenedetect").removeHandler(handler)
            rec["threading" if threading else "serial"] = {
                "result": {str(k): v for k, v in got.items()}, "reads": stream.reads, "files": written,
                "errors": handler.messages}
        out["cases"].append(rec)
    with open(os.path.join(HERE, "save_images_v1.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv)
