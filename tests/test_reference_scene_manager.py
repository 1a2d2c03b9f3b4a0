"""This package's `SceneManager` against the reference's over end_time / duration (frames, seconds, timecode
string) / frame_skip / crop / a stream that was already advanced, on golden case content_default_nostats.  The
reference SceneManager + ContentDetector results are stored in tests/golden/reference_compat.json.gz
(tests/golden/make_reference_compat.py).  Without a GPU: oracle-backed fake engine; with one: the real engine."""

import gzip
import json
import os

import pytest

from pyscenedetect_b200.compat import FrameTimecode
from tests.golden_util import case_frames, get_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_compat.json.gz")


class FrameStream:
    """A frame-by-frame stream (no read_batch), positioned like the reference's VideoStream."""

    def __init__(self, frames, fps=30.0):
        self._frames, self._n, self._fps = frames, 0, fps

    frame_rate = property(lambda self: self._fps)
    frame_size = property(lambda self: (self._frames.shape[2], self._frames.shape[1]))
    frame_number = property(lambda self: self._n)
    position = property(lambda self: FrameTimecode(max(0, self._n - 1), self._fps))

    def read(self, decode=True):
        if self._n >= len(self._frames):
            return False
        self._n += 1
        return self._frames[self._n - 1] if decode else True


def _check_settings():
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    with gzip.open(GOLDEN, "rt") as f:
        cases = json.load(f)["scene_manager_settings"]
    frames = case_frames(get_case("content_default_nostats"))
    checked = 0
    for case in cases:
        st = case["settings"]
        want = (case["frames"], case["cuts"], case["scenes"])
        sm, stream = SceneManager(batch_size=16), FrameStream(frames, 30.0)
        sm.add_detector(ContentDetector())
        sm.auto_downscale = bool(st.get("auto", False))
        if "crop" in st:
            sm.crop = tuple(st["crop"])
        for _ in range(st.get("start", 0)):
            stream.read(decode=False)
        kw = {k: v for k, v in st.items() if k in ("end_time", "duration", "frame_skip")}
        n = sm.detect_scenes(stream, **kw)
        got = (n, [c.frame_num for c in sm.get_cut_list()], [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()])
        assert got == want, st
        checked += 1
        # and the zero-copy (read_batch) path where it applies
        if "crop" not in st and not st.get("frame_skip") and not st.get("start"):
            sm = SceneManager(batch_size=16)
            sm.add_detector(ContentDetector())
            sm.auto_downscale = False
            kw = {k: v for k, v in st.items() if k in ("end_time", "duration")}
            n = sm.detect_scenes(ArrayVideoStream(frames, 30.0), **kw)
            got = (n, [c.frame_num for c in sm.get_cut_list()],
                   [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()])
            assert got == want, ("zero-copy", st)
            checked += 1
    assert checked >= 25


def test_scene_manager_settings_match_reference_fake_engine(monkeypatch):
    import numpy as np

    import pyscenedetect_b200.detectors._base as base_mod
    import pyscenedetect_b200.scene_manager as sm_mod
    from tests.fake_engine import OracleEngine

    class FakePinned:
        def __init__(self, nbytes):
            self.array = np.zeros(nbytes, np.uint8)

        def close(self):
            pass
    monkeypatch.setattr(base_mod, "Engine", OracleEngine)
    monkeypatch.setattr(sm_mod, "Engine", OracleEngine)
    monkeypatch.setattr(sm_mod, "PinnedBuffer", FakePinned)
    _check_settings()


@pytest.mark.gpu
def test_scene_manager_settings_match_reference_real_engine():
    _check_settings()
