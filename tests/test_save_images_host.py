"""save_images / save_clip_images host logic, with the numpy twin (tests/jpeg_twin.py) in place of psd_jpeg_encode:
frame selection, file names, the returned dict and the "Could not generate all output images." error reproduce the
reference (tests/golden/save_images_v1.json) on seekable streams and on numpy ArrayVideoStreams; the files hold the
twin's bytes; what cannot be exact raises ValueError."""

from __future__ import annotations

import json
import logging
import os
from fractions import Fraction

import numpy as np
import pytest

from pyscenedetect_b200 import images as I
from pyscenedetect_b200.compat import FrameTimecode
from pyscenedetect_b200.video import ArrayVideoStream
from tests import jpeg_twin as J

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "save_images_v1.json")))
CASES = {c["name"]: c for c in GOLDEN["cases"]}


class SeekableStream:
    """the VideoStream members save_images uses, over numpy frames; logs the frame each read returns"""

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


class TwinEncoder(list):
    """the frame numbers (pixel (0, 0) B) of every image encoded, and the size of every encoder call"""
    calls: list


@pytest.fixture
def twin_encoder(monkeypatch):
    """psd_jpeg_encode replaced by the twin"""
    encoded = TwinEncoder()
    encoded.calls = []

    def encode(refs, quality, device=0):
        frames = [I._host_frame(r) for r in refs]
        encoded.extend(int(f[0, 0, 0]) for f in frames)
        encoded.calls.append(len(frames))
        return [J.encode(f, quality) for f in frames]
    monkeypatch.setattr(I, "_encode_frames", encode)
    return encoded


def case_input(case):
    fps = Fraction(case["fps"]) if isinstance(case["fps"], str) else float(case["fps"])
    frames = np.zeros((case["frames"], 16, 16, 3), np.uint8)
    frames[:, 0, 0, 0] = np.arange(case["frames"]) % 256
    b = case["bounds"]
    return frames, fps, [(FrameTimecode(s, fps), FrameTimecode(e, fps)) for s, e in zip(b, b[1:])]


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("source", ["seekable", "array"])
@pytest.mark.parametrize("group_frames", [None, 2])
def test_reproduces_reference(name, source, group_frames, twin_encoder, tmp_path, caplog, monkeypatch):
    """group_frames 2: two 16x16 frames per encoder call, so a stream is read, encoded and written in several
    groups"""
    if group_frames:
        monkeypatch.setattr(I, "GROUP_BYTES", group_frames * 16 * 16 * 3)
    case = CASES[name]
    want = case["threading"]
    assert case["serial"] == want
    frames, fps, scenes = case_input(case)
    stream = SeekableStream(frames, fps) if source == "seekable" else ArrayVideoStream(frames, fps)
    template = "clip-Scene-$SCENE_NUMBER-$IMAGE_NUMBER"   # ArrayVideoStream.name is "array"
    with caplog.at_level(logging.ERROR, logger="pyscenedetect"):
        got = I.save_images(scenes, stream, num_images=case["num_images"], frame_margin=case["frame_margin"],
                            output_dir=str(tmp_path), image_name_template=template)
    assert {str(k): v for k, v in got.items()} == want["result"]
    assert sorted(os.listdir(tmp_path)) == want["files"]
    assert twin_encoder == [r % 256 for r in want["reads"]]   # pixel (0, 0) holds the frame number mod 256
    if source == "seekable":
        assert stream.reads == want["reads"]
    assert [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR] == want["errors"]
    if group_frames:
        assert max(twin_encoder.calls) <= group_frames
        assert len(twin_encoder.calls) == -(-len(want["reads"]) // group_frames)
    else:
        assert twin_encoder.calls == [len(want["reads"])]
    names = [n for v in got.values() for n in v]
    for n, frame_num in zip(names, want["reads"]):
        assert (tmp_path / n).read_bytes() == J.encode(frames[frame_num], 95)


def test_template_variables_and_quality(twin_encoder, tmp_path):
    frames, fps, scenes = case_input(CASES["twelve_images_ntsc"])
    got = I.save_images(scenes, ArrayVideoStream(frames, fps), num_images=2, encoder_param=40, output_dir=str(tmp_path),
                        image_name_template="$VIDEO_NAME-$TIMECODE-$FRAME_NUMBER-$TIMESTAMP_MS")
    first = got[0][0]
    tc = FrameTimecode(twin_encoder[0], fps)
    assert first.startswith("array-" + tc.get_timecode().replace(":", ";") + f"-{twin_encoder[0]}-")
    assert (tmp_path / first).read_bytes() == J.encode(frames[twin_encoder[0]], 40)


def test_refusals(twin_encoder, tmp_path):
    frames, fps, scenes = case_input(CASES["default_30"])
    s = ArrayVideoStream(frames, fps)
    for kw, msg in ((dict(image_extension="png"), "image_extension 'png'"), (dict(scale=0.5), "scale, height"),
                    (dict(height=10), "scale, height"), (dict(width=10), "scale, height"),
                    (dict(num_images=0), "num_images"), (dict(frame_margin=-1), "frame_margin")):
        with pytest.raises(ValueError, match=msg):
            I.save_images(scenes, s, output_dir=str(tmp_path), **kw)
    wide = SeekableStream(frames, fps)
    wide.aspect_ratio = 1.5
    with pytest.raises(ValueError, match="aspect_ratio"):
        I.save_images(scenes, wide, output_dir=str(tmp_path))
    assert I.save_images([], s) == {}
    with pytest.raises(ValueError, match="would both write"):
        I.save_clip_images([(scenes, s), (scenes, ArrayVideoStream(frames, fps))], output_dir=str(tmp_path))
    assert not os.listdir(tmp_path) and not twin_encoder


class GrayStream(SeekableStream):
    def read(self, decode=True):
        frame = super().read(decode)
        return frame if frame is False else frame[..., 0]


def test_refuses_frames_that_are_not_bgr24(twin_encoder, tmp_path):
    frames, fps, scenes = case_input(CASES["default_30"])
    with pytest.raises(ValueError, match=r"frame 1 of 'clip-Scene-001-01.jpg' is uint8 \(16, 16\)"):
        I.save_images(scenes, GrayStream(frames, fps), output_dir=str(tmp_path))
    with pytest.raises(ValueError, match="is float32"):
        I.save_images(scenes, SeekableStream(frames.astype(np.float32), fps), output_dir=str(tmp_path))
    assert not twin_encoder


def test_save_clip_images_equals_save_images_per_clip(twin_encoder, tmp_path):
    clips, names = [], []
    for k, name in enumerate(("default_30", "one_image", "past_the_end")):
        frames, fps, scenes = case_input(CASES[name])
        clips.append((scenes, ArrayVideoStream(frames, fps)))
        names.append(f"clip{k}")
    together = I.save_clip_images(clips, output_dir=str(tmp_path / "a"), names=names)
    for (scenes, stream), name, got in zip(clips, names, together):
        one = I.save_images(scenes, stream, output_dir=str(tmp_path / "b"),
                            image_name_template=f"{name}-Scene-$SCENE_NUMBER-$IMAGE_NUMBER")
        assert one == got
    assert sorted(os.listdir(tmp_path / "a")) == sorted(os.listdir(tmp_path / "b"))
    for f in os.listdir(tmp_path / "a"):
        assert (tmp_path / "a" / f).read_bytes() == (tmp_path / "b" / f).read_bytes()
