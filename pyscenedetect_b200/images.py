"""save_images (scenedetect/output/image.py:352-535) with every JPEG encoded on the GPU by psd_jpeg_encode: the same
file names, the same bytes as the reference's cv2.imencode, and the same returned dict.  `save_clip_images` does the
same for many (scene_list, video) pairs with all their images encoded together.

Frames come from where they already are: an `ArrayVideoStream` over CUDA frames is encoded in place by frame index
(no seek, no copy), one over numpy frames has only its selected frames uploaded, and any other `VideoStream` is
seeked and read on the host exactly as the reference does before its frames are uploaded.  Only what can be exact
is offered: JPEG, no resizing (`scale`, `height`, `width`) and square pixels; anything else raises ValueError."""

from __future__ import annotations

import logging
import math
import os
from string import Template

import numpy as np

from . import _capi, _dlpack
from ._capi import check
from .compat import FrameTimecode
from .engine import DeviceBuffer, gather_bgr
from .video import ArrayVideoStream

logger = logging.getLogger("pyscenedetect")

DEFAULT_TEMPLATE = "$VIDEO_NAME-Scene-$SCENE_NUMBER-$IMAGE_NUMBER"


def _generate_timecode_list(scene_list, num_images, frame_margin):
    """image.py:38-72: each scene's image timecodes, in seconds, at the scene list's frame rate"""
    frame_rate = scene_list[0][0].frame_rate
    margin_secs = FrameTimecode(timecode=frame_margin, fps=frame_rate).seconds
    result = []
    for start, end in scene_list:
        duration_secs = (end - start).seconds
        if duration_secs <= 0:
            result.append([start] * num_images)
            continue
        segment_secs = duration_secs / num_images
        timecodes = []
        for j in range(num_images):
            seg_start = start.seconds + j * segment_secs
            seg_end = start.seconds + (j + 1) * segment_secs
            if num_images == 1:
                t = start.seconds + duration_secs / 2.0
            elif j == 0:
                t = min(seg_start + margin_secs, seg_end)
            elif j == num_images - 1:
                t = max(seg_end - margin_secs, seg_start)
            else:
                t = (seg_start + seg_end) / 2.0
            timecodes.append(FrameTimecode(t, fps=frame_rate))
        result.append(timecodes)
    return result


def _output_path(file_path, output_dir) -> str:
    """platform.py get_and_create_path without creating the directories"""
    file_path = os.fspath(file_path)
    if output_dir is not None and not os.path.isabs(file_path):
        file_path = os.path.join(os.fspath(output_dir), file_path)
    return file_path


def _check_args(num_images, frame_margin, image_extension, scale, height, width):
    """image.py:418-421, then what this version cannot do exactly"""
    if num_images <= 0:
        raise ValueError("num_images must be greater than 0")
    if isinstance(frame_margin, (int, float)) and frame_margin < 0:
        raise ValueError("frame_margin must be non-negative")
    if image_extension != "jpg":
        raise ValueError(f"image_extension {image_extension!r}: only 'jpg' is encoded on the device")
    if scale or height or width:
        raise ValueError("scale, height and width are not supported: resizing (INTER_CUBIC by default) is not "
                         "done on the device")


# Frame bytes (3 per pixel) encoded per psd_jpeg_encode call.  Images are read, uploaded, encoded and written a group
# at a time, so host frames held, their device copy and the output buffers stay bounded whatever the number of images.
GROUP_BYTES = 512 << 20


class _Plan:
    """One (scene_list, video) pair: the images image.py:268-280 selects, their files, and the dict save_images
    returns.  `images` lists every selection with its file name; `frames()` reads them in order and fills
    `filenames` with the ones read.  A frame is (ArrayVideoStream, index), read in place by the encoder, or a host
    BGR array read through the stream's own seek and read, as the reference reads it (image.py:270-271).  A selection
    past the end of the stream skips the rest of that scene's images and clears `completed`."""

    def __init__(self, scene_list, video, name, num_images, frame_margin, template, output_dir):
        aspect = video.aspect_ratio
        if abs(aspect - 1.0) >= 0.01:
            raise ValueError(f"video aspect_ratio {aspect}: non-square pixels are not supported (the reference "
                             "resizes such frames)")
        self.video = video
        self.in_place = isinstance(video, ArrayVideoStream)
        self.filenames = {i: [] for i in range(len(scene_list))}
        self.images = []        # (scene index, file name, output path, FrameTimecode)
        self.completed = True
        if not scene_list:
            return
        template = Template(template)
        scene_fmt = "%0" + str(max(3, math.floor(math.log(len(scene_list), 10)) + 1)) + "d"
        image_fmt = "%0" + str(math.floor(math.log(num_images, 10)) + 2) + "d"
        total = video.duration.frame_num if self.in_place else None
        for i, timecodes in enumerate(_generate_timecode_list(scene_list, num_images, frame_margin)):
            for j, tc in enumerate(timecodes):
                if total is not None and tc.frame_num >= total:
                    self.completed = False
                    break
                file_path = "{}.{}".format(template.safe_substitute(
                    VIDEO_NAME=name,
                    SCENE_NUMBER=scene_fmt % (i + 1),
                    IMAGE_NUMBER=image_fmt % (j + 1),
                    FRAME_NUMBER=tc.frame_num,
                    TIMESTAMP_MS=int(tc.seconds * 1000),
                    TIMECODE=tc.get_timecode().replace(":", ";"),
                ), "jpg")
                self.images.append((i, file_path, _output_path(file_path, output_dir), tc))

    def frames(self, device: int = 0):
        """(output path, frame) of each image as it is read; a failed read skips the rest of its scene.  A CUDA frame
        of a stream read through seek and read is copied out on `device` (a _DeviceCopy)."""
        video = self.video
        video.reset()
        skip = None
        for i, file_path, path, tc in self.images:
            if i == skip:
                continue
            if self.in_place:
                frame = (video, tc.frame_num)
            else:
                video.seek(tc)
                frame = video.read()
                if frame is None or frame is False:
                    self.completed = False
                    skip = i
                    continue
                if _dlpack.is_dlpack(frame):
                    self.filenames[i].append(file_path)
                    yield path, _DeviceCopy(frame, getattr(video, "channel_order", "bgr"), device)
                    continue
                frame = np.asarray(frame)
                if frame.ndim != 3 or frame.shape[2] != 3 or frame.dtype != np.uint8:
                    raise ValueError(f"frame {tc.frame_num} of {file_path!r} is {frame.dtype} {frame.shape}: only "
                                     "(height, width, 3) uint8 BGR frames are encoded")
            self.filenames[i].append(file_path)
            yield path, frame


class _DeviceCopy:
    """A CUDA frame read through a stream's seek and read, gathered at once to packed BGR24 in HBM of its own: the
    stream may decode its next frame into the same memory (a decoder's pool of output buffers)."""

    def __init__(self, frame, channel_order: str, device: int):
        meta = _dlpack.import_frames(frame, device=device)
        if meta.ndim != 3:
            raise ValueError(f"a CUDA frame of shape {tuple(frame.shape)}: only (height, width, 3) uint8 BGR frames "
                             "are encoded")
        self.width, self.height = meta.width, meta.height
        self.buf = DeviceBuffer(max(1, self.width * self.height * 3), device)
        gather_bgr(frame, self.buf.ptr, None, channel_order, device)
        self.buf.download(1)   # cudaMemcpy: the gather is done before the stream's next read can overwrite the frame

    def close(self) -> None:
        self.buf.close()


def _frame_bytes(ref) -> int:
    if isinstance(ref, _DeviceCopy):
        return ref.width * ref.height * 3
    if isinstance(ref, np.ndarray):
        return ref.shape[0] * ref.shape[1] * 3
    return ref[0]._shape[1] * ref[0]._shape[2] * 3


def _host_frame(ref):
    """the BGR array of a frame reference that is not in CUDA memory, else None"""
    if isinstance(ref, np.ndarray):
        return ref
    if isinstance(ref, _DeviceCopy):
        return None
    video, index = ref
    if _dlpack.is_dlpack(video._frames):
        return None
    return video._frames[index % video._shape[0]]


def _encode_frames(refs, quality: int, device: int = 0) -> list[bytes]:
    """psd_jpeg_encode of a group of referenced frames in one call (sub-batched inside it): CUDA frames in place,
    host frames uploaded once"""
    lib = _capi.load()
    n = len(refs)
    if n == 0:
        return []
    images = (_capi.PsdJpegImage * n)()
    keep = []      # DLPack views whose memory the encoder reads
    host = [(k, f) for k, r in enumerate(refs) if (f := _host_frame(r)) is not None]
    staging = None
    if host:
        frames = [f for _, f in host]
        offsets = np.cumsum([0] + [f.nbytes for f in frames])
        staging = DeviceBuffer(max(1, int(offsets[-1])), device)
        for (k, _), f, o in zip(host, frames, offsets):
            f = np.ascontiguousarray(f)
            staging.upload(f, int(o))
            h, w = f.shape[:2]
            images[k].base = staging.ptr + int(o)
            images[k].layout = _capi.PsdFrameLayout(h * w * 3, w * 3, 3, 1)
            images[k].width, images[k].height = w, h
    views = {}
    for k, r in enumerate(refs):
        if isinstance(r, _DeviceCopy):
            images[k].base = r.buf.ptr
            images[k].layout = _capi.PsdFrameLayout(r.width * r.height * 3, r.width * 3, 3, 1)
            images[k].width, images[k].height = r.width, r.height
            continue
        if isinstance(r, np.ndarray) or not _dlpack.is_dlpack(r[0]._frames):
            continue
        video, index = r[0], r[1] % r[0]._shape[0]
        v = views.get(id(video))
        if v is None:
            v = views[id(video)] = _dlpack.import_frames(video._frames, stream=1, device=device,
                                                         channel_order=video.channel_order)
            keep.append(v)
        images[k].base = v.base + index * v.layout[0]
        images[k].layout = _capi.PsdFrameLayout(*v.layout)
        images[k].width, images[k].height = v.width, v.height
    offs = DeviceBuffer(8 * (n + 1), device)
    cap = sum(images[k].width * images[k].height for k in range(n)) + 1024 * n   # ~2.7 bits a pixel
    out = DeviceBuffer(cap, device)
    try:
        for _ in range(2):
            check(lib.psd_jpeg_encode(device, images, n, int(quality), 0, out.ptr, out.nbytes, offs.ptr, None),
                  "psd_jpeg_encode")
            ends = offs.download(8 * (n + 1)).view(np.int64)   # cudaMemcpy: waits for the encoder
            if ends[n] <= out.nbytes:
                break
            out.close()
            out = DeviceBuffer(int(ends[n]), device)
        data = out.download(int(ends[n])).tobytes()
    finally:
        out.close()
        offs.close()
        if staging is not None:
            staging.close()
    del keep
    return [data[ends[k]:ends[k + 1]] for k in range(n)]


def save_clip_images(clips, num_images: int = 3, frame_margin=1, image_extension: str = "jpg",
                     encoder_param: int = 95, image_name_template: str = DEFAULT_TEMPLATE, output_dir=None,
                     show_progress: bool | None = False, scale: float | None = None, height: int | None = None,
                     width: int | None = None, interpolation=None, threading: bool = True, names=None,
                     device: int = 0) -> list[dict]:
    """`save_images` for every `(scene_list, video)` pair of `clips` (e.g. `ClipResult.scene_list()` with the stream
    given to detect_clips), with their images encoded together, GROUP_BYTES of frames per encoder call: one dict per
    clip, each what `save_images` gives that clip.  `names`: each clip's $VIDEO_NAME (default: its stream's `name`, which is "array" for every
    ArrayVideoStream).  ValueError before any file is written when two clips would write the same path."""
    clips = list(clips)
    names = [v.name for _, v in clips] if names is None else list(names)
    if len(names) != len(clips):
        raise ValueError(f"{len(names)} names for {len(clips)} clips")
    _check_args(num_images, frame_margin, image_extension, scale, height, width)
    plans = [_Plan(scenes, video, name, num_images, frame_margin, image_name_template, output_dir)
             for (scenes, video), name in zip(clips, names)]
    owner = {}
    for c, plan in enumerate(plans):
        for _, _, path, _ in plan.images:
            key = os.path.normcase(os.path.abspath(path))
            if owner.setdefault(key, c) != c:
                raise ValueError(f"clips {owner[key]} and {c} would both write {path}: give each clip its own name "
                                 "(names=...) or image_name_template")
    quality = 95 if encoder_param is None else int(encoder_param)   # cv2's default JPEG quality
    group, group_bytes = [], 0

    def flush():
        try:
            for (path, _), data in zip(group, _encode_frames([ref for _, ref in group], quality, device)):
                os.makedirs(os.path.split(os.path.abspath(path))[0], exist_ok=True)
                with open(path, "wb") as f:
                    f.write(data)
        finally:
            for _, ref in group:
                if isinstance(ref, _DeviceCopy):
                    ref.close()
            group.clear()

    for plan in plans:
        for path, ref in plan.frames(device):
            nbytes = _frame_bytes(ref)
            if group and group_bytes + nbytes > GROUP_BYTES:
                flush()
                group_bytes = 0
            group.append((path, ref))
            group_bytes += nbytes
    flush()
    for plan in plans:
        if not plan.completed:
            logger.error("Could not generate all output images.")
    return [plan.filenames for plan in plans]


def save_images(scene_list, video, num_images: int = 3, frame_margin=1, image_extension: str = "jpg",
                encoder_param: int = 95, image_name_template: str = DEFAULT_TEMPLATE, output_dir=None,
                show_progress: bool | None = False, scale: float | None = None, height: int | None = None,
                width: int | None = None, interpolation=None, threading: bool = True,
                device: int = 0) -> dict:
    """image.py:352-535 on the GPU: `num_images` JPEG images of every scene, named by `image_name_template`, with the
    bytes cv2.imencode writes at quality `encoder_param`; returns {scene index: [file names]}.  `show_progress`,
    `interpolation` and `threading` change nothing here (no resizing; frames are read, encoded and written in groups of
    GROUP_BYTES).  ValueError for an
    `image_extension` other than "jpg", for `scale` / `height` / `width`, and for a stream whose aspect_ratio is not
    within 0.01 of 1, or a frame read from the stream that is not (height, width, 3) uint8."""
    if not scene_list:
        return {}
    return save_clip_images([(scene_list, video)], num_images, frame_margin, image_extension, encoder_param,
                            image_name_template, output_dir, show_progress, scale, height, width, interpolation,
                            threading, names=[video.name], device=device)[0]


__all__ = ["save_images", "save_clip_images"]
