"""psd_jpeg_encode and save_images on the GPU: every file equals cv2.imencode byte for byte.

* the size / quality / content matrix of tests/jpeg_cases.py, plus 3840x2160 and 7680x4320;
* every frame layout the engine takes (packed BGR, RGB with channel stride -1, NCHW permutes, odd crops, steps, a
  negative row stride);
* mixed sizes in one call, a batch over several workspace sub-batches, and an out_cap that forces one regrow;
* save_images on CUDA and numpy ArrayVideoStreams (the golden cases recorded from the reference included, also in
  several encoder calls), and save_clip_images over 50 clips against save_images per clip;
* the encoder kernels do not spill to local memory."""

from __future__ import annotations

import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from tests import jpeg_cases as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_device_count() >= 1, "no CUDA device: GPU tests need an H100 (sm_90)"
    torch.cuda.set_device(0)
    return lib


def cv2_jpeg(bgr, q):
    return cv2.imencode(".jpg", np.ascontiguousarray(bgr), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


def encode(lib, images, quality, workspace_cap=0, out_cap=None):
    """images: [(base pointer, (frame, row, pixel, channel) strides, width, height)] -> (files, first total)"""
    import torch
    from pyscenedetect_b200 import _capi
    n = len(images)
    arr = (_capi.PsdJpegImage * n)()
    for k, (base, lay, w, h) in enumerate(images):
        arr[k].base, arr[k].layout, arr[k].width, arr[k].height = base, _capi.PsdFrameLayout(*lay), w, h
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    cap = out_cap if out_cap is not None else sum(w * h * 3 + 2048 for _, _, w, h in images)
    out = torch.empty(max(cap, 1), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _capi.check(lib.psd_jpeg_encode(0, arr, n, quality, workspace_cap, out.data_ptr(), cap, offs.data_ptr(), None),
                "psd_jpeg_encode")
    torch.cuda.synchronize()
    ends = offs.cpu().numpy()
    first_total = int(ends[n])
    if first_total > cap:
        out = torch.empty(first_total, dtype=torch.uint8, device="cuda")
        _capi.check(lib.psd_jpeg_encode(0, arr, n, quality, workspace_cap, out.data_ptr(), first_total,
                                        offs.data_ptr(), None), "psd_jpeg_encode")
        torch.cuda.synchronize()
        ends = offs.cpu().numpy()
    data = out[:int(ends[n])].cpu().numpy().tobytes()
    return [data[ends[k]:ends[k + 1]] for k in range(n)], first_total


def packed(t):
    """a packed (H, W, 3) BGR CUDA tensor as an encoder image"""
    h, w = t.shape[:2]
    return (t.data_ptr(), (h * w * 3, w * 3, 3, 1), w, h)


def test_matrix_equals_cv2(lib):
    import torch
    by_q = {}
    for c, w, h, q in K.cases(large=True):
        by_q.setdefault(q, []).append(K.frame(c, w, h))
    for w, h in ((3840, 2160), (7680, 4320)):
        by_q[95].append(K.frame("scene", w, h))
        by_q[95].append(K.frame("random", w, h, seed=1))
    for q, frames in by_q.items():
        dev = [torch.from_numpy(f).cuda() for f in frames]
        got, _ = encode(lib, [packed(t) for t in dev], q)
        for f, g in zip(frames, got):
            assert g == cv2_jpeg(f, q), (q, f.shape)


def test_every_layout_equals_cv2(lib):
    import torch
    base = K.frame("scene", 97, 61)
    nhwc = torch.from_numpy(np.stack([base, K.frame("random", 97, 61)])).cuda()
    cases = []
    # packed BGR
    cases.append((packed(nhwc[1]), nhwc[1].cpu().numpy()))
    # RGB with channel stride -1: the tensor holds R, G, B
    rgb = nhwc[..., [2, 1, 0]].contiguous()
    cases.append(((rgb[0].data_ptr() + 2, (0, 97 * 3, 3, -1), 97, 61), base))
    # NCHW permuted to NHWC
    nchw = nhwc.permute(0, 3, 1, 2).contiguous()
    hw = 97 * 61
    cases.append(((nchw[0].data_ptr(), (3 * hw, 97, 1, hw), 97, 61), base))
    # crops with odd offsets and steps
    crop = nhwc[0, 3:58:1, 5:90]
    cases.append(((crop.data_ptr(), (0, crop.stride(0), crop.stride(1), 1), crop.shape[1], crop.shape[0]),
                  base[3:58, 5:90]))
    step = nhwc[0, 1::3, 2::2]
    cases.append(((step.data_ptr(), (0, step.stride(0), step.stride(1), 1), step.shape[1], step.shape[0]),
                  base[1::3, 2::2]))
    # negative row stride: bottom row first
    last = nhwc[0, 60]
    cases.append(((last.data_ptr(), (0, -97 * 3, 3, 1), 97, 61), base[::-1]))
    for q in (50, 95):
        got, _ = encode(lib, [c for c, _ in cases], q)
        for (_, want), g in zip(cases, got):
            assert g == cv2_jpeg(want, q)


def test_batches_sub_batches_and_regrow(lib):
    import torch
    rng = np.random.default_rng(3)
    frames = [K.frame(["scene", "random", "smooth"][k % 3], int(rng.integers(1, 300)), int(rng.integers(1, 200)),
                      seed=k) for k in range(60)]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    imgs = [packed(t) for t in dev]
    want = [cv2_jpeg(f, 90) for f in frames]
    one, _ = encode(lib, imgs, 90)
    assert one == want
    several, _ = encode(lib, imgs, 90, workspace_cap=2 << 20)    # a few images per sub-batch
    assert several == want
    regrown, first_total = encode(lib, imgs, 90, out_cap=sum(len(x) for x in want) // 2)
    assert first_total == sum(len(x) for x in want) and regrown == want


def _scenes(n_frames, fps, cuts):
    from pyscenedetect_b200 import FrameTimecode
    bounds = [0, *cuts, n_frames]
    return [(FrameTimecode(a, fps), FrameTimecode(b, fps)) for a, b in zip(bounds, bounds[1:])]


def test_save_images_cuda_and_numpy_streams(lib, tmp_path):
    import torch
    from pyscenedetect_b200.images import save_images
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = render_frames(ScenePlan(90, seed=4, min_len=10, max_len=30).params, 160, 90)
    scenes = _scenes(90, 30.0, [20, 21, 55])
    for kind, stream in (("cuda", ArrayVideoStream(torch.from_numpy(frames).cuda())),
                         ("numpy", ArrayVideoStream(frames))):
        for q in (75, 95):
            out = tmp_path / f"{kind}{q}"
            got = save_images(scenes, stream, num_images=3, encoder_param=q, output_dir=str(out),
                              image_name_template="$SCENE_NUMBER-$IMAGE_NUMBER-$FRAME_NUMBER")
            assert sorted(got) == [0, 1, 2, 3]
            for i, names in got.items():
                assert len(names) == 3
                for name in names:
                    frame_num = int(name.split("-")[2].split(".")[0])
                    assert (out / name).read_bytes() == cv2_jpeg(frames[frame_num], q), (kind, name)


@pytest.mark.parametrize("group_frames", [None, 3])
def test_save_images_golden_cases(lib, tmp_path, monkeypatch, caplog, group_frames):
    """every case of tests/golden/save_images_v1.json (recorded from the reference save_images) on CUDA and numpy
    ArrayVideoStreams: the reference's file names, dict and error log, and each file the bytes cv2.imencode writes
    for the frame the reference read; group_frames 3: three frames per encoder call"""
    import logging

    import torch
    from pyscenedetect_b200 import images as I
    from pyscenedetect_b200.video import ArrayVideoStream
    from tests.test_save_images_host import CASES, case_input
    if group_frames:
        monkeypatch.setattr(I, "GROUP_BYTES", group_frames * 16 * 16 * 3)
    for name, case in sorted(CASES.items()):
        want = case["threading"]
        frames, fps, scenes = case_input(case)
        for kind, stream in (("cuda", ArrayVideoStream(torch.from_numpy(frames).cuda(), fps)),
                             ("numpy", ArrayVideoStream(frames, fps))):
            out = tmp_path / f"{name}-{kind}"
            caplog.clear()
            with caplog.at_level(logging.ERROR, logger="pyscenedetect"):
                got = I.save_images(scenes, stream, num_images=case["num_images"],
                                    frame_margin=case["frame_margin"], output_dir=str(out),
                                    image_name_template="clip-Scene-$SCENE_NUMBER-$IMAGE_NUMBER")
            assert {str(k): v for k, v in got.items()} == want["result"], (name, kind)
            assert sorted(os.listdir(out)) == want["files"], (name, kind)
            assert [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR] == want["errors"]
            files = [f for v in got.values() for f in v]
            for f, frame_num in zip(files, want["reads"]):
                assert (out / f).read_bytes() == cv2_jpeg(frames[frame_num], 95), (name, kind, f)


def test_save_clip_images_equals_save_images_per_clip(lib, tmp_path):
    import torch
    from pyscenedetect_b200.images import save_clip_images, save_images
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream
    rng = np.random.default_rng(5)
    clips, names = [], []
    for k in range(50):
        w, h, n = int(rng.integers(16, 200)), int(rng.integers(16, 120)), int(rng.integers(5, 60))
        frames = render_frames(ScenePlan(n, seed=k, min_len=3, max_len=20).params, w, h)
        cuts = sorted(set(int(c) for c in rng.integers(1, n, size=int(rng.integers(0, 4)))))
        stream = ArrayVideoStream(torch.from_numpy(frames).cuda() if k % 2 else frames)
        clips.append((_scenes(n, 24.0, cuts), stream))
        names.append(f"clip{k:02d}")
    together = save_clip_images(clips, output_dir=str(tmp_path / "a"), names=names)
    for (scenes, stream), name, got in zip(clips, names, together):
        one = save_images(scenes, stream, output_dir=str(tmp_path / "b"),
                          image_name_template=f"{name}-Scene-$SCENE_NUMBER-$IMAGE_NUMBER")
        assert one == got
        for files in got.values():
            for f in files:
                assert (tmp_path / "a" / f).read_bytes() == (tmp_path / "b" / f).read_bytes()
    with pytest.raises(ValueError, match="would both write"):
        save_clip_images(clips[:2], output_dir=str(tmp_path / "c"))


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="needs cuobjdump")
def test_encoder_kernels_do_not_spill():
    from pyscenedetect_b200 import _capi
    out = subprocess.run([CUOBJDUMP, "-sass", _capi.LIB_PATH], capture_output=True, text=True, timeout=600).stdout
    funcs = out.split("Function : ")
    jpeg = [f for f in funcs if f.startswith("_ZN3psd") and "jpeg_" in f.split("\n", 1)[0]]
    assert len(jpeg) == 5, [f.split("\n", 1)[0] for f in jpeg]
    for f in jpeg:
        assert " LDL" not in f and " STL" not in f, f"{f.split(chr(10), 1)[0]} spills to local memory"
