#!/usr/bin/env python
"""Benchmark of scene images encoded on the device (psd_jpeg_encode, pyscenedetect_b200/images.py).

Part 1, the encoder alone: --frames resident synthetic frames (psd_synth_frames) at 1280x720 and 1920x1080, quality
95, encoded by
  psd_jpeg_encode   one call for all the frames (CUDA events around the call, best of --reps)
  cv2               cv2.imencode of host copies on a thread pool of every host core (cv2 releases the GIL)
  nvjpeg            torchvision.io.encode_jpeg of the frames on CUDA (nvJPEG: a speed reference only; its bytes
                    differ, and `nvjpeg_equal` counts the files equal to cv2's)
reported as images/s and input GB/s (3 bytes a pixel read), with `equal` the psd_jpeg_encode files equal to cv2's.

Part 2, end to end, on bench_clips.py's 1000-clip set (1280x720 clips of 48 to 240 frames sliced from a resident
pool, ContentDetector() + AdaptiveDetector()): detect_clips, then
  device            save_clip_images of every clip's scenes (3 images a scene, quality 95)
  host              each clip's images through the reference's save_images pipeline (threading=True): the selected
                    frames read (copied out to numpy) on the calling thread, cv2.imencode on one encode thread, the
                    files written on one save thread, with queues of 4 items between them
both into a temporary directory; reported: seconds, images/s, launches per clip of the device arm, and how many
files are equal byte for byte.  Each run reads the card's name and power limit.  Prints one JSON line; writes only
under the temporary directory.

    python bench_save_images.py [--frames 64] [--clips 1000] [--reps 5]
"""

from __future__ import annotations

import argparse
import json
import os
import queue
import sys
import tempfile
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_clips import RATES, card_info, detectors  # noqa: E402


def encoder_alone(lib, n, w, h, reps, dev):
    import torch
    import torchvision

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan
    import cv2

    fb = w * h * 3
    frames = torch.empty((n, h, w, 3), dtype=torch.uint8, device=f"cuda:{dev}")
    synth_frames_device(frames.data_ptr(), ScenePlan(n, seed=1, min_len=1, max_len=3).params, w, h, device=dev)
    torch.cuda.synchronize()
    host = frames.cpu().numpy()
    images = (_capi.PsdJpegImage * n)()
    for k in range(n):
        images[k].base = frames.data_ptr() + k * fb
        images[k].layout = _capi.PsdFrameLayout(fb, 3 * w, 3, 1)
        images[k].width, images[k].height = w, h
    offs = torch.zeros(n + 1, dtype=torch.int64, device=frames.device)
    out = torch.empty(n * fb, dtype=torch.uint8, device=frames.device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def device_once():
        e0.record()
        _capi.check(lib.psd_jpeg_encode(dev, images, n, 95, 0, out.data_ptr(), out.numel(), offs.data_ptr(), None),
                    "psd_jpeg_encode")
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    device_once()
    t_dev = min(device_once() for _ in range(reps))
    ends = offs.cpu().numpy()
    data = out[:int(ends[n])].cpu().numpy().tobytes()
    ours = [data[ends[k]:ends[k + 1]] for k in range(n)]

    pool = ThreadPoolExecutor(os.cpu_count())

    def cv2_once():
        t0 = time.perf_counter()
        res = list(pool.map(lambda f: cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes(), host))
        return time.perf_counter() - t0, res

    cv2_once()
    t_cv2, ref = min((cv2_once() for _ in range(reps)), key=lambda x: x[0])
    pool.shutdown()

    chw = [f.permute(2, 0, 1).flip(0).contiguous() for f in frames]   # RGB planes, as encode_jpeg takes them

    def nvjpeg_once():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = torchvision.io.encode_jpeg(chw, quality=95)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, res

    nvjpeg_once()
    t_nv, nv = min((nvjpeg_once() for _ in range(reps)), key=lambda x: x[0])
    nv_bytes = [x.cpu().numpy().tobytes() for x in nv]

    def rate(t):
        return {"s": round(t, 5), "images_per_s": round(n / t, 1), "input_GB_per_s": round(n * fb / t / 1e9, 2)}
    return {"size": f"{w}x{h}", "frames": n, "psd_jpeg_encode": rate(t_dev), "cv2": rate(t_cv2),
            "cv2_threads": os.cpu_count(), "nvjpeg": rate(t_nv),
            "equal": sum(a == b for a, b in zip(ours, ref)), "nvjpeg_equal": sum(a == b for a, b in zip(nv_bytes, ref)),
            "mean_file_bytes": int(np.mean([len(x) for x in ref]))}


def end_to_end(lib, n_clips, dev, tmp):
    import cv2
    import torch

    from pyscenedetect_b200.clips import detect_clips, save_clip_images
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.images import _Plan
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    w, h, n_pool = 1280, 720, 1024
    fb = w * h * 3
    pool = torch.empty((n_pool, h, w, 3), dtype=torch.uint8, device=f"cuda:{dev}")
    plan = ScenePlan(n_pool, seed=0)
    for i in range(0, n_pool, 256):
        synth_frames_device(pool.data_ptr() + i * fb, plan.params[i:i + 256], w, h, device=dev)
    torch.cuda.synchronize()
    rng = np.random.default_rng(0)
    lengths = rng.integers(48, 241, size=n_clips)
    starts = [int(rng.integers(0, n_pool - n + 1)) for n in lengths]
    rates = [RATES[i % len(RATES)] for i in range(n_clips)]
    names = [f"clip{k:04d}" for k in range(n_clips)]

    def streams():
        return [ArrayVideoStream(pool[s:s + n], fps) for s, n, fps in zip(starts, lengths, rates)]

    def device_arm(out_dir):
        ss = streams()
        res = detect_clips(ss, detectors(), device=dev)
        maps = save_clip_images([(r.scene_list(), v) for r, v in zip(res, ss)], output_dir=out_dir, names=names,
                                device=dev)
        return sum(len(x) for m in maps for x in m.values())

    def host_arm(out_dir):
        # the reference's default threading=True pipeline (image.py _ImageExtractor.run): this thread reads each
        # selected frame (copied out to numpy), one thread encodes, one writes, through queues of 4 items
        ss = streams()
        res = detect_clips(ss, detectors(), device=dev)
        encode_q, save_q = queue.Queue(4), queue.Queue(4)

        def encoder():
            while (item := encode_q.get())[0] is not None:
                frame, path = item
                save_q.put((cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY, 95])[1], path))
            save_q.put((None, None))

        def saver():
            while (item := save_q.get())[0] is not None:
                item[0].tofile(item[1])

        threads = [threading.Thread(target=encoder), threading.Thread(target=saver)]
        for t in threads:
            t.start()
        n = 0
        for r, v, name in zip(res, ss, names):
            p = _Plan(r.scene_list(), v, name, 3, 1, "$VIDEO_NAME-Scene-$SCENE_NUMBER-$IMAGE_NUMBER", out_dir)
            for path, (video, index) in p.frames():
                os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
                encode_q.put((video._frames[index].cpu().numpy(), path))
                n += 1
        encode_q.put((None, None))
        for t in threads:
            t.join()
        return n

    device_arm(os.path.join(tmp, "warm"))
    l0 = lib.psd_launch_count()
    t0 = time.perf_counter()
    n_dev = device_arm(os.path.join(tmp, "device"))
    torch.cuda.synchronize()
    t_dev = time.perf_counter() - t0
    launches = lib.psd_launch_count() - l0
    t0 = time.perf_counter()
    n_host = host_arm(os.path.join(tmp, "host"))
    t_host = time.perf_counter() - t0
    files = sorted(os.listdir(os.path.join(tmp, "host")))
    equal = sum(open(os.path.join(tmp, "device", f), "rb").read() == open(os.path.join(tmp, "host", f), "rb").read()
                for f in files if os.path.exists(os.path.join(tmp, "device", f)))
    return {"clips": n_clips, "size": f"{w}x{h}", "images": {"device": n_dev, "host": n_host},
            "device": {"s": round(t_dev, 3), "images_per_s": round(n_dev / t_dev, 1),
                       "launches_per_clip": round(launches / n_clips, 2)},
            "host": {"s": round(t_host, 3), "images_per_s": round(n_host / t_host, 1)},
            "speedup": round(t_host / t_dev, 2), "files": len(files), "equal_files": int(equal)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)

    import torch

    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_save_images.py needs a CUDA device")
    torch.cuda.set_device(args.device)
    result = {"bench": "save_images", **card_info(args.device), "quality": 95, "encoder": [], "end_to_end": None}
    for w, h in ((1280, 720), (1920, 1080)):
        result["encoder"].append(encoder_alone(lib, args.frames, w, h, args.reps, args.device))
    with tempfile.TemporaryDirectory() as tmp:
        result["end_to_end"] = end_to_end(lib, args.clips, args.device, tmp)
    ok = (all(e["equal"] == e["frames"] for e in result["encoder"])
          and result["end_to_end"]["equal_files"] == result["end_to_end"]["files"]
          == result["end_to_end"]["images"]["device"])
    result["all_equal"] = bool(ok)
    print(json.dumps(result))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
