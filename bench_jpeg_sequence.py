"""JPEG image sequences on the GPU: psd_jpeg_decode alone, SceneManager.detect_scenes(ImageSequenceStream) end to end,
and cv2.imread on every host core feeding SceneManager through page-locked frames, on synthetic 1920x1080 frames
(noise, a gradient and text) written by cv2 at quality 95, 4:2:0.  Where torchvision's decode_jpeg runs on CUDA,
nvJPEG is a reference point, with how many of its frames equal cv2's.  Prints one JSON line; files go to a temporary
directory."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def synth(w, h, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    f = np.stack([(x * 255 // (w - 1)), (y * 255 // (h - 1)), ((x + y + seed * 40) % 256)], -1)
    f = (f + rng.integers(-20, 21, (h, w, 3))).clip(0, 255).astype(np.uint8)
    cv2.putText(f, f"frame {seed}", (w // 8, h // 2), cv2.FONT_HERSHEY_SIMPLEX, h / 300, (255, 255, 255), 3)
    return f


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - the numbers are still printed, with the reason the card is unknown
        return {"name": None, "error": str(e)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=32, help="distinct synthetic frames, cycled")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args(argv)
    import torch

    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.image_sequence import DeviceDecoder, ImageSequenceStream
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream

    w, h = 1920, 1080
    tmp = tempfile.mkdtemp(prefix="psd_jpeg_seq_")
    datas = [cv2.imencode(".jpg", synth(w, h, i // 4), [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()
             for i in range(a.distinct)]
    paths = []
    for i in range(a.frames):
        p = os.path.join(tmp, f"f_{i:05d}.jpg")
        with open(p, "wb") as f:
            f.write(datas[i % a.distinct])
        paths.append(p)
    in_bytes = sum(len(datas[i % a.distinct]) for i in range(a.batch))
    res = {"card": card(), "frames": a.frames, "size": [w, h], "mean_file_bytes": float(np.mean([len(d) for d in datas]))}

    # arm 1: psd_jpeg_decode of one batch of files already read into memory
    dec = DeviceDecoder()
    out = dec.allocate(a.batch, h, w)
    batch = [datas[i % a.distinct] for i in range(a.batch)]
    names = [f"frame {i}" for i in range(a.batch)]
    dec.decode(batch, names, out)
    torch.cuda.synchronize()
    ok = all(np.array_equal(out[i].cpu().numpy(), cv2.imdecode(np.frombuffer(batch[i], np.uint8), cv2.IMREAD_COLOR))
             for i in range(min(a.batch, a.distinct)))
    times = []
    for _ in range(a.repeats * 4):
        t0 = time.perf_counter()
        dec.decode(batch, names, out)   # ends in a device synchronise (the error flags)
        times.append(time.perf_counter() - t0)
    t = float(np.median(times))
    res["decode"] = {"images_per_s": a.batch / t, "input_GBps": in_bytes / t / 1e9,
                     "output_GBps": a.batch * w * h * 3 / t / 1e9, "batch": a.batch, "equal_to_cv2": ok,
                     "timing": "host clock around read-to-flags, median; includes the pinned copy and the H2D copy"}

    def detect(video):
        sm = SceneManager(batch_size=a.batch)
        sm.add_detector(ContentDetector())
        t0 = time.perf_counter()
        sm.detect_scenes(video)
        cuts = [c.frame_num for c in sm.get_cut_list()]
        return time.perf_counter() - t0, cuts

    # arm 2: SceneManager on the stream, end to end (file reads included)
    detect(ImageSequenceStream(paths[:a.batch * 2], batch_size=a.batch))
    e2e = [detect(ImageSequenceStream(paths, batch_size=a.batch)) for _ in range(a.repeats)]
    t_seq = float(np.median([x[0] for x in e2e]))
    res["sequence_e2e"] = {"frames_per_s": a.frames / t_seq, "cuts": e2e[0][1]}

    # arm 3: cv2.imread on every host core into page-locked frames, then SceneManager
    ncpu = os.cpu_count() or 1
    pinned = torch.empty((a.frames, h, w, 3), dtype=torch.uint8, pin_memory=True).numpy()

    def imread_arm():
        t0 = time.perf_counter()
        with ThreadPoolExecutor(ncpu) as ex:
            for i, f in enumerate(ex.map(cv2.imread, paths)):
                pinned[i] = f
        t1 = time.perf_counter()
        td, cuts = detect(ArrayVideoStream(pinned, fps=25.0, pinned=True))
        return t1 - t0 + td, cuts

    arms = [imread_arm() for _ in range(a.repeats)]
    t_cpu = float(np.median([x[0] for x in arms]))
    res["imread_e2e"] = {"frames_per_s": a.frames / t_cpu, "host_cores": ncpu, "cuts": arms[0][1]}
    res["sequence_beats_imread"] = t_seq < t_cpu
    res["cuts_equal"] = e2e[0][1] == arms[0][1]

    # nvJPEG reference point
    try:
        from torchvision.io import decode_jpeg
        ts = [torch.frombuffer(bytearray(d), dtype=torch.uint8) for d in batch]
        imgs = decode_jpeg(ts, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.repeats):
            imgs = decode_jpeg(ts, device="cuda")
        torch.cuda.synchronize()
        tn = (time.perf_counter() - t0) / a.repeats
        equal = sum(np.array_equal(im.permute(1, 2, 0).flip(-1).cpu().numpy(),
                                   cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_COLOR))
                    for im, d in zip(imgs, batch))
        res["nvjpeg"] = {"images_per_s": a.batch / tn, "frames_equal_to_cv2": int(equal), "of": a.batch}
    except Exception as e:  # noqa: BLE001 - torchvision is optional
        res["nvjpeg"] = {"unavailable": f"{type(e).__name__}: {e}"}
    for p in paths:
        os.remove(p)
    os.rmdir(tmp)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
