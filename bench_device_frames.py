"""Frames already on the GPU: what psd_gather_bgr moves, what the engine scores per layout, and what SceneManager
reaches over resident frames next to the same frames from host memory.

    python bench_device_frames.py [--frames 1024] [--scene-frames 1000] [--repeat 10] [--reps 5]

Prints the card and its power limit, then one JSON line.  Every layout's per-frame integers are checked against the
packed BGR submission, the gathers against torch's own permute / flip, and the SceneManager cut lists against the
host run, in the same run as the timing.  Needs an sm_90 GPU; nothing is written to the tree."""

from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np
import torch

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, reps: int) -> float:
    """Median seconds of fn() ending in a device synchronise."""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def gather_rates(packed: torch.Tensor, reps: int) -> dict:
    from pyscenedetect_b200.engine import gather_bgr
    n, h, w, _ = packed.shape
    out = {}
    dst = torch.empty_like(packed)
    nchw = packed.permute(0, 3, 1, 2).contiguous()
    for name, (src, order, want) in {
        "nchw_bgr": (nchw.permute(0, 2, 3, 1), "bgr", packed),
        "packed_rgb": (packed, "rgb", packed.flip(-1)),
    }.items():
        held = []

        def run():
            held.append(gather_bgr(src, dst.data_ptr(), w * h * 3, channel_order=order))
        gather_bgr(src, dst.data_ptr(), w * h * 3, channel_order=order)
        torch.cuda.synchronize()
        assert torch.equal(dst, want), name
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        run()
        ev0.record()
        for _ in range(reps):
            run()
        ev1.record()
        torch.cuda.synchronize()
        s = ev0.elapsed_time(ev1) / 1e3 / reps
        moved = 6 * n * h * w
        out[name] = {"frames": n, "ms": round(s * 1e3, 3), "GB_per_s": round(moved / s / 1e9, 1),
                     "share_of_3.35TB_per_s": round(moved / s / HBM_PEAK, 3)}
        held.clear()
    return out


def engine_rates(packed: torch.Tensor, reps: int) -> dict:
    from pyscenedetect_b200.engine import F_HSV, Engine
    n, h, w, _ = packed.shape
    rgb = packed.flip(-1).contiguous()
    nchw = packed.permute(0, 3, 1, 2).contiguous()
    layouts = {"packed_bgr": (packed, "bgr"), "packed_rgb": (rgb, "rgb"), "nchw": (nchw.permute(0, 2, 3, 1), "bgr")}
    out = {}
    for size in [(w, h), (256, 144)]:
        key = "full_res" if size == (w, h) else "auto_downscaled_256x144"
        ref = None
        out[key] = {}
        for name, (frames, order) in layouts.items():
            eng = Engine(w, h, F_HSV, width=size[0], height=size[1], max_batch=256)

            def run():
                eng.reset()
                eng.submit(frames, channel_order=order)
                eng.sync()
            s = timed(run, reps)
            sums = eng.read_sums().tobytes()
            ref = sums if ref is None else ref
            out[key][name] = {"frames_per_s": round(n / s), "parity": sums == ref}
            eng.close()
    del rgb, nchw
    return out


def scene_rates(frames_dev: torch.Tensor, repeat: int) -> dict:
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.video import ArrayVideoStream
    from pyscenedetect_b200.engine import PinnedBuffer
    frames_host = frames_dev.cpu().numpy()
    pinned = PinnedBuffer(frames_host.nbytes)   # the public API's fastest host input (bench.py's e2e)
    frames_pinned = pinned.array.reshape(frames_host.shape)
    np.copyto(frames_pinned, frames_host)
    total = frames_dev.shape[0] * repeat
    out = {"frames": total}
    host_cuts = None
    for batch in (64, 2048):
        row = {}
        cuts = {}
        # the host runs' staging is 2 x batch frames of page-locked and device memory: 64 only (cuts do not depend
        # on the batch size)
        sources = (("device", frames_dev, False), ("host_pageable", frames_host, False),
                   ("host_pinned", frames_pinned, True))
        for where, src, is_pinned in sources[:3 if batch == 64 else 1]:
            def run():
                sm = SceneManager(batch_size=batch)
                sm.add_detector(ContentDetector())
                sm.detect_scenes(ArrayVideoStream(src, 30.0, pinned=is_pinned, repeat=repeat))
                torch.cuda.synchronize()
                return [c.frame_num for c in sm.get_cut_list()]
            run()   # warm-up: engine creation, staging buffers
            t0 = time.perf_counter()
            cuts[where] = run()
            row[where + "_frames_per_s"] = round(total / (time.perf_counter() - t0))
        host_cuts = cuts.get("host_pageable", host_cuts)
        row["parity_with_host"] = cuts["device"] == host_cuts and cuts.get("host_pinned", host_cuts) == host_cuts
        row["cuts"] = len(cuts["device"])
        out[f"batch_{batch}"] = row
    pinned.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024, help="resident 1080p frames for the gather and engine rates")
    ap.add_argument("--scene-frames", type=int, default=1000, help="distinct resident 1080p frames for SceneManager")
    ap.add_argument("--repeat", type=int, default=10, help="SceneManager reads the distinct frames this many times")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan
    info = card()
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    w, h = 1920, 1080
    packed = torch.empty((args.frames, h, w, 3), dtype=torch.uint8, device="cuda")
    synth_frames_device(packed.data_ptr(), ScenePlan(args.frames, seed=1, min_len=10, max_len=90).params, w, h)
    result = {"card": info, "gather_1080p": gather_rates(packed, args.reps), "engine_1080p_F_HSV": engine_rates(packed, args.reps)}
    del packed
    torch.cuda.empty_cache()
    scene = torch.empty((args.scene_frames, h, w, 3), dtype=torch.uint8, device="cuda")
    synth_frames_device(scene.data_ptr(), ScenePlan(args.scene_frames, seed=2, min_len=10, max_len=90).params, w, h)
    result["scene_manager_1080p_content"] = scene_rates(scene, args.repeat)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
