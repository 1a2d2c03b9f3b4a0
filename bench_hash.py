#!/usr/bin/env python
"""Benchmark of HashDetector's per-frame hash pass (psd_hash_rows_kernel + psd_hash_finish_kernel) over hash sizes.

For each (size, lowpass) and frame size, --frames synthetic frames are rendered into HBM once and submitted
--reps times in batches of --batch; the device time per frame is the engine's CUDA-event time of its kernels
(`Engine.timing_ms`, median over the reps).  Next to it: the reference call sequence (oracle/ref_detectors.py
`hash_frame`: cv2 gray, INTER_AREA, cv2.dct, numpy.median) per frame on one host core, over --host-frames frames.
The card's power limit and the SM clock sampled during the device runs are part of the result.  Prints one
JSON line; writes nothing.

    python bench_hash.py [--frames 512] [--reps 5]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HASHES = [(8, 2), (16, 2), (32, 3), (64, 4), (256, 1)]
SHAPES = [(274, 154), (1920, 1080)]   # auto-downscaled 1080p, full 1080p


def card_info(device: int) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, smax = [x.strip() for x in out.split(",")[:3]]
        return {"card": name, "power_limit": power, "sm_max_clock": smax}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"card": None, "power_limit": None, "sm_max_clock": None}


def sm_clock(device: int) -> str | None:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i", str(device)],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-frames", type=int, default=8)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)

    import numpy as np

    from oracle import ref_detectors as R
    from pyscenedetect_b200.engine import F_HASH, DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan, render_frames

    plan = ScenePlan(args.frames, seed=5, min_len=10, max_len=40)
    rows = []
    clocks = []
    for w, h in SHAPES:
        fbytes = w * h * 3
        buf = DeviceBuffer(args.frames * fbytes, args.device)
        synth_frames_device(buf.ptr, plan.params, w, h, device=args.device)
        host = render_frames(plan.params[:args.host_frames], w, h)
        for size, lowpass in HASHES:
            n = size * lowpass
            row = {"width": w, "height": h, "size": size, "lowpass": lowpass, "n": n}
            if n > min(w, h):
                row["skipped"] = "frame smaller than the hash image"
                rows.append(row)
                continue
            eng = Engine(w, h, F_HASH, device=args.device, max_batch=args.batch, hash_size=size, hash_lowpass=lowpass)
            eng.submit_device(buf.ptr, min(args.batch, args.frames), fbytes)   # warm-up
            eng.sync()
            per = []
            for _ in range(args.reps):
                eng.reset()
                eng.timing_reset()
                for f0 in range(0, args.frames, args.batch):
                    eng.submit_device(buf.ptr + f0 * fbytes, min(args.batch, args.frames - f0), fbytes)
                eng.sync()
                clocks.append(sm_clock(args.device))
                per.append(1000.0 * eng.timing_ms()[1] / args.frames)
            eng.close()
            t0 = time.perf_counter()
            for f in host:
                R.hash_frame(f, size, lowpass)
            host_us = 1e6 * (time.perf_counter() - t0) / len(host)
            row.update(gpu_us_per_frame=round(statistics.median(per), 3), gpu_us_spread=[round(min(per), 3),
                       round(max(per), 3)], cv2_us_per_frame_one_core=round(host_us, 1))
            rows.append(row)
            print(json.dumps(row), file=sys.stderr)
        buf.close()
    print(json.dumps({"bench": "hash_pass", **card_info(args.device), "sm_clock_samples": sorted(set(c for c in clocks if c)),
                      "frames": args.frames, "batch": args.batch, "reps": args.reps, "rows": rows}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
