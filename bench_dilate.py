#!/usr/bin/env python
"""Benchmark of the edge dilation (ContentDetector's cv2.dilate with a k x k box) over kernel sizes.

For each frame size and kernel size, --frames synthetic frames are rendered into HBM once and submitted --reps
times in batches of --batch.  Two numbers per row, both per frame:

* `edge_path_us`: the engine's CUDA events around each batch minus those around its score pass
  (`Engine.timing_ms`), i.e. thresholds, Canny classify, hysteresis, dilation and the edge SAD; median over reps;
* `dilate_us`: the device time of the dilation kernels alone, from one extra rep under torch.profiler (CUPTI
  kernel records): the register-ring kernel (k <= 17) or the two passes of the separable dilation (k >= 19).

Before timing, --check frames per row are compared with cv2.dilate(cv2.Canny(V)) (oracle/ref_detectors.py
`detect_edges`).  The card's name, power limit and the SM clock sampled during the runs are printed on the same
line.  Prints one JSON line; writes nothing.

    python bench_dilate.py [--frames 256] [--reps 3] [--ks 5,13,19,33,63,65,127,255,1023]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_hash import card_info, sm_clock  # noqa: E402

KS = "5,13,19,33,63,65,127,255,1023"
SHAPES = [(1920, 1080), (3840, 2160)]
DILATE_KERNELS = ("dilate", "hdil_rows", "vdil_cols")


def dilate_device_us(eng, buf_ptr: int, frames: int, batch: int, fbytes: int) -> float:
    """Device time of the dilation kernels of one pass over the frames, per frame (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    eng.reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f0 in range(0, frames, batch):
            eng.submit_device(buf_ptr + f0 * fbytes, min(batch, frames - f0), fbytes)
        eng.sync()
    total = 0.0
    for ev in prof.key_averages():
        if any(s in ev.key for s in DILATE_KERNELS):
            total += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    return total / frames


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=2)
    ap.add_argument("--ks", default=KS)
    ap.add_argument("--shapes", default=",".join(f"{w}x{h}" for w, h in SHAPES))
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)

    import cv2
    import numpy as np

    from oracle import ref_detectors as R
    from pyscenedetect_b200.engine import F_EDGES, DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan, render_frames

    ks = [int(x) for x in args.ks.split(",")]
    shapes = [tuple(int(v) for v in s.split("x")) for s in args.shapes.split(",")]
    plan = ScenePlan(args.frames, seed=5, min_len=10, max_len=40)
    rows, clocks = [], []
    for w, h in shapes:
        fbytes = w * h * 3
        buf = DeviceBuffer(args.frames * fbytes, args.device)
        synth_frames_device(buf.ptr, plan.params, w, h, device=args.device)
        host = render_frames(plan.params[:args.check], w, h) if args.check else None
        lums = [cv2.split(cv2.cvtColor(f, cv2.COLOR_BGR2HSV))[2] for f in host] if args.check else []
        for k in ks:
            row = {"width": w, "height": h, "k": k}
            if lums:
                chk = Engine(w, h, F_EDGES, device=args.device, max_batch=len(lums), edge_kernel_size=k)
                chk.submit(host)
                kernel = np.ones((k, k), np.uint8)
                row["checked_frames_equal_cv2"] = sum(
                    bool(np.array_equal(chk.debug_plane(3, j), R.detect_edges(lum, kernel))) for j, lum in enumerate(lums))
                row["checked_frames"] = len(lums)
                chk.close()
            eng = Engine(w, h, F_EDGES, device=args.device, max_batch=args.batch, edge_kernel_size=k)
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
                total, score, _ = eng.timing_ms()
                per.append(1000.0 * (total - score) / args.frames)
            row["edge_path_us"] = round(statistics.median(per), 3)
            row["edge_path_us_spread"] = [round(min(per), 3), round(max(per), 3)]
            try:
                row["dilate_us"] = round(dilate_device_us(eng, buf.ptr, args.frames, args.batch, fbytes), 3)
            except Exception as exc:   # torch or its profiler missing: the events above still stand
                row["dilate_us"] = f"not measured ({type(exc).__name__})"
            eng.close()
            rows.append(row)
            print(json.dumps(row), file=sys.stderr)
        buf.close()
    print(json.dumps({"bench": "edge_dilate", **card_info(args.device),
                      "sm_clock_samples": sorted(set(c for c in clocks if c)), "frames": args.frames,
                      "batch": args.batch, "reps": args.reps, "rows": rows}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
