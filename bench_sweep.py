#!/usr/bin/env python
"""Benchmark of the device parameter sweep (pyscenedetect_b200/sweep.py).

10 000 synthetic 1080p frames are rendered into HBM and scored once (ContentDetector's HSV pass at full
size).  Then, for G in --cells, a grid of G ContentDetector cells and one of G AdaptiveDetector cells is
evaluated with the ScenePlan's cuts as ground-truth hard cuts: the timed grid stage is the metric scans +
psd_sweep_cuts + psd_sweep_eval (host clock ending in a device sync).  The same cells then run as a loop of
single-cell `DeviceCuts` calls in this process; `parity` is true when every cell's batched counts equal
the host evaluation (tests/sweep_model.py) of its single-cell cuts.  Prints one JSON line; writes nothing.

    python bench_sweep.py [--frames 10000] [--cells 1,64,1024,8192] [--reps 3]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card_info(device: int) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return {"card": name, "power_limit": power}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"card": None, "power_limit": None}


def content_grid(g: int) -> list[dict]:
    msl = (0, 5, 10, 15, 30, 60, 90, 120)
    return [dict(threshold=8.0 + 50.0 * (i // len(msl)) / max(1, g // len(msl)), min_scene_len=msl[i % len(msl)])
            for i in range(g)]


def adaptive_grid(g: int) -> list[dict]:
    keys = [(w, m) for w in (1, 2, 3, 4) for m in (5.0, 10.0, 15.0, 20.0)]
    per = -(-g // len(keys))
    return [dict(window_width=keys[i // per][0], min_content_val=keys[i // per][1],
                 adaptive_threshold=1.5 + 3.0 * (i % per) / per, min_scene_len=(0, 15)[i % 2]) for i in range(g)]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=10000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--cells", default="1,64,1024,8192")
    ap.add_argument("--tolerances", default="0,1")
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of each grid stage (median reported)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.frames < 2 or args.reps < 1:
        ap.error("--frames must be >= 2 and --reps >= 1")

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    from pyscenedetect_b200.device_cuts import DeviceCuts, cuts_for_detector
    from pyscenedetect_b200.engine import DeviceBuffer, synth_frames_device
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan
    from tests import sweep_model

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_sweep.py needs a CUDA device")
    n, w, h, dev = args.frames, args.width, args.height, args.device
    fps = 30.0
    cells = [int(x) for x in args.cells.split(",")]
    tols = tuple(int(x) for x in args.tolerances.split(","))
    plan = ScenePlan(n, seed=0)
    gt = GroundTruth(plan.cut_frames)
    fbytes = w * h * 3
    frames = DeviceBuffer(n * fbytes, dev)  # resident in HBM
    for i in range(0, n, 1000):
        synth_frames_device(frames.ptr + i * fbytes, plan.params[i:i + 1000], w, h, device=dev)

    result = {"bench": "sweep", **card_info(dev), "frames": n, "size": f"{w}x{h}", "tolerances": list(tols),
              "cells": cells, "grid": {}}
    probe = ParameterSweep(ContentDetector, [{}], device=dev)
    engine = probe.groups[0].make_engine(w, h, w, h, device=dev, max_batch=256)
    engine.submit_device(frames.ptr, min(n, 256), fbytes)  # warm-up of the score pass
    engine.sync()
    engine.reset()
    t0 = time.perf_counter()
    engine.submit_device(frames.ptr, n, fbytes)
    engine.sync()
    result["score_pass_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    frames.close()

    parity = True
    for name, cls, make in (("content", ContentDetector, content_grid), ("adaptive", AdaptiveDetector, adaptive_grid)):
        per = {}
        for g in cells:
            grid = make(g)
            sw = ParameterSweep(cls, grid, tolerances=tols, device=dev, max_cuts_per_cell=n)
            assert len(sw.groups) == 1 and sw.groups[0] == probe.groups[0]
            sw.run_scored([engine], fps, gt)  # warm-up
            times = []
            for _ in range(args.reps):
                r = sw.run_scored([engine], fps, gt)
                times.append(r.grid_ms)
            grid_ms = sorted(times)[len(times) // 2]
            dc = DeviceCuts(engine, max_cuts=n)
            t0 = time.perf_counter()
            single = [cuts_for_detector(dc, cls(**kw), fps) for kw in grid]
            loop_ms = (time.perf_counter() - t0) * 1e3
            for k, raw in enumerate(single):
                pred = sweep_model.predicted_list(raw, n)
                ok = r.cuts(k) == pred if k < 64 else r.raw_count(k) == len(raw)
                for t in tols:
                    want_h, _ = sweep_model.score(pred, gt.hard_cuts, [], t)
                    ok = ok and (*r.hard(k, t), int(r.hard_offset(k, t)[0]), r.hard_offset(k, t)[1]) == want_h
                parity = parity and bool(ok)
            per[str(g)] = {"grid_ms": round(grid_ms, 3), "single_cell_loop_ms": round(loop_ms, 3),
                           "cell_frames_per_s": round(g * n / (grid_ms / 1e3), 1),
                           "metric_arrays": len(sw.metric_keys)}
        result["grid"][name] = per
    result["parity"] = parity
    engine.close()
    print(json.dumps(result))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
