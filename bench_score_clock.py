#!/usr/bin/env python
"""Fused HSV pass against the SM clock: bench.py's workload shape (resident device-rendered frames, default
10 000 at 1920x1080, F_HSV, an engine with max_batch=2048) scored --steps times, with the SM clock and the power
draw sampled over the timed region.  A step takes tens of milliseconds, so the default timed region is 50 steps
long: long enough for a power-capped card to settle at the clock it holds under this load.

frames/s comes from the engine's CUDA events (`Engine.timing_ms`: score launches alone, and everything the
engine enqueued per step).  The pass is bound by instruction issue when the card runs below full clock (a
power-capped H100) and by HBM at full clock, so frames/s per MHz of median SM clock is the figure that
compares two builds across cards of different power limits while the clock sets the pace.  The clocks are
only queried (`nvidia-smi --query-gpu`); nothing is set.  Prints one JSON line; writes nothing.

    python bench_score_clock.py [--frames 10000] [--steps 50] [--warmup 5]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card_info(device: int) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, smax = [x.strip() for x in out.split(",")[:3]]
        return {"card": name, "power_limit_w": float(power), "sm_max_mhz": float(smax)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"card": None, "power_limit_w": None, "sm_max_mhz": None}


class Sampler:
    """SM clock and power draw every 25 ms from a read-only nvidia-smi query, kept for a time window."""

    def __init__(self, device: int):
        self.device = device
        self.samples: list[tuple[float, float, float]] = []   # (arrival time, MHz, W)
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits",
                                          "-lms", "25", "-i", str(self.device)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            return

        def pump():
            for line in self.proc.stdout:
                try:
                    mhz, watts = (float(x) for x in line.split(",")[:2])
                except ValueError:
                    continue
                self.samples.append((time.perf_counter(), mhz, watts))
        threading.Thread(target=pump, daemon=True).start()

    def stop(self, t0: float, t1: float) -> dict:
        if self.proc is None:
            return {"sm_mhz_median": None, "power_w_median": None, "samples": 0}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            self.proc.wait()
        # nvidia-smi takes ~0.1 s to start, so it runs from before the warm-up and is cut to the timed region here
        inside = [(m, w) for t, m, w in self.samples if t0 <= t <= t1]
        if not inside:
            return {"sm_mhz_median": None, "power_w_median": None, "samples": 0}
        return {"sm_mhz_median": statistics.median(m for m, _ in inside),
                "power_w_median": statistics.median(w for _, w in inside), "samples": len(inside)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=10000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--max-batch", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.frames < 1 or args.steps < 1 or args.warmup < 0:
        ap.error("--frames and --steps must be >= 1 and --warmup >= 0")

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import F_HSV, DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan

    lib = _capi.load()
    w, h, n = args.width, args.height, args.frames
    fbytes = w * h * 3
    buf = DeviceBuffer(n * fbytes, args.device)
    synth_frames_device(buf.ptr, ScenePlan(n, seed=args.seed).params, w, h, device=args.device)
    eng = Engine(w, h, F_HSV, device=args.device, max_batch=args.max_batch)

    def step() -> tuple[float, float, int]:
        eng.reset()
        eng.timing_reset()
        eng.submit_device(buf.ptr, n, fbytes)
        eng.sync()
        return eng.timing_ms()

    sampler = Sampler(args.device)
    sampler.start()
    for _ in range(args.warmup):
        step()
    launches0 = lib.psd_launch_count()
    total_ms = score_ms = 0.0
    score_launches = 0
    t0 = time.perf_counter()
    for _ in range(args.steps):
        tot, sc, k = step()
        total_ms += tot
        score_ms += sc
        score_launches += k
    t1 = time.perf_counter()
    clocks = sampler.stop(t0, t1)
    kernel_launches = lib.psd_launch_count() - launches0
    eng.close()
    buf.close()

    fps = n * args.steps / (score_ms / 1000.0)
    mhz = clocks["sm_mhz_median"]
    print(json.dumps({
        "bench": "score_clock", **card_info(args.device),
        "workload": f"F_HSV, {n} resident {w}x{h} frames per step, max_batch={args.max_batch}",
        "steps": args.steps, "warmup": args.warmup,
        "frames_per_s": fps,
        "frames_per_s_engine_total": n * args.steps / (total_ms / 1000.0),
        "score_launches_per_step": score_launches / args.steps,
        "kernel_launches_per_step": kernel_launches / args.steps,
        **clocks,
        "frames_per_s_per_mhz": fps / mhz if mhz else None,
    }))
    return 0


if __name__ == "__main__":
    sys.exit(main())
