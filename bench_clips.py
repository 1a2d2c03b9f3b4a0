#!/usr/bin/env python
"""Benchmark of many-clip detection (pyscenedetect_b200/clips.py) against one SceneManager per clip.

A pool of synthetic 1280x720 frames is rendered into HBM by psd_synth_frames; each clip is an `ArrayVideoStream`
over a slice of the pool, with a seeded length in [48, 240] frames and a frame rate from (24, 25, 30000/1001, 30).
The detectors are ContentDetector() + AdaptiveDetector(), auto-downscaled (to 256x144).  Four arms, alternated within
the run, each timed on the host clock ending in a device synchronise:

  clips_cuda       detect_clips over the CUDA clips
  per_clip_cuda    a fresh SceneManager + detectors per CUDA clip
  clips_host       detect_clips over page-locked host copies of the clips
  per_clip_host    a fresh SceneManager + detectors per page-locked host clip

Host arms run the first --host-clips clips, as slices of a page-locked copy of the pool (their frames cross
PCIe).  Reported per arm: clips/s, frames/s and library launches per clip (psd_launch_count); `equal` is true
when every clip's cut list is the same in every arm and every round.
Prints one JSON line; writes nothing.

    python bench_clips.py [--clips 1000] [--host-clips 100] [--pool 1024] [--rounds 2]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RATES = (24, 25, Fraction(30000, 1001), 30)


def card_info(device: int) -> dict:
    """Name, power limit and maximum SM clock of the card, read in one nvidia-smi call."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")[:3]]
        return {"card": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"card": None, "power_limit": None, "max_sm_clock": None}


def detectors():
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    return [ContentDetector(), AdaptiveDetector()]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=100)
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the four arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1 or args.rounds < 1:
        ap.error("--pool must be >= 240, --clips and --rounds >= 1")

    import torch

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.engine import PinnedBuffer, synth_frames_device
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_clips.py needs a CUDA device")
    dev, w, h, bs = args.device, args.width, args.height, args.batch_size
    torch.cuda.set_device(dev)
    fb = w * h * 3
    pool = torch.empty((args.pool, h, w, 3), dtype=torch.uint8, device=f"cuda:{dev}")
    plan = ScenePlan(args.pool, seed=args.seed)
    for i in range(0, args.pool, 256):
        synth_frames_device(pool.data_ptr() + i * fb, plan.params[i:i + 256], w, h, device=dev)
    torch.cuda.synchronize()
    rng = np.random.default_rng(args.seed)
    lengths = rng.integers(48, 241, size=args.clips)
    starts = [int(rng.integers(0, args.pool - n + 1)) for n in lengths]
    rates = [RATES[i % len(RATES)] for i in range(args.clips)]
    n_host = min(args.host_clips, args.clips)
    host_frames = int(lengths[:n_host].sum())
    pinned = PinnedBuffer(args.pool * fb)  # a page-locked copy of the pool: host clips are slices of it
    host_pool = pinned.array.reshape(args.pool, h, w, 3)
    for i in range(0, args.pool, 256):
        host_pool[i:i + 256] = pool[i:i + 256].cpu().numpy()

    def cuda_streams(k):
        return [ArrayVideoStream(pool[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def host_streams(k):
        return [ArrayVideoStream(host_pool[s:s + n], fps, pinned=True)
                for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def batched(streams):
        return [r.cut_frames for r in detect_clips(streams, detectors(), batch_size=bs, device=dev)]

    def per_clip(streams):
        out = []
        for v in streams:
            sm = SceneManager(device=dev, batch_size=bs)
            for d in detectors():
                sm.add_detector(d)
            sm.detect_scenes(v)
            out.append([c.frame_num for c in sm.get_cut_list()])
        return out

    arms = {"clips_cuda": (batched, cuda_streams, args.clips), "per_clip_cuda": (per_clip, cuda_streams, args.clips),
            "clips_host": (batched, host_streams, n_host), "per_clip_host": (per_clip, host_streams, n_host)}
    for fn, make, _ in arms.values():  # warm-up: library load, first engines, allocator pools
        fn(make(4))
    torch.cuda.synchronize()

    best, cuts, stable = {}, {}, True
    for _ in range(args.rounds):
        for name, (fn, make, k) in arms.items():
            streams = make(k)
            l0 = lib.psd_launch_count()
            t0 = time.perf_counter()
            got = fn(streams)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            launches = lib.psd_launch_count() - l0
            stable = stable and cuts.setdefault(name, got) == got
            if name not in best or dt < best[name]["s"]:
                best[name] = {"s": dt, "launches": launches}
    equal = (cuts["clips_cuda"] == cuts["per_clip_cuda"] and cuts["clips_host"] == cuts["per_clip_host"]
             and cuts["clips_host"] == cuts["clips_cuda"][:n_host] and stable)
    total = {"cuda": int(lengths.sum()), "host": host_frames}
    result = {"bench": "clips", **card_info(dev), "size": f"{w}x{h}", "scored": "256x144",
              "detectors": "ContentDetector() + AdaptiveDetector()", "batch_size": bs, "pool_frames": args.pool,
              "clips": {"cuda": args.clips, "host": n_host}, "frames": total, "rounds": args.rounds, "arms": {}}
    for name, b in best.items():
        k = arms[name][2]
        f = total["host" if name.endswith("host") else "cuda"]
        result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(k / b["s"], 1),
                                "frames_per_s": round(f / b["s"], 1), "launches_per_clip": round(b["launches"] / k, 2)}
    result["speedup_cuda"] = round(best["per_clip_cuda"]["s"] / best["clips_cuda"]["s"], 2)
    result["speedup_host"] = round(best["per_clip_host"]["s"] / best["clips_host"]["s"], 2)
    result["cuts_total"] = sum(len(c) for c in cuts["clips_cuda"])
    result["equal"] = bool(equal)
    pinned.close()
    print(json.dumps(result))
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
