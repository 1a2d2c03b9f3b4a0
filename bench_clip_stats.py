#!/usr/bin/env python
"""Benchmark of per-frame metrics over many clips: `detect_clips(stats=True)` against one
`SceneManager(StatsManager())` per clip that saves its CSV.

The clips are those of bench_clips.py: slices of a pool of synthetic 1280x720 frames rendered into HBM, with seeded
lengths in [48, 240] frames and rates from (24, 25, 30000/1001, 30); ContentDetector() + AdaptiveDetector(),
auto-downscaled to 256x144.  Three arms, alternated within the run, each timed on the host clock and ending with
every result on the host:

  clips_stats      detect_clips(stats=True): cut lists and every clip's CSV bytes
  clips            detect_clips(stats=False): cut lists only
  per_clip_stats   a fresh SceneManager(StatsManager()) + detectors per clip, then save_to_csv into memory

Reported per arm: clips/s, frames/s and library launches per clip (psd_launch_count).  `equal` is true when every
clip's CSV bytes are the same in both stats arms, and every cut list the same in all three, in every round.
Prints one JSON line; writes nothing.

    python bench_clip_stats.py [--clips 1000] [--pool 1024] [--rounds 2]
"""

from __future__ import annotations

import argparse
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_clips import RATES, card_info, detectors  # noqa: E402


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the three arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1 or args.rounds < 1:
        ap.error("--pool must be >= 240, --clips and --rounds >= 1")

    import torch

    from pyscenedetect_b200 import StatsManager, _capi
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_clip_stats.py needs a CUDA device")
    dev, w, h, bs = args.device, args.width, args.height, args.batch_size
    card = card_info(dev)
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

    def streams(k):
        return [ArrayVideoStream(pool[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def batched(stats):
        def run(videos):
            res = detect_clips(videos, detectors(), batch_size=bs, device=dev, stats=stats)
            return [r.cut_frames for r in res], [r.stats_csv for r in res]
        return run

    def per_clip(videos):
        cuts, texts = [], []
        for v in videos:
            sm = SceneManager(StatsManager(), device=dev, batch_size=bs)
            for d in detectors():
                sm.add_detector(d)
            sm.detect_scenes(v)
            f = io.StringIO()
            sm.stats_manager.save_to_csv(f)
            cuts.append([c.frame_num for c in sm.get_cut_list()])
            texts.append(f.getvalue().encode())
        return cuts, texts

    arms = {"clips_stats": batched(True), "clips": batched(False), "per_clip_stats": per_clip}
    for fn in arms.values():  # warm-up: library load, first engines, allocator pools
        fn(streams(4))
    torch.cuda.synchronize()

    best, seen, stable = {}, {}, True
    for _ in range(args.rounds):
        for name, fn in arms.items():
            videos = streams(args.clips)
            l0 = lib.psd_launch_count()
            t0 = time.perf_counter()
            got = fn(videos)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            launches = lib.psd_launch_count() - l0
            stable = stable and seen.setdefault(name, got) == got
            if name not in best or dt < best[name]["s"]:
                best[name] = {"s": dt, "launches": launches}
    equal = (seen["clips_stats"][1] == seen["per_clip_stats"][1]
             and seen["clips_stats"][0] == seen["clips"][0] == seen["per_clip_stats"][0] and stable)
    frames = int(lengths.sum())
    texts = seen["clips_stats"][1]
    result = {"bench": "clip_stats", **card, "size": f"{w}x{h}", "scored": "256x144",
              "detectors": "ContentDetector() + AdaptiveDetector()", "batch_size": bs, "pool_frames": args.pool,
              "clips": args.clips, "frames": frames, "rounds": args.rounds,
              "csv_rows": sum(t.count(b"\n") - 1 for t in texts), "csv_bytes": sum(len(t) for t in texts), "arms": {}}
    for name, b in best.items():
        result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(args.clips / b["s"], 1),
                                "frames_per_s": round(frames / b["s"], 1),
                                "launches_per_clip": round(b["launches"] / args.clips, 2)}
    result["speedup_vs_per_clip"] = round(best["per_clip_stats"]["s"] / best["clips_stats"]["s"], 2)
    result["stats_cost_vs_clips"] = round(best["clips_stats"]["s"] / best["clips"]["s"], 2)
    result["equal"] = bool(equal)
    print(json.dumps(result))
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
