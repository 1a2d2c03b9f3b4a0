#!/usr/bin/env python
"""Benchmark of windowed many-clip detection: `detect_clips(..., crop=, duration=, frame_skip=)` against one
`SceneManager` per clip running `detect_scenes` with the same window and crop.

The clips are those of bench_clips.py: slices of a pool of synthetic 1280x720 frames rendered into HBM, with seeded
lengths in [48, 240] frames and rates from (24, 25, 30000/1001, 30); ContentDetector() + AdaptiveDetector(),
auto-downscaled.  Four windows: frame_skip=1, duration="2s", a crop (a 1200x640 box), and the three together.
Two inputs: CUDA clips read as views of the pool, and host clips (numpy slices of a pageable copy of the pool; fewer
of them, since one SceneManager per host clip is slow).  The two arms are alternated within the run, each timed on
the host clock and ending with every result on the host.

Reported per window and input: clips/s, frames read/s and library launches per clip (psd_launch_count) of both arms.
`equal` is true when every clip's frame count, cut list, scene list and end position are the same in both arms, in
every round.  Prints one JSON line per window and input; writes nothing.

    python bench_clip_windows.py [--clips 1000] [--host-clips 20] [--pool 1024] [--rounds 2]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_clips import RATES, card_info, detectors  # noqa: E402

CROP = (40, 40, 1239, 679)  # inclusive: 1200x640, the bars of a letterboxed frame cut away
WINDOWS = {
    "frame_skip_1": dict(frame_skip=1),
    "duration_2s": dict(duration="2s"),
    "crop": dict(crop=CROP),
    "all_three": dict(frame_skip=1, duration="2s", crop=CROP),
}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=20)
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the two arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1 or args.host_clips < 0 or args.rounds < 1:
        ap.error("--pool must be >= 240, --clips and --rounds >= 1, --host-clips >= 0")

    import torch

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_clip_windows.py needs a CUDA device")
    dev, w, h, bs = args.device, args.width, args.height, args.batch_size
    card = card_info(dev)
    torch.cuda.set_device(dev)
    fb = w * h * 3
    pool = torch.empty((args.pool, h, w, 3), dtype=torch.uint8, device=f"cuda:{dev}")
    plan = ScenePlan(args.pool, seed=args.seed)
    for i in range(0, args.pool, 256):
        synth_frames_device(pool.data_ptr() + i * fb, plan.params[i:i + 256], w, h, device=dev)
    torch.cuda.synchronize()
    host_pool = pool.cpu().numpy() if args.host_clips else None
    rng = np.random.default_rng(args.seed)
    n_max = max(args.clips, args.host_clips)
    lengths = rng.integers(48, 241, size=n_max)
    starts = [int(rng.integers(0, args.pool - n + 1)) for n in lengths]
    rates = [RATES[i % len(RATES)] for i in range(n_max)]

    def streams(k, src):
        return [ArrayVideoStream(src[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def batched(window):
        def run(videos):
            res = detect_clips(videos, detectors(), batch_size=bs, device=dev, **window)
            return [(r.frames, r.cut_frames, [(a.frame_num, b.frame_num) for a, b in r.scene_list()],
                     r.end.frame_num if r.end is not None else None) for r in res]
        return run

    def per_clip(window):
        kw = {k: v for k, v in window.items() if k != "crop"}

        def run(videos):
            out = []
            for v in videos:
                sm = SceneManager(device=dev, batch_size=bs)
                sm.crop = window.get("crop")
                for d in detectors():
                    sm.add_detector(d)
                n = sm.detect_scenes(v, **kw)
                out.append((n, [c.frame_num for c in sm.get_cut_list()],
                            [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list()],
                            sm._last_pos.frame_num if sm._last_pos is not None else None))
            return out
        return run

    status = 0
    inputs = [("cuda", pool, args.clips)] + ([("host", host_pool, args.host_clips)] if args.host_clips else [])
    for wname, window in WINDOWS.items():
        for src_name, src, n_clips in inputs:
            arms = {"clips": batched(window), "per_clip": per_clip(window)}
            for fn in arms.values():  # warm-up: library load, first engines, allocator pools
                fn(streams(4, src))
            torch.cuda.synchronize()
            best, seen, stable = {}, {}, True
            for _ in range(args.rounds):
                for name, fn in arms.items():
                    videos = streams(n_clips, src)
                    l0 = lib.psd_launch_count()
                    t0 = time.perf_counter()
                    got = fn(videos)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    launches = lib.psd_launch_count() - l0
                    stable = stable and seen.setdefault(name, got) == got
                    if name not in best or dt < best[name]["s"]:
                        best[name] = {"s": dt, "launches": launches}
            equal = seen["clips"] == seen["per_clip"] and stable
            frames = sum(r[0] for r in seen["clips"])
            result = {"bench": "clip_windows", **card, "window": wname,
                      "args": {k: list(v) if isinstance(v, tuple) else v for k, v in window.items()},
                      "input": src_name, "size": f"{w}x{h}", "detectors": "ContentDetector() + AdaptiveDetector()",
                      "batch_size": bs, "clips": n_clips, "frames_read": frames, "rounds": args.rounds, "arms": {}}
            for name, b in best.items():
                result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(n_clips / b["s"], 1),
                                        "frames_read_per_s": round(frames / b["s"], 1),
                                        "launches_per_clip": round(b["launches"] / n_clips, 2)}
            result["speedup_vs_per_clip"] = round(best["per_clip"]["s"] / best["clips"]["s"], 2)
            result["equal"] = bool(equal)
            print(json.dumps(result), flush=True)
            status |= 0 if equal else 1
    return status


if __name__ == "__main__":
    sys.exit(main())
