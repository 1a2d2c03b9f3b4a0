#!/usr/bin/env python
"""Benchmark of many-clip detection with a window per clip: `detect_clips(..., windows=[...])` against one
`detect_clips` call per distinct window and one `SceneManager` per clip.

The clips are those of bench_clips.py: slices of a pool of synthetic 1280x720 frames rendered into HBM, with seeded
lengths in [48, 240] frames and rates from (24, 25, 30000/1001, 30); ContentDetector() + AdaptiveDetector(),
auto-downscaled.  Each clip gets a seeded window: one of eight letterbox / pillarbox crops, a duration drawn from
1.0 to 4.0 s in tenths, and a frame_skip of 0, 1 or 2, as a dataset manifest of mixed sources and segments gives
them.  Two inputs: CUDA clips read as views of the pool, and the first --host-clips clips as numpy slices of a
pageable copy of the pool.  The three arms are alternated within the run, each timed on the host clock and ending with
every result on the host:

  windows      one detect_clips(videos, windows=...) over every clip
  per_window   one detect_clips(crop=, duration=, frame_skip=) per distinct window, over the clips that have it
  per_clip     a fresh SceneManager + detectors per clip, running detect_scenes with the clip's window and crop

Reported per input: clips/s, frames read/s and library launches per clip (psd_launch_count) of every arm, and the
number of distinct windows.  `equal` is true when every clip's frame count, cut list, scene list and end position are
the same in every arm, in every round.  Prints one JSON line per input; writes nothing.

    python bench_clip_window_lists.py [--clips 1000] [--host-clips 20] [--pool 1024] [--rounds 2]
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

# inclusive (X0, Y0, X1, Y1) boxes of a 1280x720 frame: 1.85:1, 2.39:1, 2.2:1, 2:1 and 2.13:1 letterboxes, a 4:3
# pillarbox, the 1200x640 box of bench_clip_windows.py and the whole frame
CROPS = [(0, 14, 1279, 705), (0, 92, 1279, 627), (0, 69, 1279, 650), (0, 40, 1279, 679), (0, 60, 1279, 659),
         (160, 0, 1119, 719), (40, 40, 1239, 679), (0, 0, 1279, 719)]


def clip_windows(n: int, seed: int) -> list:
    rng = np.random.default_rng(seed + 1)
    return [{"crop": CROPS[int(rng.integers(len(CROPS)))], "duration": round(float(rng.integers(10, 41)) / 10, 1),
             "frame_skip": int(rng.integers(0, 3))} for _ in range(n)]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=20)
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the three arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1 or args.host_clips < 0 or args.rounds < 1:
        ap.error("--pool must be >= 240, --clips and --rounds >= 1, --host-clips >= 0")
    if (args.width, args.height) != (1280, 720):
        ap.error("the crops are boxes of a 1280x720 frame")

    import torch

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_clip_window_lists.py needs a CUDA device")
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
    windows = clip_windows(n_max, args.seed)

    def streams(k, src):
        return [ArrayVideoStream(src[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def summary(r):
        return (r.frames, r.cut_frames, [(a.frame_num, b.frame_num) for a, b in r.scene_list()],
                r.end.frame_num if r.end is not None else None)

    def with_windows(videos):
        res = detect_clips(videos, detectors(), batch_size=bs, device=dev, windows=windows[:len(videos)])
        return [summary(r) for r in res]

    def per_window(videos):
        by = {}
        for i, wd in enumerate(windows[:len(videos)]):
            by.setdefault(tuple(sorted(wd.items())), []).append(i)
        out = [None] * len(videos)
        for key, idx in by.items():
            res = detect_clips([videos[i] for i in idx], detectors(), batch_size=bs, device=dev, **dict(key))
            for i, r in zip(idx, res):
                out[i] = summary(r)
        return out

    def per_clip(videos):
        out = []
        for v, wd in zip(videos, windows):
            sm = SceneManager(device=dev, batch_size=bs)
            sm.crop = wd["crop"]
            for d in detectors():
                sm.add_detector(d)
            n = sm.detect_scenes(v, duration=wd["duration"], frame_skip=wd["frame_skip"])
            out.append((n, [c.frame_num for c in sm.get_cut_list()],
                        [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list()],
                        sm._last_pos.frame_num if sm._last_pos is not None else None))
        return out

    status = 0
    inputs = [("cuda", pool, args.clips)] + ([("host", host_pool, args.host_clips)] if args.host_clips else [])
    arms = {"windows": with_windows, "per_window": per_window, "per_clip": per_clip}
    for src_name, src, n_clips in inputs:
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
        equal = stable and seen["windows"] == seen["per_window"] == seen["per_clip"]
        frames = sum(r[0] for r in seen["windows"])
        distinct = len({tuple(sorted(wd.items())) for wd in windows[:n_clips]})
        result = {"bench": "clip_window_lists", **card, "input": src_name, "size": f"{w}x{h}",
                  "detectors": "ContentDetector() + AdaptiveDetector()", "batch_size": bs, "clips": n_clips,
                  "distinct_windows": distinct, "frames_read": frames, "rounds": args.rounds, "arms": {}}
        for name, b in best.items():
            result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(n_clips / b["s"], 1),
                                    "frames_read_per_s": round(frames / b["s"], 1),
                                    "launches_per_clip": round(b["launches"] / n_clips, 2)}
        result["speedup_vs_per_window"] = round(best["per_window"]["s"] / best["windows"]["s"], 2)
        result["speedup_vs_per_clip"] = round(best["per_clip"]["s"] / best["windows"]["s"], 2)
        result["equal"] = bool(equal)
        print(json.dumps(result), flush=True)
        status |= 0 if equal else 1
    return status


if __name__ == "__main__":
    sys.exit(main())
