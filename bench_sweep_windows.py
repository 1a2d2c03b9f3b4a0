#!/usr/bin/env python
"""Benchmark of the parameter sweep with a window per clip (`ParameterSweep.run_clips(windows=...)`): each clip's crop,
duration and frame_skip under every setting in one read of each clip, against one run_clips per distinct window and one
sweep per clip.

The clips and windows are bench_clip_window_lists.py's: slices of a pool of synthetic 1280x720 frames rendered into HBM,
lengths in [48, 240] frames, rates from (24, 25, 30000/1001, 30), each with one of eight letterbox / pillarbox crops, a
duration of 1.0 to 4.0 s and a frame_skip of 0 to 2; the first --host-clips of them are also read from a pageable host
copy of the pool.  Ground truth is each slice's ScenePlan cuts over the whole slice, past the window's end too.  For a
ContentDetector grid and an AdaptiveDetector grid of --cells cells (bench_sweep.py's grid builders) under the two
settings of SETTINGS, three arms run alternately for --rounds rounds (best time reported), each timed on the host clock
around work that ends in a device synchronise:

  windows      one ParameterSweep(settings=SETTINGS).run_clips(windows=...) over every clip
  per_window   one sweep per distinct window, its crop and frame_skip added to every setting, run_clips(duration=) over
               the clips that have it
  per_clip     the same sweep per clip

Reported per arm: clips/s and library launches per clip (psd_launch_count).  `equal` is true when every (setting, cell,
clip) count, cut list sample and end frame, and every cell total, is the same in every arm.  Prints one JSON line per
(detector, input); writes nothing.

    python bench_sweep_windows.py [--clips 1000] [--host-clips 20] [--cells 64] [--rounds 2]
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

from bench_clip_window_lists import clip_windows  # noqa: E402
from bench_sweep_settings import RATES, counts  # noqa: E402

SETTINGS = [{}, {"auto_downscale": False, "downscale": 4}]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=20)
    ap.add_argument("--cells", type=int, default=64)
    ap.add_argument("--tolerances", default="0,1")
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the three arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1 or args.host_clips < 0 or args.rounds < 1 or args.cells < 1:
        ap.error("--pool must be >= 240, --clips, --cells and --rounds >= 1, --host-clips >= 0")

    import torch

    from bench_clips import card_info
    from bench_sweep import adaptive_grid, content_grid
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_sweep_windows.py needs a CUDA device")
    dev, w, h, bs = args.device, 1280, 720, args.batch_size
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
    pool_cuts = np.asarray(plan.cut_frames, dtype=np.int64)
    gts = [GroundTruth([int(c) - s for c in pool_cuts if s < c < s + n]) for s, n in zip(starts, lengths)]
    tols = tuple(int(t) for t in args.tolerances.split(","))
    n_set = len(SETTINGS)

    def streams(k, src):
        return [ArrayVideoStream(src[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def sweep(cls, grid, settings):
        # clips are at most 240 frames: no cell can emit more than 256 cuts in one
        return ParameterSweep(cls, grid, tolerances=tols, batch_size=bs, device=dev, max_cuts_per_cell=256,
                              settings=settings)

    def with_window(wd):
        return [{**s, "crop": wd["crop"], "frame_skip": wd["frame_skip"]} for s in SETTINGS]

    status = 0
    inputs = [("cuda", pool, args.clips)] + ([("host", host_pool, args.host_clips)] if args.host_clips else [])
    for det, cls, make in (("content", ContentDetector, content_grid), ("adaptive", AdaptiveDetector, adaptive_grid)):
        grid = make(args.cells)
        g = len(grid)
        for src_name, src, n_clips in inputs:
            by_window = {}
            for i, wd in enumerate(windows[:n_clips]):
                by_window.setdefault(tuple(sorted(wd.items())), []).append(i)

            def together():
                sw = sweep(cls, grid, SETTINGS)
                r = sw.run_clips(streams(n_clips, src), gts[:n_clips], windows=windows[:n_clips])
                return [(r, list(range(n_clips)))], [sw]

            def apart(groups):
                videos = streams(n_clips, src)
                out, sws = [], []
                for idx in groups:
                    wd = windows[idx[0]]
                    sw = sweep(cls, grid, with_window(wd))
                    r = sw.run_clips([videos[i] for i in idx], [gts[i] for i in idx], duration=wd["duration"])
                    out.append((r, idx))
                    sws.append(sw)
                return out, sws

            arms = {"windows": together, "per_window": lambda: apart(list(by_window.values())),
                    "per_clip": lambda: apart([[i] for i in range(n_clips)])}
            warm = streams(4, src)  # first engines, allocator pools
            sweep(cls, grid, SETTINGS).run_clips(warm, gts[:4], windows=windows[:4])
            for i in range(4):
                sweep(cls, grid, with_window(windows[i])).run_clips(streams(4, src)[i:i + 1], gts[i:i + 1],
                                                                    duration=windows[i]["duration"])
            torch.cuda.synchronize()
            best, seen = {}, {}
            for _ in range(args.rounds):
                for name, fn in arms.items():
                    l0 = lib.psd_launch_count()
                    t0 = time.perf_counter()
                    got = fn()
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    launches = lib.psd_launch_count() - l0
                    seen[name] = got
                    if name not in best or dt < best[name]["s"]:
                        best[name] = {"s": dt, "launches": launches}

            def table(arm):
                """(setting * cells + cell, clip) counts, end frames [setting][clip], summed cell totals, sample cuts."""
                results, sws = seen[arm]
                c = np.zeros((n_set * g, n_clips, len(tols) * 5 + 4), dtype=np.int64)
                ends = np.zeros((n_set, n_clips), dtype=np.int64)
                cuts = {}
                for r, idx in results:
                    c[:, idx] = counts(r, n_set * g, len(idx), tols)
                    for jj, j in enumerate(idx):
                        ends[:, j] = [r.end_frame(jj, setting=s) for s in range(n_set)]
                        if j % 13 == 0:
                            cuts[j] = [r.cuts(k, jj) for k in range(0, n_set * g, 7)]
                tot = np.zeros((n_set * g, len(tols) * 5 + 3))
                for sw in sws:
                    tot += [[x for t in tols for x in (t_.hard[t].matched, t_.hard[t].false_positives,
                                                       t_.hard[t].missed, *t_.hard_offset[t])]
                            + [t_.fades.matched, t_.fades.false_positives, t_.fades.missed] for t_ in sw.totals()]
                return c, ends, tot, cuts

            ref = table("windows")
            equal = True
            for name in ("per_window", "per_clip"):
                other = table(name)
                equal = equal and all(np.array_equal(a, b) for a, b in zip(ref[:3], other[:3])) and ref[3] == other[3]
            result = {"bench": "sweep_windows", **card, "detector": det, "cells": g, "settings": n_set,
                      "input": src_name, "size": f"{w}x{h}", "batch_size": bs, "clips": n_clips,
                      "distinct_windows": len(by_window), "frames": int(sum(lengths[:n_clips])),
                      "tolerances": list(tols), "rounds": args.rounds, "arms": {}}
            for name, b in best.items():
                result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(n_clips / b["s"], 1),
                                        "launches_per_clip": round(b["launches"] / n_clips, 2)}
            result["speedup_vs_per_window"] = round(best["per_window"]["s"] / best["windows"]["s"], 2)
            result["speedup_vs_per_clip"] = round(best["per_clip"]["s"] / best["windows"]["s"], 2)
            result["equal"] = bool(equal)
            print(json.dumps(result), flush=True)
            status |= 0 if equal else 1
    return status


if __name__ == "__main__":
    sys.exit(main())
