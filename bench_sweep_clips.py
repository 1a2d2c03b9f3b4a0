#!/usr/bin/env python
"""Benchmark of the parameter sweep over many clips (`ParameterSweep.run_clips`) against a loop of
`ParameterSweep.run`, one call per clip.

The clip set is bench_clips.py's: a pool of synthetic 1280x720 frames rendered into HBM by psd_synth_frames, and
--clips `ArrayVideoStream`s over slices of it with seeded lengths in [48, 240] frames and rates from
(24, 25, 30000/1001, 30), auto-downscaled (to 256x144).  Each clip's ground truth is its ScenePlan's cuts inside the
slice.  For G in --cells, a grid of G ContentDetector cells and one of G AdaptiveDetector cells (bench_sweep.py's grid
builders) run in two arms, each timed on the host clock around work that ends in a device synchronise:

  run_clips   one ParameterSweep.run_clips over every clip
  run_loop    a loop of ParameterSweep.run, one call per clip

Reported per arm: clips/s, frames/s and library launches per clip (psd_launch_count).  `parity` is true when every
(cell, clip) count (cut list, raw count, hard counts and offsets at every tolerance, fade counts) and every cell total
is equal between the two arms.  Prints one JSON line; writes nothing.

    python bench_sweep_clips.py [--clips 1000] [--cells 1,64,1024] [--pool 1024]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RATES = (24, 25, Fraction(30000, 1001), 30)


def _hard_arrays(r, n_cells, n_clips, tols, per_clip: bool):
    """Every (cell, clip) count as one int64 array, for the parity check; from a ClipSweepResult (per_clip False) or
    from a list of per-clip SweepResults."""
    out = np.zeros((n_cells, n_clips, len(tols) * 5 + 4), dtype=np.int64)
    for j in range(n_clips):
        for k in range(n_cells):
            at = (k,) if per_clip else (k, j)
            res = r[j] if per_clip else r
            row = []
            for t in tols:
                row += [*res.hard(*at, t), *res.hard_offset(*at, t)]
            out[k, j] = row + [*res.fades(*at), res.raw_count(*at)]
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--cells", default="1,64,1024")
    ap.add_argument("--tolerances", default="0,1")
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or args.clips < 1:
        ap.error("--pool must be >= 240 and --clips >= 1")

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
        raise SystemExit("bench_sweep_clips.py needs a CUDA device")
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
    pool_cuts = np.asarray(plan.cut_frames, dtype=np.int64)
    gts = [GroundTruth([int(c) - s for c in pool_cuts if s < c < s + n]) for s, n in zip(starts, lengths)]
    tols = tuple(int(t) for t in args.tolerances.split(","))
    frames_total = int(lengths.sum())

    def streams(k):
        return [ArrayVideoStream(pool[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def timed(fn):
        l0 = lib.psd_launch_count()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0, lib.psd_launch_count() - l0

    result = {"bench": "sweep_clips", **card_info(dev), "size": f"{w}x{h}", "scored": "256x144", "batch_size": bs,
              "pool_frames": args.pool, "clips": args.clips, "frames": frames_total, "tolerances": list(tols),
              "gt_cuts": sum(len(g.hard_cuts) for g in gts), "grids": []}
    parity_all = True
    for det, cls, make in (("content", ContentDetector, content_grid), ("adaptive", AdaptiveDetector, adaptive_grid)):
        for g in (int(x) for x in args.cells.split(",")):
            grid = make(g)
            # clips are at most 240 frames: no cell can emit more than 256 cuts in one
            sweep = lambda: ParameterSweep(cls, grid, tolerances=tols, batch_size=bs, device=dev,  # noqa: E731
                                           max_cuts_per_cell=256)
            sweep().run_clips(streams(4), gts[:4])  # warm-up: first engines, allocator pools
            batched = sweep()
            r, s_b, l_b = timed(lambda: batched.run_clips(streams(args.clips), gts))
            loop = sweep()
            rs, s_l, l_l = timed(lambda: [loop.run(v, gt) for v, gt in zip(streams(args.clips), gts)])
            parity = bool(np.array_equal(_hard_arrays(r, g, args.clips, tols, False),
                                         _hard_arrays(rs, g, args.clips, tols, True))
                          and all(r.cuts(k, j) == rs[j].cuts(k) for k in range(g) for j in range(0, args.clips, 97))
                          and [(t.hard, t.hard_offset, t.fades) for t in batched.totals()]
                          == [(t.hard, t.hard_offset, t.fades) for t in loop.totals()])
            parity_all = parity_all and parity
            arms = {}
            for name, s, launches in (("run_clips", s_b, l_b), ("run_loop", s_l, l_l)):
                arms[name] = {"s": round(s, 3), "clips_per_s": round(args.clips / s, 1),
                              "frames_per_s": round(frames_total / s, 1),
                              "launches_per_clip": round(launches / args.clips, 2)}
            result["grids"].append({"detector": det, "cells": g, "arms": arms, "speedup": round(s_l / s_b, 2),
                                    "parity": parity})
            del r, rs
    result["parity"] = parity_all
    print(json.dumps(result))
    return 0 if parity_all else 1


if __name__ == "__main__":
    sys.exit(main())
