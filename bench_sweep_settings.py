#!/usr/bin/env python
"""Benchmark of the parameter sweep over settings (`ParameterSweep(settings=...)`): one read of each clip for every
(auto_downscale, downscale, crop, frame_skip) setting, against one single-setting sweep per setting on fresh streams.

The clip set is bench_clips.py's: --clips `ArrayVideoStream`s over slices of a pool of synthetic 1280x720 frames
rendered into HBM by psd_synth_frames, lengths in [48, 240] frames, rates from (24, 25, 30000/1001, 30), and the
first --host-clips of them copied to pageable host memory.  Ground truth is each slice's ScenePlan cuts.  For a
ContentDetector grid and an AdaptiveDetector grid of --cells cells (bench_sweep.py's grid builders) over the five
settings of SETTINGS, two arms run alternately for --rounds rounds (best time reported), each timed on the host clock
around work that ends in a device synchronise:

  settings     one ParameterSweep(settings=SETTINGS).run_clips over every clip
  per_setting  one ParameterSweep(settings=[s]).run_clips per setting, each on fresh streams

Reported per arm: clips/s, library launches per clip (psd_launch_count) and host-to-device frame bytes per clip
(the settings path's upload count; the per-setting arm's {} sweep submits host frames through the engine, counted as
the frames it scores).  `equal` is true when every (cell, clip) count and every cell total is equal between the arms.
Prints one JSON line per (detector, input); writes nothing.

    python bench_sweep_settings.py [--clips 1000] [--host-clips 20] [--cells 64] [--rounds 2]
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
SETTINGS = [{}, {"frame_skip": 1}, {"frame_skip": 3}, {"auto_downscale": False, "downscale": 2},
            {"crop": (0, 60, 1279, 659), "frame_skip": 1}]


def counts(r, n_cells, n_clips, tols):
    """Every (cell, clip) count of a ClipSweepResult as one int64 array."""
    out = np.zeros((n_cells, n_clips, len(tols) * 5 + 4), dtype=np.int64)
    for k in range(n_cells):
        for j in range(n_clips):
            row = []
            for t in tols:
                row += [*r.hard(k, j, t), *r.hard_offset(k, j, t)]
            out[k, j] = row + [*r.fades(k, j), r.raw_count(k, j)]
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=20)
    ap.add_argument("--cells", type=int, default=64)
    ap.add_argument("--tolerances", default="0,1")
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the two arms (best reported)")
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
        raise SystemExit("bench_sweep_settings.py needs a CUDA device")
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
    pool_cuts = np.asarray(plan.cut_frames, dtype=np.int64)
    gts = [GroundTruth([int(c) - s for c in pool_cuts if s < c < s + n]) for s, n in zip(starts, lengths)]
    tols = tuple(int(t) for t in args.tolerances.split(","))

    def streams(k, src):
        return [ArrayVideoStream(src[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def sweep(cls, grid, settings):
        # clips are at most 240 frames: no cell can emit more than 256 cuts in one
        return ParameterSweep(cls, grid, tolerances=tols, batch_size=bs, device=dev, max_cuts_per_cell=256,
                              settings=settings)

    status = 0
    inputs = [("cuda", pool, args.clips)] + ([("host", host_pool, args.host_clips)] if args.host_clips else [])
    for det, cls, make in (("content", ContentDetector, content_grid), ("adaptive", AdaptiveDetector, adaptive_grid)):
        grid = make(args.cells)
        for src_name, src, n_clips in inputs:
            frames_host = sum(int(n) for n in lengths[:n_clips]) * fb if src_name == "host" else 0

            def together():
                sw = sweep(cls, grid, SETTINGS)
                r = sw.run_clips(streams(n_clips, src), gts[:n_clips])
                return [r], [sw], r.upload_bytes or 0

            def apart():
                rs, sws, up = [], [], 0
                for s in SETTINGS:
                    sw = sweep(cls, grid, [s])
                    r = sw.run_clips(streams(n_clips, src), gts[:n_clips])
                    rs.append(r)
                    sws.append(sw)
                    # the {} sweep submits host frames through the engine: every frame it reads crosses once
                    up += r.upload_bytes if r.upload_bytes is not None else frames_host
                return rs, sws, up

            arms = {"settings": together, "per_setting": apart}
            for settings in [SETTINGS] + [[s] for s in SETTINGS]:  # warm-up: first engines, allocator pools
                sweep(cls, grid, settings).run_clips(streams(4, src), gts[:4])
            torch.cuda.synchronize()
            best, seen = {}, {}
            for _ in range(args.rounds):
                for name, fn in arms.items():
                    l0 = lib.psd_launch_count()
                    t0 = time.perf_counter()
                    rs, sws, up = fn()
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    launches = lib.psd_launch_count() - l0
                    seen[name] = (rs, sws)
                    if name not in best or dt < best[name]["s"]:
                        best[name] = {"s": dt, "launches": launches, "upload": up}
            (r_all,), (sw_all,) = seen["settings"]
            r_each, sw_each = seen["per_setting"]
            g = len(grid)
            got = counts(r_all, len(r_all), n_clips, tols)
            want = np.concatenate([counts(r, g, n_clips, tols) for r in r_each])
            tot = lambda ts: [(t.hard, t.hard_offset, t.fades) for t in ts]  # noqa: E731
            equal = bool(np.array_equal(got, want)
                         and tot(sw_all.totals()) == [x for sw in sw_each for x in tot(sw.totals())]
                         and all(r_all.end_frame(j, setting=s) == r_each[s].end_frame(j)
                                 for s in range(len(SETTINGS)) for j in range(n_clips))
                         and all(r_all.cuts(s * g + k, j) == r_each[s].cuts(k, j) for s in range(len(SETTINGS))
                                 for k in range(0, g, 7) for j in range(0, n_clips, 13)))
            result = {"bench": "sweep_settings", **card, "detector": det, "cells": g, "settings": len(SETTINGS),
                      "input": src_name, "size": f"{w}x{h}", "batch_size": bs, "clips": n_clips,
                      "frames": int(sum(lengths[:n_clips])), "tolerances": list(tols), "rounds": args.rounds,
                      "arms": {}}
            for name, b in best.items():
                result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(n_clips / b["s"], 1),
                                        "launches_per_clip": round(b["launches"] / n_clips, 2),
                                        "h2d_frame_bytes_per_clip": round(b["upload"] / n_clips)}
            result["speedup_vs_per_setting"] = round(best["per_setting"]["s"] / best["settings"]["s"], 2)
            result["equal"] = equal
            print(json.dumps(result), flush=True)
            status |= 0 if equal else 1
    return status


if __name__ == "__main__":
    sys.exit(main())
