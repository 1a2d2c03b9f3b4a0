#!/usr/bin/env python
"""Benchmark of the sweep over detector sets (`ParameterSweep(detector_sets=...)`): every detector of every set from one
read of each clip, against the per-class sweeps or the per-combination `detect_clips` a user runs without it.

The clip set is bench_clips.py's: --clips `ArrayVideoStream`s over slices of a pool of synthetic 1280x720 frames
rendered into HBM by psd_synth_frames, lengths in [48, 240] frames, rates from (24, 25, 30000/1001, 30), and the
first --host-clips of them copied to pageable host memory.  Ground truth is each slice's ScenePlan cuts.  Two
comparisons, each arm timed on the host clock around work that ends in a device synchronise, arms alternating for
--rounds rounds (best time reported):

  classes  five --cells-cell grids (ContentDetector, AdaptiveDetector, ThresholdDetector, HistogramDetector,
           HashDetector), every cell a one-detector set:
             sets       one ParameterSweep(detector_sets=...).run_clips over every clip
             per_class  one ParameterSweep(cls, grid).run_clips per class, each on fresh streams
           on the CUDA clips and on the host clips;
  combos   8 AdaptiveDetectors x 8 ThresholdDetectors, every pair a two-detector set (64 cells, 16 automata):
             sets           one ParameterSweep(detector_sets=...).run_clips
             detect_clips   one detect_clips per pair, its cut lists scored on the host (tests/sweep_model.py's rules)
           on the first --combo-clips CUDA clips (a subset: the detect_clips arm reads every clip 64 times).

Reported per arm: clips/s, library launches per clip (psd_launch_count) and host frame bytes per clip submitted to
the engines, counted at `Engine.submit` (every host submission is copied to the device).
`equal` is true when every (cell, clip) cut list and count is equal between the arms.  Prints one JSON line per
comparison and input; writes nothing.

    python bench_sweep_sets.py [--clips 1000] [--host-clips 20] [--combo-clips 200] [--cells 64] [--rounds 2]
"""

from __future__ import annotations

import argparse
import bisect
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


def grids(g: int) -> dict:
    """Five g-cell grids, bench_sweep.py's for ContentDetector and AdaptiveDetector."""
    from bench_sweep import adaptive_grid, content_grid
    msl = (0, 5, 10, 15, 30, 60, 90, 120)
    per = -(-g // len(msl))
    return {
        "content": content_grid(g),
        "adaptive": adaptive_grid(g),
        "threshold": [dict(threshold=4 + 60 * (i // len(msl)) // per, min_scene_len=msl[i % len(msl)],
                           fade_bias=(-0.5, 0.0, 0.5)[i % 3]) for i in range(g)],
        "histogram": [dict(threshold=0.02 + 0.3 * (i // len(msl)) / per, bins=(64, 128, 256)[i % 3],
                           min_scene_len=msl[i % len(msl)]) for i in range(g)],
        "hash": [dict(threshold=0.1 + 0.4 * (i // len(msl)) / per, min_scene_len=msl[i % len(msl)]) for i in range(g)],
    }


def score(preds, gt, tol):
    """benchmark/evaluator.py's hard-cut matching of one predicted list (tests/sweep_model.py, restated):
    (matched, false_positives, missed)."""
    used_g = [False] * len(gt)
    used_p = [False] * len(preds)
    matched = 0
    for d in range(tol + 1):
        for i, p in enumerate(preds):
            if used_p[i]:
                continue
            for g in ((p - d, p + d) if d else (p,)):
                j = bisect.bisect_left(gt, g)
                if j < len(gt) and gt[j] == g and not used_g[j]:
                    used_g[j] = used_p[i] = True
                    matched += 1
                    break
    return matched, len(preds) - matched, len(gt) - matched


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--host-clips", type=int, default=20)
    ap.add_argument("--combo-clips", type=int, default=200)
    ap.add_argument("--cells", type=int, default=64)
    ap.add_argument("--tolerances", default="0,1")
    ap.add_argument("--pool", type=int, default=1024, help="frames in the resident pool the clips are slices of")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the arms (best reported)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)
    if args.pool < 240 or min(args.clips, args.rounds, args.cells, args.combo_clips) < 1 or args.host_clips < 0:
        ap.error("--pool must be >= 240, --clips, --combo-clips, --cells and --rounds >= 1, --host-clips >= 0")

    import torch

    from bench_clips import card_info
    from pyscenedetect_b200 import _capi, scene_manager
    from pyscenedetect_b200 import detectors as D
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.engine import synth_frames_device
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_sweep_sets.py needs a CUDA device")

    class CountingEngine(scene_manager.Engine):
        """The engine, counting the host frame bytes submitted to it (each submission copies them to the device)."""
        host_bytes = 0

        def submit(self, frames, pinned=False, channel_order="bgr"):
            if isinstance(frames, np.ndarray):
                CountingEngine.host_bytes += frames.nbytes
            return super().submit(frames, pinned=pinned, channel_order=channel_order)

    scene_manager.Engine = CountingEngine  # the engines of SceneManager, detect_clips and the sweeps
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
    n_max = max(args.clips, args.host_clips, args.combo_clips)
    lengths = rng.integers(48, 241, size=n_max)
    starts = [int(rng.integers(0, args.pool - n + 1)) for n in lengths]
    rates = [RATES[i % len(RATES)] for i in range(n_max)]
    pool_cuts = np.asarray(plan.cut_frames, dtype=np.int64)
    gts = [GroundTruth([int(c) - s for c in pool_cuts if s < c < s + n]) for s, n in zip(starts, lengths)]
    tols = tuple(int(t) for t in args.tolerances.split(","))
    classes = {"content": D.ContentDetector, "adaptive": D.AdaptiveDetector, "threshold": D.ThresholdDetector,
               "histogram": D.HistogramDetector, "hash": D.HashDetector}
    g5 = grids(args.cells)

    def streams(k, src):
        return [ArrayVideoStream(src[s:s + n], fps) for s, n, fps in zip(starts[:k], lengths[:k], rates[:k])]

    def timed(arms, warm):
        warm()
        torch.cuda.synchronize()
        best, seen = {}, {}
        for _ in range(args.rounds):
            for name, fn in arms.items():
                l0, b0 = lib.psd_launch_count(), CountingEngine.host_bytes
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                launches, up = lib.psd_launch_count() - l0, CountingEngine.host_bytes - b0
                seen[name] = out
                if name not in best or dt < best[name]["s"]:
                    best[name] = {"s": dt, "launches": launches, "upload": up}
        return best, seen

    def report(kind, src_name, n_clips, best, equal, extra):
        result = {"bench": "sweep_sets", **card, "comparison": kind, "input": src_name, "size": f"{w}x{h}",
                  "batch_size": bs, "clips": n_clips, "frames": int(sum(lengths[:n_clips])), "tolerances": list(tols),
                  "rounds": args.rounds, **extra, "arms": {}}
        for name, b in best.items():
            result["arms"][name] = {"s": round(b["s"], 3), "clips_per_s": round(n_clips / b["s"], 1),
                                    "launches_per_clip": round(b["launches"] / n_clips, 2),
                                    "h2d_frame_bytes_per_clip": round(b["upload"] / n_clips)}
        names = list(best)
        result[f"speedup_vs_{names[1]}"] = round(best[names[1]]["s"] / best[names[0]]["s"], 2)
        result["equal"] = equal
        print(json.dumps(result), flush=True)
        return 0 if equal else 1

    def cell_counts(r, k, j):
        return (r.cuts(k, j), [r.hard(k, j, t) for t in tols], [r.hard_offset(k, j, t) for t in tols], r.fades(k, j))

    status = 0
    # -- classes: one sweep over every class's cells against one sweep per class
    singles = [classes[c](**p) for c in classes for p in g5[c]]
    inputs = [("cuda", pool, args.clips)] + ([("host", host_pool, args.host_clips)] if args.host_clips else [])
    for src_name, src, n_clips in inputs:
        def together():
            sw = ParameterSweep(detector_sets=singles, tolerances=tols, batch_size=bs, device=dev,
                                max_cuts_per_cell=256)
            return sw.run_clips(streams(n_clips, src), gts[:n_clips])

        def apart():
            rs = []
            for c in classes:
                sw = ParameterSweep(classes[c], g5[c], tolerances=tols, batch_size=bs, device=dev,
                                    max_cuts_per_cell=256)
                rs.append(sw.run_clips(streams(n_clips, src), gts[:n_clips]))
            return rs

        def warm():
            ParameterSweep(detector_sets=singles, tolerances=tols, batch_size=bs, device=dev).run_clips(
                streams(4, src), gts[:4])
            for c in classes:
                ParameterSweep(classes[c], g5[c], tolerances=tols, batch_size=bs, device=dev).run_clips(
                    streams(4, src), gts[:4])

        best, seen = timed({"sets": together, "per_class": apart}, warm)
        r_all, r_each = seen["sets"], seen["per_class"]
        equal, k = True, 0
        for c, r in zip(classes, r_each):
            for g in range(len(g5[c])):
                equal &= all(cell_counts(r_all, k + g, j) == cell_counts(r, g, j) for j in range(n_clips))
            k += len(g5[c])
        status |= report("classes", src_name, n_clips, best, equal,
                         {"cells": len(singles), "automata": len(singles)})

    # -- combos: Adaptive x Threshold pairs in one sweep against one detect_clips per pair
    n_clips = args.combo_clips
    ad = [D.AdaptiveDetector(**p) for p in g5["adaptive"][::max(1, len(g5["adaptive"]) // 8)][:8]]
    th = [D.ThresholdDetector(**p) for p in g5["threshold"][::max(1, len(g5["threshold"]) // 8)][:8]]
    pairs = [[a, t] for a in ad for t in th]

    def combo_sweep():
        sw = ParameterSweep(detector_sets=pairs, tolerances=tols, batch_size=bs, device=dev)
        r = sw.run_clips(streams(n_clips, pool), gts[:n_clips])
        return [[(r.cuts(k, j), [r.hard(k, j, t) for t in tols]) for j in range(n_clips)]
                for k in range(len(pairs))]

    def combo_detect():
        out = []
        for pair in pairs:
            res = detect_clips(streams(n_clips, pool), pair, batch_size=bs, device=dev)
            row = []
            for j, cr in enumerate(res):
                preds = cr.cut_frames + [cr.end.frame_num + 1] if cr.cut_frames else []
                row.append((preds, [score(preds, gts[j].hard_cuts, t) for t in tols]))
            out.append(row)
        return out

    def warm():
        ParameterSweep(detector_sets=pairs, tolerances=tols, batch_size=bs, device=dev).run_clips(
            streams(4, pool), gts[:4])
        detect_clips(streams(4, pool), pairs[0], batch_size=bs, device=dev)

    best, seen = timed({"sets": combo_sweep, "detect_clips": combo_detect}, warm)
    status |= report("combos", "cuda", n_clips, best, seen["sets"] == seen["detect_clips"],
                     {"cells": len(pairs), "automata": len(ad) + len(th)})
    return status


if __name__ == "__main__":
    sys.exit(main())
