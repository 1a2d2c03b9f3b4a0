#!/usr/bin/env python
"""Benchmark of mixed detectors in one engine: several dilation kernel sizes / hash geometries per upload.

1080p synthetic frames sit in page-locked host memory (what a decoder hands over).  For each mix, with the
auto-downscale on (scored at 256x144) and off (scored at 1920x1080):

* content: ContentDetector(kernel_size=5) + AdaptiveDetector(kernel_size=7) with a StatsManager (both use the edge
  component);
* hash: HashDetector(size=8) + HashDetector(size=16);

it times one SceneManager with both detectors (one engine, two slots) against two SceneManagers with one detector
each (the frames uploaded, resized and scored twice), counts the library's kernel launches per batch of each arm,
and checks that the two arms give the same cuts and metrics.  Then ParameterSweep over HashDetector sizes {8, 16}
x 64 thresholds: `run` (one engine) against the per-group way (one engine per pixel group, fed the same batches,
then `run_scored`).  Prints one JSON line with the card name and power limit; writes nothing.

    python bench_shared_pass.py [--frames 300] [--batch 64] [--reps 3]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_sweep import card_info  # noqa: E402


def _mix(name):
    from pyscenedetect_b200.detectors import AdaptiveDetector, ContentDetector, HashDetector
    if name == "content":
        return [lambda: ContentDetector(kernel_size=5), lambda: AdaptiveDetector(kernel_size=7)], True
    return [lambda: HashDetector(size=8), lambda: HashDetector(size=16)], False


def _run(makers, frames, fps, stats, auto, batch, dev):
    """One SceneManager over `frames` with a detector from each maker -> (seconds, launches, cuts, metrics)."""
    from pyscenedetect_b200 import FrameTimecode, StatsManager, _capi
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    lib = _capi.load()
    sm_stats = StatsManager() if stats else None
    sm = SceneManager(sm_stats, device=dev, batch_size=batch)
    sm.auto_downscale = auto
    dets = [m() for m in makers]
    for d in dets:
        sm.add_detector(d)
    c0 = lib.psd_launch_count()
    t0 = time.perf_counter()
    sm.detect_scenes(ArrayVideoStream(frames, fps, pinned=True))
    dt = time.perf_counter() - t0
    launches = lib.psd_launch_count() - c0
    metrics = None
    if sm_stats is not None:
        keys = sorted({k for d in dets for k in d.get_metrics()})
        metrics = [dict(zip(keys, sm_stats.get_metrics(FrameTimecode(t, fps), keys))) for t in range(frames.shape[0])]
    return dt, launches, [c.frame_num for c in sm.get_cut_list()], metrics


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of each arm (median reported)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)

    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.detectors import HashDetector
    from pyscenedetect_b200.engine import PinnedBuffer
    from pyscenedetect_b200.scene_manager import FrameBatches, SceneManager
    from pyscenedetect_b200.sweep import ParameterSweep
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    from pyscenedetect_b200.video import ArrayVideoStream

    lib = _capi.load()
    if lib.psd_device_count() < 1:
        raise SystemExit("bench_shared_pass.py needs a CUDA device")
    n, w, h, dev, fps = args.frames, args.width, args.height, args.device, 30.0
    pinned = PinnedBuffer(n * w * h * 3)
    frames = pinned.array.reshape(n, h, w, 3)
    plan = ScenePlan(n, seed=0)
    for i in range(0, n, 100):
        frames[i:i + 100] = render_frames(plan.params[i:i + 100], w, h)
    batches = -(-n // args.batch)
    result = {"bench": "shared_pass", **card_info(dev), "frames": n, "size": f"{w}x{h}", "batch": args.batch,
              "mixes": {}}
    equal = True
    for mix in ("content", "hash"):
        makers, stats = _mix(mix)
        for auto in (True, False):
            _run(makers, frames[:args.batch], fps, stats, auto, args.batch, dev)   # warm-up
            one, two = [], []
            for _ in range(args.reps):
                one.append(_run(makers, frames, fps, stats, auto, args.batch, dev))
                two.append([_run([m], frames, fps, stats, auto, args.batch, dev) for m in makers])
            t_one = sorted(r[0] for r in one)[len(one) // 2]
            t_two = sorted(sum(x[0] for x in r) for r in two)[len(two) // 2]
            cuts_two = sorted(set(c for x in two[0] for c in x[2]))
            ok = one[0][2] == cuts_two
            if stats:   # every metric, frame by frame; where both detectors write a key the later one wins
                for t, row in enumerate(one[0][3]):
                    want = {}
                    for x in two[0]:
                        want.update({k: v for k, v in x[3][t].items() if v is not None})
                    ok = ok and {k: v for k, v in row.items() if v is not None} == want
            equal = equal and ok
            result["mixes"][f"{mix}_{'auto_downscale' if auto else 'full_size'}"] = {
                "one_scene_manager_fps": round(n / t_one, 1), "two_scene_managers_fps": round(n / t_two, 1),
                "launches_per_batch_one": round(one[0][1] / batches, 2),
                "launches_per_batch_two": round(sum(x[1] for x in two[0]) / batches, 2), "equal": ok}

    # the sweep: HashDetector sizes {8, 16} x 64 thresholds
    grid = [dict(size=s, threshold=0.05 + 0.6 * i / 64) for s in (8, 16) for i in range(64)]
    sw = ParameterSweep(HashDetector, grid, batch_size=args.batch, device=dev)
    video = lambda: ArrayVideoStream(frames, fps, pinned=True)  # noqa: E731

    def per_group():
        fw, fh = w, h
        box, (cw, ch), (sw_, sh_) = SceneManager()._geometry(fw, fh)
        engines = [g.make_engine(cw, ch, sw_, sh_, dev, args.batch) for g in sw.groups]
        gather = FrameBatches(video(), box, (cw, ch), args.batch)
        while True:
            item = gather.next()
            for e in engines:
                e.sync()
            if item is None:
                break
            for e in engines:
                e.submit(item[1], pinned=item[2])
        gather.close()
        r = sw.run_scored(engines, fps)
        cuts = [r.cuts(k) for k in range(len(grid))]
        for e in engines:
            e.close()
        return cuts

    def one_engine():
        r = sw.run(video())
        return [r.cuts(k) for k in range(len(grid))]

    sweep = {}
    for name, fn in (("per_group_engines", per_group), ("run", one_engine)):
        fn()   # warm-up
        times, cuts = [], None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            cuts = fn()
            times.append(time.perf_counter() - t0)
        sweep[name] = {"fps": round(n / sorted(times)[len(times) // 2], 1), "cuts": cuts}
    sweep_equal = sweep["run"].pop("cuts") == sweep["per_group_engines"].pop("cuts")
    result["sweep_hash_8_16_x64"] = {**sweep, "groups": len(sw.groups), "equal": sweep_equal}
    result["equal"] = bool(equal and sweep_equal)
    pinned.close()
    print(json.dumps(result))
    return 0 if result["equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
