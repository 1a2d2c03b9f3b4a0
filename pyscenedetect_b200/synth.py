"""Deterministic integer-only synthetic BGR24 frame sequences (SURVEY.md §8(d)).

The reference's own fixtures are encoded videos (tests/resources/*.mp4, not shipped with
the reference's source package), so parity and benchmarks run on a seeded synthetic sequence instead: hard
cuts at known frames, slow in-scene drift, low-amplitude per-pixel noise, fades to black
in every 3rd scene that is long enough (so ThresholdDetector's fade FSM fires) and a two-frame colour flash in
every 7th scene (so FlashFilter's MERGE/SUPPRESS branches fire).  All arithmetic is
32-bit unsigned so that this numpy generator and the CUDA generator
(`psd_synth_frames`, csrc/synth.cu) agree bit for bit.

This module is host-side product code (bench.py and the tests both use it); it is not
part of the oracle.
"""

from __future__ import annotations

import numpy as np

# Per-frame parameter row layout shared with csrc/synth.cu (int32 each).
#   0..2  A[c]   x-gradient coefficient for channel c (B,G,R)
#   3..5  B[c]   y-gradient coefficient
#   6..8  C[c]   (x*y)>>8 coefficient
#   9..11 O[c]   constant offset + in-scene drift
#   12    gain   0..256 fade gain
#   13    seed_t per-frame noise seed
#   14    scene index (informational)
#   15    noise shift (29 => [-4,3], 30 => [-2,1], 32 => no noise)
#   16..18 span[c] per-scene contrast (64..256): v = lo + ((v * span) >> 8)
#   19..21 lo[c]   per-scene black level (0..256-span)
#   22..23 spare
PARAMS_PER_FRAME = 24

_M32 = 0xFFFFFFFF


def mix32(x: int) -> int:
    """lowbias32 integer hash on a Python int, 32-bit wrap-around."""
    x &= _M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & _M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & _M32
    x ^= x >> 16
    return x


def _mix32_np(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.uint32, copy=True)
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x7FEB352D)
    x ^= x >> np.uint32(15)
    x *= np.uint32(0x846CA68B)
    x ^= x >> np.uint32(16)
    return x


class ScenePlan:
    """Seeded list of scenes -> per-frame parameter table + ground-truth cut frames."""

    def __init__(self, n_frames: int, seed: int = 0, noise_shift: int = 30,
                 min_len: int = 24, max_len: int = 240):
        assert n_frames > 0
        self.n_frames = int(n_frames)
        self.seed = int(seed)
        state = mix32(self.seed ^ 0xA5A5A5A5)

        def nxt() -> int:
            nonlocal state
            state = mix32(state + 0x9E3779B9)
            return state

        params = np.zeros((self.n_frames, PARAMS_PER_FRAME), dtype=np.int32)
        cuts: list[int] = []
        fades: list[int] = []
        t = 0
        scene = 0
        while t < self.n_frames:
            length = min_len + nxt() % (max_len - min_len + 1)
            A = [1 + nxt() % 48 for _ in range(3)]
            B = [1 + nxt() % 48 for _ in range(3)]
            C = [nxt() % 16 for _ in range(3)]
            O = [nxt() % 256 for _ in range(3)]
            span = [64 + nxt() % 193 for _ in range(3)]
            lo = [nxt() % (257 - s) for s in span]
            fade = (scene % 3 == 2) and length >= 36
            flash = (scene % 7 == 3) and length >= 30
            mid = length // 2
            if scene > 0:
                cuts.append(t)
            for j in range(length):
                if t >= self.n_frames:
                    break
                gain = 256
                if fade:
                    gain = max(0, min(256, (abs(j - mid) - 4) * 32))
                    if j == mid:
                        fades.append(t)
                row = params[t]
                row[0:3] = A
                row[3:6] = B
                row[6:9] = C
                row[9:12] = [o + (j >> 2) + (128 if (flash and j in (8, 9)) else 0) for o in O]
                row[12] = gain
                st = mix32((self.seed * 0x9E3779B9 + t * 0x85EBCA6B + 1) & _M32)
                row[13] = st - (1 << 32) if st >= (1 << 31) else st
                row[14] = scene
                row[15] = noise_shift
                row[16:19] = span
                row[19:22] = lo
                t += 1
            scene += 1
        self.params = params
        self.cut_frames = cuts
        self.fade_frames = fades
        self.n_scenes = scene


def render_frames(params: np.ndarray, width: int, height: int,
                  first: int = 0, count: int | None = None) -> np.ndarray:
    """Render frames [first, first+count) of a plan to a (count, H, W, 3) uint8 BGR array."""
    params = np.asarray(params, dtype=np.int32)
    if count is None:
        count = params.shape[0] - first
    out = np.empty((count, height, width, 3), dtype=np.uint8)
    x = np.arange(width, dtype=np.uint32)[None, :]
    y = np.arange(height, dtype=np.uint32)[:, None]
    xy = (x * y) >> np.uint32(8)
    idx3 = (y * np.uint32(width) + x) * np.uint32(3)
    for i in range(count):
        row = params[first + i].view(np.uint32)
        gain = np.uint32(row[12])
        seed_t = np.uint32(row[13])
        nshift = int(params[first + i][15])
        for c in range(3):
            p = (np.uint32(row[c]) * x + np.uint32(row[3 + c]) * y + np.uint32(row[6 + c]) * xy) >> np.uint32(4)
            v = (p + np.uint32(row[9 + c])) & np.uint32(255)
            v = np.uint32(row[19 + c]) + ((v * np.uint32(row[16 + c])) >> np.uint32(8))
            v = (v * gain) >> np.uint32(8)
            vi = v.astype(np.int32)
            if nshift < 32:
                h = _mix32_np(seed_t + idx3 + np.uint32(c))
                n = (h >> np.uint32(nshift)).astype(np.int32) - np.int32(1 << (31 - nshift))
                vi = vi + n
            out[i, :, :, c] = np.clip(vi, 0, 255).astype(np.uint8)
    return out


def synth_sequence(n_frames: int, width: int, height: int, seed: int = 0,
                   noise_shift: int = 30) -> tuple[np.ndarray, ScenePlan]:
    plan = ScenePlan(n_frames, seed=seed, noise_shift=noise_shift)
    return render_frames(plan.params, width, height), plan
