"""The cases of the hash-pass matrix (test_gpu_hash_matrix.py) and the frames they run: shared with the CPU tests
that pin the stage twin (tests/hash_twin.py) to oracle/intmath.py and cv2 at the same geometries."""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from pyscenedetect_b200.synth import ScenePlan, render_frames


@dataclass(frozen=True)
class Case:
    name: str
    W: int
    H: int
    geos: tuple              # ((size, lowpass), ...): slot order
    content: tuple           # frame kinds (see frame())


_ALL = ("plan", "noise", "black", "solid", "mirror", "hgrad", "vgrad")
_FEW = ("plan", "hgrad", "mirror")

# what each case is for: tests/hash_plan_twin.py names the branches, test_gpu_hash_matrix.py checks they are all hit
CASES = [
    # nine geometries on 1080p: a second rows launch, the block height set by n = 1 (a later slot) and capped by the
    # frame width, integer areas 1920x1080 (m = 1) to 16x9, float geometries with and without partial taps
    Case("1080p_nine_geometries", 1920, 1080,
         ((8, 2), (1, 1), (2, 1), (3, 1), (5, 3), (9, 1), (17, 1), (12, 10), (4, 1)), _ALL + ("area_tie",)),
    Case("1080p_eight_geometries", 1920, 1080, ((8, 2), (2, 1), (3, 1), (5, 3), (9, 1), (17, 1), (12, 10), (4, 1)),
         ("plan", "hgrad")),
    Case("1000x37_ragged_block", 1000, 37, ((37, 1),), _ALL),                 # 6 rows per CTA, 37 % 6 = 1
    Case("131x97_two_geometries", 131, 97, ((21, 1), (7, 3)), _ALL),          # 12 rows per CTA, 97 % 12 = 1
    Case("256x144_no_whole_pixel_run", 256, 144, ((72, 2),), _ALL),         # scale 1.78: cells without a run
    Case("64x64_area_1x1", 64, 64, ((8, 8), (16, 4), (1, 64)), _ALL),
    Case("1080p_n512_fold_cap", 1920, 1080, ((128, 4),), _FEW),             # one row per CTA, column loop
    Case("1024_2x2_m65536", 1024, 1024, ((256, 2),), ("plan", "vgrad")),     # 2x2 integer path, fold cap
    Case("4k_area_480x270", 3840, 2160, ((4, 2), (2, 2)), _FEW + ("area_tie",)),   # integer sums above 2^24
]

# Engine only: more frames than one sub-batch (n = 1000: 24 frames per sub-batch), with a geometry whose budget
# allows the whole batch
SUB_BATCH = Case("1080p_sub_batches", 1920, 1080, ((100, 10), (8, 2)), ("plan", "noise", "hgrad", "vgrad", "mirror"))
SUB_BATCH_FRAMES, SUB_BATCH_MAX_BATCH = 26, 32

# scored frame sizes and geometries the rows kernel refused before its block height was capped by the frame width
WIDE_FRAMES = [((1280, 720), ((1, 1),)), ((1920, 1080), ((1, 1), (2, 1))), ((3840, 2160), ((4, 1), (2, 2))),
               ((7680, 4320), ((4, 2),))]


# An integer-path cell whose block sum s, a grey level or two from a half-integer mean, rounds differently as
# float32(s) * float32(1 / area) (OpenCV) and as float32(s) / area: (frame size) -> (block w, h, the two grey levels of alternate columns, what to
# add to the block's sum).  The rest of the frame is 200, so the cell's value shows in the normalised image.
AREA_TIES = {(1920, 1080): (640, 360, (129, 130), -2), (3840, 2160): (480, 270, (128, 129), 1)}


def frame(kind: str, W: int, H: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if kind == "plan":
        return render_frames(ScenePlan(3, seed=seed, min_len=1, max_len=2).params[seed % 3:seed % 3 + 1], W, H)[0]
    if kind == "noise":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "black":
        return np.zeros((H, W, 3), np.uint8)
    if kind == "solid":
        return np.broadcast_to(rng.integers(1, 256, 3, dtype=np.uint8), (H, W, 3)).copy()
    if kind == "mirror":   # symmetric left-right and top-bottom
        q = rng.integers(0, 256, ((H + 1) // 2, (W + 1) // 2, 3), dtype=np.uint8)
        q = np.concatenate([q, q[:, ::-1][:, W % 2:]], axis=1)
        return np.ascontiguousarray(np.concatenate([q, q[::-1][H % 2:]], axis=0))
    if kind == "hgrad":
        g = (np.arange(W) * 255 // max(1, W - 1)).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(g[None, :, None], (H, W, 3)))
    if kind == "vgrad":
        g = (np.arange(H) * 255 // max(1, H - 1)).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(g[:, None, None], (H, W, 3)))
    if kind == "area_tie":
        bw, bh, (lo, hi), extra = AREA_TIES[(W, H)]
        f = np.full((H, W, 3), 200, np.uint8)
        f[:bh, :bw] = np.where(np.arange(bw) % 2 == 0, lo, hi).astype(np.uint8)[None, :, None]
        for i in range(abs(extra)):   # one grey level at a time on distinct pixels
            f[1, 2 * i + (0 if extra > 0 else 1)] += np.uint8(1) if extra > 0 else np.uint8(255)
        return f
    raise ValueError(kind)


def frames(case: Case) -> np.ndarray:
    return np.stack([frame(k, case.W, case.H, 7 * i + case.W) for i, k in enumerate(case.content)])
