"""The JPEG parity matrix shared by the twin test (CPU) and the device encoder test: sizes, qualities and contents
that reach every branch of the encoder (edges and dummy blocks, the quality scaling, byte stuffing, ZRL runs, the
largest DC category)."""

from __future__ import annotations

import numpy as np

SIZES = [(1, 1), (7, 9), (8, 8), (9, 8), (15, 17), (16, 16), (17, 16), (24, 23), (37, 53), (1280, 720),
         (1920, 1080), (1080, 1920)]   # (width, height)
QUALITIES = [0, 1, 10, 49, 50, 51, 75, 95, 100]
CONTENTS = ["random", "smooth", "scene", "black", "white", "grey", "stuffing", "zrl", "dc_jump"]


def frame(content: str, width: int, height: int, seed: int = 0) -> np.ndarray:
    """(height, width, 3) uint8 BGR"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width]
    if content == "random":
        return rng.integers(0, 256, (height, width, 3), dtype=np.uint8)
    if content == "smooth":
        return np.stack([(xx * 3 + yy) % 256, (yy * 5) % 256, ((xx + yy) * 2) % 256], -1).astype(np.uint8)
    if content == "scene":
        from pyscenedetect_b200.synth import ScenePlan, render_frames
        return render_frames(ScenePlan(3, seed=seed, min_len=1, max_len=2).params, width, height)[1]
    if content in ("black", "white", "grey"):
        return np.full((height, width, 3), {"black": 0, "white": 255, "grey": 128}[content], np.uint8)
    if content == "stuffing":
        # saturated high-frequency noise: long codes of 1-bits, so the stream is full of 0xFF bytes
        return (rng.integers(0, 2, (height, width, 3)) * 255).astype(np.uint8)
    if content == "zrl":
        # the highest horizontal DCT basis function in every block: one AC at zigzag index 28, after a run of 27 zeros
        v = 128 + 100 * np.cos((2 * (xx % 8) + 1) * 7 * np.pi / 16)
        return np.repeat(np.round(v).astype(np.uint8)[..., None], 3, -1)
    if content == "dc_jump":
        # 16x16 black / white checkerboard: DC differences of the largest category at high quality
        return np.where((((yy // 16) + (xx // 16)) % 2 == 0)[..., None], 0, 255).astype(np.uint8).repeat(3, -1)
    raise ValueError(content)


def cases(large: bool):
    """(content, width, height, quality): every content and quality at the small sizes; at the large ones
    (large=True) every quality with random content and every content at quality 95"""
    for w, h in SIZES:
        big = w * h > 10_000
        if big and not large:
            continue
        for q in QUALITIES:
            for c in CONTENTS:
                if not big or c == "random" or q == 95:
                    yield c, w, h, q
