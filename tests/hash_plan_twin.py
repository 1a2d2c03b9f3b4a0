"""Python twin of the host decisions of the hash pass (csrc/hash_kernels.cu: `hash_plan_create`, `launch_hash`,
`launch_hash_finish`) and of the kernel branches they select.  The GPU hash matrix uses it to name the branches its
cases reach and to fail when one is not reached; no comparison of a result depends on it.  test_hash_plan_twin.py
pins the constants below to the source text, so a change of a decision there fails loudly instead of silently
thinning the coverage."""

from __future__ import annotations

import math
from dataclasses import dataclass

from pyscenedetect_b200._capi import hash_words

ROWS_MAX_GEO = 8                 # kHashRowsMaxGeo: geometries per rows launch
WORKSPACE_BYTES = 512 << 20      # kHashWorkspaceBytes: row buffers + finish workspaces of one sub-batch
STATIC_SMEM = 2048               # kHashStaticSmem: the finish kernel's static shared memory, rounded up
ROWS_SMEM_BYTES = 200 * 1024     # kHashRowsSmemBytes: the rows kernel's gray block
FOLD_CAP = 8                     # hash_plan_create: `p->levels < 8`
ROWS_THREADS = 256               # the rows kernel's block: 256 / n rows per CTA
H100_SMEM_OPTIN = 232448         # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KiB)


@dataclass(frozen=True)
class Plan:
    W: int
    H: int
    size: int
    lowpass: int
    n: int
    fast: bool
    area_w: int
    area_h: int
    levels: tuple            # folded lengths, level 0 (= n) first
    ws_doubles: int
    global_ws: bool
    batch: int
    words: int

    @property
    def m(self) -> int:
        return self.size * self.size


def plan(W: int, H: int, size: int, lowpass: int, max_batch: int, force_global: bool = False,
         smem_optin: int = H100_SMEM_OPTIN) -> Plan:
    n = size * lowpass
    if size < 1 or lowpass < 1 or W < n or H < n:
        raise ValueError("refused by hash_plan_create")
    levels = [n]
    while levels[-1] % 2 == 0 and levels[-1] > 1 and len(levels) < FOLD_CAP:
        levels.append(levels[-1] // 2)
    m = size * size
    ws_doubles = ((2 * n * n + 2 * size * n + (m + 1) // 2) + 1) & ~1
    global_ws = force_global or ws_doubles * 8 > smem_optin - STATIC_SMEM
    per_frame = H * n * 4 + (ws_doubles * 8 if global_ws else 0)
    batch = max(1, min(max_batch, WORKSPACE_BYTES // per_frame))
    return Plan(W, H, size, lowpass, n, W % n == 0 and H % n == 0, W // n, H // n, tuple(levels), ws_doubles,
                global_ws, batch, hash_words(size))


def pitch(W: int) -> int:
    return ((W + 3) & ~3) + 4


def rows_per_cta(W: int, n_min: int) -> int:
    """The block height `launch_hash` picks (ValueError where it refuses the frame width)."""
    if pitch(W) > ROWS_SMEM_BYTES:
        raise ValueError("frame too wide for the hash rows kernel")
    return max(1, min(ROWS_THREADS // n_min, ROWS_SMEM_BYTES // pitch(W)))


def rows_per_cta_parent(W: int, n_min: int) -> int:
    """The block height before the shared-memory cap: max(1, 256 / n), refused past 200 KiB."""
    r = max(1, ROWS_THREADS // n_min)
    if r * pitch(W) > ROWS_SMEM_BYTES:
        raise ValueError("frame too wide for the hash rows kernel")
    return r


@dataclass(frozen=True)
class Launch:
    rows_per_cta: int
    pitch: int
    batch: int
    sub_batches: tuple       # frames of each sub-batch
    rows_launches: int
    finish_launches: int


def launch(plans: list, n_frames: int) -> Launch:
    W = plans[0].W
    n_min = min(p.n for p in plans)
    batch = min(p.batch for p in plans)
    r = rows_per_cta(W, n_min)
    subs = tuple(min(batch, n_frames - f0) for f0 in range(0, n_frames, batch))
    per_sub_rows = math.ceil(len(plans) / ROWS_MAX_GEO)
    return Launch(r, pitch(W), batch, subs, per_sub_rows * len(subs), len(plans) * len(subs))


def x_taps(ssize: int, n: int) -> list:
    """(first partial tap, whole-pixel run length, last partial tap) of each destination cell, as
    hash_plan_create's area_tab / xmid tables split them."""
    scale = ssize / n
    out = []
    for dx in range(n):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        sx1, sx2 = math.ceil(fsx1), math.floor(fsx2)
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        out.append((sx1 - fsx1 > 1e-3, max(0, sx2 - sx1), fsx2 - sx2 > 1e-3))
    return out


def branches(plans: list, n_frames: int, aligned: bool = True) -> set:
    """Kernel branches and host decisions one `launch_hash` call over `plans` reaches.  `aligned`: the frames'
    base address and stride are multiples of 16 (the IDP4A gray path also needs W % 16 == 0)."""
    W, H = plans[0].W, plans[0].H
    L = launch(plans, n_frames)
    got = {"gray16" if (W % 16 == 0 and aligned) else "gray_bytes"}
    n_min = min(p.n for p in plans)
    if L.rows_per_cta > 1 and H % L.rows_per_cta:
        got.add("rows_ragged_block")
    if n_min > ROWS_THREADS:
        got.add("rows_column_loop")
    if L.rows_per_cta < max(1, ROWS_THREADS // n_min):
        got.add("rows_block_capped_by_width")
    if len(plans) > 1 and plans[0].n != n_min:
        got.add("block_set_by_later_geometry")
    got.add(f"geometries_{len(plans)}")
    if L.rows_launches > len(L.sub_batches):
        got.add("second_rows_launch")
    if len({p.fast for p in plans}) == 2:
        got.add("fast_and_float_mixed")
    if len(L.sub_batches) > 1:
        got.add("sub_batches")
        if len({p.batch for p in plans}) > 1:
            got.add("sub_batches_mixed_budgets")
    for p in plans:
        if p.fast:
            if p.area_w == 1 and p.area_h == 1:
                got.add("fast_1x1")
            elif p.area_w == 2 and p.area_h == 2:
                got.add("fast_2x2")
            else:
                got.add("fast_general")
                if 255 * p.area_w * p.area_h > 1 << 24:
                    got.add("fast_sum_above_2^24")
        else:
            for first, run, last in x_taps(W, p.n):
                got.add("float_first_tap" if first else "float_no_first_tap")
                got.add("float_run" if run else "float_run_empty")
                if last:
                    got.add("float_last_tap")
        got.add("ws_global" if p.global_ws else "ws_shared")
        lv = p.levels
        if len(lv) == 1:
            got.add("fold_one_level")
        elif len(lv) == FOLD_CAP and lv[-1] % 2 == 0:
            got.add("fold_capped")
        else:
            got.add("fold_several_levels")
        m = p.m
        if m == 1:
            got.add("median_m_1")
        elif m == 65536:
            got.add("median_m_65536")
        got.add("median_m_odd" if m % 2 else "median_m_even")
        got.add("words_4" if p.words == 4 else "words_5" if p.words == 5 else
                "words_above_32" if p.words > 32 else "words_6_to_32")
    return got


REQUIRED = {
    "gray16", "gray_bytes",
    "fast_1x1", "fast_2x2", "fast_general", "fast_sum_above_2^24",
    "float_first_tap", "float_run", "float_run_empty", "float_last_tap",
    "rows_ragged_block", "rows_column_loop", "rows_block_capped_by_width", "block_set_by_later_geometry",
    "geometries_1", "geometries_2", "geometries_8", "geometries_9", "second_rows_launch", "fast_and_float_mixed",
    "ws_shared", "ws_global", "fold_one_level", "fold_several_levels", "fold_capped",
    "median_m_1", "median_m_odd", "median_m_even", "median_m_65536",
    "words_4", "words_5", "words_above_32",
    "sub_batches", "sub_batches_mixed_budgets",
}
