"""CPU checks of the twin of the hash pass's host decisions (tests/hash_plan_twin.py): its constants against the
source text of csrc/hash_kernels.cu, the block height unchanged wherever the frame fitted before it was capped by the
frame width, the refused widths, and the branches the GPU hash matrix's cases reach."""

import os
import re

import pytest

from tests import hash_plan_twin as P
from tests.hash_matrix_cases import CASES, SUB_BATCH, SUB_BATCH_FRAMES, SUB_BATCH_MAX_BATCH, WIDE_FRAMES

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pyscenedetect_b200", "csrc",
                   "hash_kernels.cu")


def _src():
    with open(SRC) as f:
        return f.read()


def test_constants_match_source():
    s = _src()
    assert re.search(r"constexpr int kHashRowsMaxGeo = (\d+);", s).group(1) == str(P.ROWS_MAX_GEO)
    assert re.search(r"constexpr int kHashStaticSmem = (\d+);", s).group(1) == str(P.STATIC_SMEM)
    m = re.search(r"constexpr int64_t kHashWorkspaceBytes = \(int64_t\)(\d+) << (\d+);", s)
    assert int(m.group(1)) << int(m.group(2)) == P.WORKSPACE_BYTES
    m = re.search(r"constexpr int kHashRowsSmemBytes = (\d+) \* (\d+);", s)
    assert int(m.group(1)) * int(m.group(2)) == P.ROWS_SMEM_BYTES
    assert "p->levels < 8)" in s and P.FOLD_CAP == 8
    assert "std::max(1, std::min(256 / n_min, kHashRowsSmemBytes / pitch))" in s
    assert "const int pitch = ((W + 3) & ~3) + 4;" in s
    assert "psd_hash_rows_kernel(" in s and "__launch_bounds__(256)" in s
    assert "kHashWorkspaceBytes / per_frame" in s
    assert "((2 * n64 * n64 + 2 * (int64_t)size * n64 + (m + 1) / 2) + 1) & ~(int64_t)1" in s


def test_block_height_unchanged_where_the_frame_fitted():
    fitted = capped = 0
    for W in list(range(1, 2100)) + [2560, 3840, 4096, 7680, 15360, 50000, 204796]:
        for n in (1, 2, 3, 4, 7, 8, 16, 21, 37, 64, 100, 128, 255, 256, 257, 512, 1000):
            try:
                old = P.rows_per_cta_parent(W, n)
            except ValueError:
                new = P.rows_per_cta(W, n)
                assert 1 <= new < max(1, 256 // n) and new * P.pitch(W) <= P.ROWS_SMEM_BYTES
                capped += 1
                continue
            assert P.rows_per_cta(W, n) == old, (W, n)
            fitted += 1
    assert fitted and capped


def test_only_rows_wider_than_the_block_are_refused():
    assert P.rows_per_cta(204796, 1) == 1
    with pytest.raises(ValueError):
        P.rows_per_cta(204797, 1)


@pytest.mark.parametrize("wh,geos", WIDE_FRAMES)
def test_wide_frames_were_refused_and_now_run(wh, geos):
    W, H = wh
    n_min = min(s * lp for s, lp in geos)
    with pytest.raises(ValueError):
        P.rows_per_cta_parent(W, n_min)
    plans = [P.plan(W, H, s, lp, 16) for s, lp in geos]
    assert P.launch(plans, 2).rows_per_cta * P.pitch(W) <= P.ROWS_SMEM_BYTES


def test_sub_batch_budgets():
    big, small = (P.plan(1920, 1080, s, lp, SUB_BATCH_MAX_BATCH) for s, lp in SUB_BATCH.geos)
    assert big.global_ws and big.batch == 24 and small.batch == SUB_BATCH_MAX_BATCH
    L = P.launch([big, small], SUB_BATCH_FRAMES)
    assert L.sub_batches == (24, 2) and L.rows_launches == 2 and L.finish_launches == 4
    nine = [P.plan(1920, 1080, s, lp, 8) for s, lp in CASES[0].geos]
    assert P.launch(nine, 7).rows_launches == 2


def matrix_branches() -> set:
    """The branches the GPU hash matrix's runs reach, as test_gpu_hash_matrix.py runs them."""
    got = set()
    for c in CASES:
        n = len(c.content)
        got |= P.branches([P.plan(c.W, c.H, s, lp, n, force_global=True) for s, lp in c.geos], n)
        got |= P.branches([P.plan(c.W, c.H, s, lp, 64) for s, lp in c.geos], n)
    c = CASES[4]
    got |= P.branches([P.plan(c.W, c.H, s, lp, 8, force_global=True) for s, lp in c.geos], 8, aligned=False)
    got |= P.branches([P.plan(SUB_BATCH.W, SUB_BATCH.H, s, lp, SUB_BATCH_MAX_BATCH) for s, lp in SUB_BATCH.geos],
                      SUB_BATCH_FRAMES)
    for (W, H), geos in WIDE_FRAMES:
        got |= P.branches([P.plan(W, H, s, lp, 16) for s, lp in geos], 2)
    return got


def test_matrix_reaches_every_branch():
    missing = P.REQUIRED - matrix_branches()
    assert not missing, sorted(missing)
