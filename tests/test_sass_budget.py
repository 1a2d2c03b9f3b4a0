"""Static checks on the compiled sm_90a code (no GPU needed): the fused pass really uses the
instructions DESIGN.md says it does, nothing spills to local memory, and the two loops whose
instruction count IS the performance (the kernel is issue-bound) stay within their budgets.  Runs on
the in-tree libpsd_b200.so that __graft_entry__.build() produces; skipped without cuobjdump."""

import os
import re
import shutil
import subprocess

import pytest

from pyscenedetect_b200 import _capi

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP) or not os.path.exists(_capi.LIB_PATH),
                                reason="needs cuobjdump and the built library")

WS_HSV_V7 = "_ZN3psd19psd_score_ws_kernelILj1EEEvNS_9ScoreArgsE"
CLASSIFY = "_ZN3psd31psd_canny_classify_pairs_kernelILb1EEEvPKhPKiPjS5_Phiiiiil"
HYST = "_ZN3psd20psd_hyst_bits_kernelEPjPKjPhPiiiiiil"
LINE = re.compile(r"^\s+/\*([0-9a-f]{4})\*/\s+(?:@!?U?P\d\s+)?([A-Za-z0-9_.]+)")


def sass(function):
    out = subprocess.run([CUOBJDUMP, "-sass", "-fun", function, _capi.LIB_PATH], capture_output=True, text=True,
                         timeout=300).stdout
    rows = [(int(m.group(1), 16), m.group(2), line) for line in out.splitlines() if (m := LINE.match(line))]
    assert rows, f"{function} not found in {_capi.LIB_PATH}"
    return rows


def loops(rows):
    """(start index, end index) of every backward branch"""
    addr_to_idx = {a: i for i, (a, _, _) in enumerate(rows)}
    res = []
    for i, (a, op, line) in enumerate(rows):
        m = re.search(r"BRA\s+(?:!?U?P\d,\s*)?0x([0-9a-f]+)", line)
        if op.startswith("BRA") and m and int(m.group(1), 16) < a and int(m.group(1), 16) in addr_to_idx:
            res.append((addr_to_idx[int(m.group(1), 16)], i))
    return res


def test_ws_kernel_instruction_mix_and_budget():
    rows = sass(WS_HSV_V7)
    ops = [op for _, op, _ in rows]
    for needed in ("UBLKCP.S.G", "SYNCS.ARRIVE.TRANS64", "VIMNMX3.U16x2", "HFMA2", "HADD2.F32", "HSET2.EQ.AND",
                   "IDP.2A.LO.U16.U8", "VABSDIFF4.U8.ACC", "FFMA.RZ", "FFMA.RM", "LDS.128", "ATOMS.ADD"):
        assert any(o.startswith(needed) for o in ops), f"{needed} missing from the fused pass"
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "the fused pass spills to local memory"
    # consumer loop = the innermost backward branch whose body holds the 3 LDS.128 of each of its 2 or 4 frames
    bodies = [rows[a:b + 1] for a, b in loops(rows)]

    def n_lds(b):
        return sum(op == "LDS.128" for _, op, _ in b)
    main = max(n_lds(b) for b in bodies if n_lds(b) in (6, 12))
    cons = min((b for b in bodies if n_lds(b) == main), key=len)
    per_frame = len(cons) / (main // 3)
    assert per_frame <= 350, f"consumer loop grew to {per_frame} instructions per frame (16 px per thread)"
    # no warp reduction / election code on the consumer side any more
    assert not any(op.startswith(("REDUX", "UFLO")) for _, op, _ in cons)


def test_edge_kernels_use_the_instructions_the_design_names():
    """classify: 16-bit lane pairs (PRMT expansion, binary16 arithmetic, VIMNMX3 + HSET2 suppression, FP32 FMAs
    for the sector, IDP.2A bit packing), no shared memory, a per-row instruction budget;
    hysteresis: bit reversal for the downward run fill, a grid barrier (cooperative launch), no spills."""
    rows = sass(CLASSIFY)
    ops = [op for _, op, _ in rows]
    for needed in ("PRMT", "HFMA2", "HADD2", "HADD2.F32", "FFMA", "VIMNMX3.U16x2", "HSET2.GT", "IDP.2A", "LDG.E.64"):
        assert any(o.startswith(needed) for o in ops), f"{needed} missing from the classify kernel"
    assert not any(o.startswith(("LDS", "STS", "SHFL", "BAR")) for o in ops)
    assert sum(o.startswith(("LDL", "STL")) for o in ops) <= 64   # 128-register cap (2 CTAs / SM): a few words spill
    # the row loop makes six rows per trip (two sum sets x three magnitude rows): 8 pixels per thread and row
    body = max((rows[a:b + 1] for a, b in loops(rows)), key=len)
    assert not any(op.startswith(("I2F", "F2I", "F2F")) for _, op, _ in body)   # no conversion instructions
    assert sum(op.startswith("STG") for _, op, _ in body) == 12
    assert len(body) / 6 <= 300, f"classify grew to {len(body) / 6:.0f} instructions per 8-pixel row"
    rows = sass(HYST)
    ops = [op for _, op, _ in rows]
    assert any(o.startswith("BREV") for o in ops) and any(o.startswith("SHFL") for o in ops)
    assert sum(o.startswith(("LDL", "STL")) for o in ops) <= 8
