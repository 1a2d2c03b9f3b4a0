"""Python twin of psd_clip_union (clip_kernels.cu) on top of tests/sweep_settings_twin.py, so that `ParameterSweep` with
`detector_sets` runs on a box with no GPU.  Each (list, clip) cut list is sorted and de-duplicated in place, and each
(cell, clip) gets the sorted union of its member lists, written to the same device arrays the kernels write, with the
entry's argument checks and its counting and writing calls."""

from __future__ import annotations

import numpy as np

from pyscenedetect_b200 import _capi
from tests import sweep_settings_twin
from tests.clip_twin import _array


def union_lists(lists, n_clips, cell_offsets, cell_lists, n_cells) -> list:
    """(cell, clip) unions, cell-major, of the (list, clip) lists `lists` (list-major)."""
    out = []
    for k in range(n_cells):
        for j in range(n_clips):
            members = cell_lists[cell_offsets[k]:cell_offsets[k + 1]]
            out.append(sorted({int(x) for i in members for x in lists[i * n_clips + j]}))
    return out


class Lib(sweep_settings_twin.Lib):
    unsorted_inputs = 0  # member lists the counting call found out of order (before its in-place sort)

    def psd_clip_union(self, cuts, cut_offsets, n_lists, n_clips, cuts_total, max_cuts, cell_offsets, cell_lists,
                       n_cells, unique, out_cuts, out_cap, out_offsets, out_over, st):
        co = [int(cell_offsets[k]) for k in range(n_cells + 1)]
        assert co[0] == 0 and all(1 <= b - a <= _capi.SWEEP_MAX_MEMBERS for a, b in zip(co, co[1:]))
        cl = [int(cell_lists[i]) for i in range(co[-1])]
        assert all(0 <= i < n_lists for i in cl)
        assert out_cuts or out_cap == 0
        m_in = n_lists * n_clips
        off = _array(cut_offsets, np.int64, m_in + 1)
        assert int(off[-1]) == cuts_total
        c = _array(cuts, np.int64) if cuts_total else np.zeros(0, np.int64)
        u = _array(unique, np.int32, m_in)
        o = _array(out_offsets, np.int64, n_cells * n_clips + 1)
        if not out_cuts:  # counting call: sort every list in place, count every union, scan
            self._count("psd_clip_union", 3)
            over = -1
            for t in range(m_in):
                b, e = int(off[t]), int(off[t + 1])
                if e - b > max_cuts:
                    over = t if over < 0 else over
                    u[t] = 0
                    continue
                Lib.unsorted_inputs += list(c[b:e]) != sorted(c[b:e])
                x = sorted({int(v) for v in c[b:e]})
                c[b:b + len(x)] = x
                u[t] = len(x)
            _array(out_over, np.int64, 1)[0] = over
            lists = [c[int(off[t]):int(off[t]) + int(u[t])].tolist() for t in range(m_in)]
            o[:] = np.concatenate([[0], np.cumsum([len(x) for x in union_lists(lists, n_clips, co, cl, n_cells)])])
            return 0
        # writing call: the unions of what the counting call left
        self._count("psd_clip_union", 1)
        lists = [c[int(off[t]):int(off[t]) + int(u[t])].tolist() for t in range(m_in)]
        unions = union_lists(lists, n_clips, co, cl, n_cells)
        assert [len(x) for x in unions] == np.diff(o).tolist(), "the writing call's arguments differ from the count's"
        if o[-1] <= out_cap and o[-1]:
            _array(out_cuts, np.int64, int(o[-1]))[:] = [x for v in unions for x in v]
        return 0
