"""tests/sweep_sets_twin.py's library with psd_clip_cuts_tables_steps: a step per (table, clip).  Cell k runs over
tables[cell_table[k]] as tests/clip_steps_twin.py runs psd_clip_cuts_steps over one table, each clip with that table's
own frame_step[j], which is what the entry promises."""

from __future__ import annotations

import numpy as np

from tests import clip_steps_twin, sweep_sets_twin
from tests.clip_twin import _array


def cut_lists_tables_steps(cells, n_cells, tables, cell_table, n_clips, mf) -> list:
    """Every (cell, clip) list, cell-major: cell k over its own table, with that table's per-clip steps."""
    lists = []
    for k in range(n_cells):
        t = tables[cell_table[k] if cell_table is not None else 0]
        steps = _array(t.frame_step, np.int64, n_clips)
        assert (steps >= 1).all()
        lists += clip_steps_twin.clip_cut_lists_steps(
            [cells[k]], 1, _array(t.offsets, np.int64, n_clips + 1), _array(t.first_frame, np.int64, n_clips), n_clips,
            mf[k * n_clips:(k + 1) * n_clips], steps, _array(t.end_frame, np.int64, n_clips) if t.end_frame else None)
    return lists


class Lib(sweep_sets_twin.Lib, clip_steps_twin.Lib):
    def psd_clip_cuts_tables_steps(self, cells, n_cells, tables, n_tables, cell_table, n_clips, min_frames, cuts, cap,
                                   cut_offsets, st):
        assert n_tables >= 1 and all(tables[i].frame_step for i in range(n_tables))
        assert cell_table is None or all(0 <= cell_table[k] < n_tables for k in range(n_cells))
        self._count("psd_clip_cuts_tables_steps", 3)
        lists = cut_lists_tables_steps(cells, n_cells, tables, cell_table, n_clips,
                                       _array(min_frames, np.int64, n_cells * n_clips))
        o = _array(cut_offsets, np.int64, n_cells * n_clips + 1)
        o[:] = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        if o[-1] <= cap and o[-1]:
            _array(cuts, np.int64, int(o[-1]))[:] = [c for x in lists for c in x]
        return 0
