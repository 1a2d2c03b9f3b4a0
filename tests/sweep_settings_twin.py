"""Python twins of psd_clip_cuts_tables and psd_clip_eval_tables (clip_kernels.cu), and an engine that scores frames
from twin device memory through `Engine.submit_layout`, so that `ParameterSweep` with settings runs on a box with no
GPU.  Cell k reads clip table tables[cell_table[k]]: its cut lists come from tests/clip_window_twin.py's stepped
automata, its predicted lists end at that table's end frames and are scored by tests/sweep_model.py, as
tests/sweep_clip_twin.py scores one table."""

from __future__ import annotations

import numpy as np

from tests import clip_twin, clip_window_twin, sweep_clip_twin, sweep_model
from tests.clip_twin import _array
from tests.fake_engine import OracleEngine


class SettingsEngine(clip_twin.ClipEngine):
    """ClipEngine that also takes frames from twin device memory with a (frame, row, pixel, channel) stride layout."""

    layouts = []  # (frames, layout) of every submit_layout

    def submit_layout(self, base, n, layout):
        fs, rs, ps, cs = layout
        assert (ps, cs) == (3, 1) and n >= 1
        owner = max(p for p in clip_twin.MEMORY if p <= base)
        data = clip_twin.MEMORY[owner].data
        off = base - owner
        last = off + (n - 1) * fs + (self.src_height - 1) * rs + (self.src_width - 1) * ps + 2
        assert 0 <= off and last <= data.size, "a layout reaches past its buffer"
        frames = np.lib.stride_tricks.as_strided(data[off:], shape=(n, self.src_height, self.src_width, 3),
                                                 strides=(fs, rs, ps, cs), writeable=False)
        SettingsEngine.layouts.append((n, tuple(layout)))
        OracleEngine.submit(self, np.ascontiguousarray(frames))


def _table(t, n_clips):
    """(offsets, first frames, end frames or None, step) of a PsdClipTable, from twin memory."""
    off = _array(t.offsets, np.int64, n_clips + 1)
    first = _array(t.first_frame, np.int64, n_clips) if t.first_frame else None
    end = _array(t.end_frame, np.int64, n_clips) if t.end_frame else None
    return off, first, end, int(t.frame_step)


def cut_lists_tables(cells, n_cells, tables, cell_table, n_clips, mf) -> list:
    """Every (cell, clip) list, cell-major: cell k over its own table, as one psd_clip_cuts_step call per cell."""
    lists = []
    for k in range(n_cells):
        off, first, end, step = _table(tables[cell_table[k] if cell_table is not None else 0], n_clips)
        lists += clip_window_twin.clip_cut_lists([cells[k]], 1, off, first, n_clips, mf[k * n_clips:], step, end)
    return lists


class Lib(clip_window_twin.Lib, sweep_clip_twin.Lib):
    def psd_clip_cuts_tables(self, cells, n_cells, tables, n_tables, cell_table, n_clips, min_frames, cuts, cap,
                             cut_offsets, st):
        assert n_tables >= 1 and all(tables[i].frame_step >= 1 for i in range(n_tables))
        assert cell_table is None or all(0 <= cell_table[k] < n_tables for k in range(n_cells))
        self._count("psd_clip_cuts_tables", 3)
        lists = cut_lists_tables(cells, n_cells, tables, cell_table, n_clips,
                                 _array(min_frames, np.int64, n_cells * n_clips))
        o = _array(cut_offsets, np.int64, n_cells * n_clips + 1)
        o[:] = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        if o[-1] <= cap and o[-1]:
            _array(cuts, np.int64, int(o[-1]))[:] = [c for x in lists for c in x]
        return 0

    def psd_clip_eval_tables(self, cuts, cut_offsets, n_cells, n_clips, cuts_total, max_cuts, tables, n_tables,
                             cell_table, gt_offsets, gt_cuts, n_gt, fade_offsets, fades, n_fades, tolerances, n_tol,
                             workspace, workspace_bytes_, out_n_pred, out_hard, out_fades, out_totals_hard,
                             out_totals_fades, out_over, st):
        assert workspace_bytes_ >= sweep_clip_twin.workspace_bytes(n_cells, n_clips, n_tol, cuts_total, n_gt, n_fades)
        self._count("psd_clip_eval_tables", 3)
        m = n_cells * n_clips
        off = _array(cut_offsets, np.int64, m + 1)
        assert int(off[-1]) == cuts_total
        c = _array(cuts, np.int64)
        ends = [_array(tables[i].end_frame, np.int64, n_clips) for i in range(n_tables)]
        go, fo = _array(gt_offsets, np.int64, n_clips + 1), _array(fade_offsets, np.int64, n_clips + 1)
        gt = _array(gt_cuts, np.int64, n_gt) if n_gt else []
        fd = _array(fades, np.int64, 2 * n_fades).reshape(-1, 2) if n_fades else []
        n_pred = _array(out_n_pred, np.int32, m)
        hard = _array(out_hard, np.int64, m * n_tol * 5).reshape(m, n_tol, 5)
        fc = _array(out_fades, np.int64, m * 3).reshape(m, 3)
        over = -1
        for t in range(m):
            k, j = divmod(t, n_clips)
            end = ends[cell_table[k] if cell_table is not None else 0]
            b, e = int(off[t]), int(off[t + 1])
            if e - b > max_cuts:
                n_pred[t], hard[t], fc[t] = -1, 0, 0
                over = t if over < 0 else over
                continue
            preds = sweep_model.predicted_list(c[b:e], int(end[j]))
            c[b:b + max(0, len(preds) - 1)] = preds[:-1]
            n_pred[t] = len(preds)
            hc = [int(x) for x in gt[go[j]:go[j + 1]]]
            fs = [(int(a), int(z)) for a, z in fd[fo[j]:fo[j + 1]]]
            for q in range(n_tol):
                h, f = sweep_model.score(preds, hc, fs, int(tolerances[q]))
                hard[t, q] = h
                if q == 0:
                    fc[t] = f
        _array(out_totals_hard, np.int64, n_cells * n_tol * 5)[:] = hard.reshape(n_cells, n_clips, -1).sum(1).ravel()
        _array(out_totals_fades, np.int64, n_cells * 3)[:] = fc.reshape(n_cells, n_clips, 3).sum(1).ravel()
        _array(out_over, np.int64, 1)[0] = over
        return 0
