"""Python twin of psd_clip_eval (clip_kernels.cu), on top of the clip-kernel twin of tests/clip_twin.py, so that
`ParameterSweep.run_clips` runs on a box with no GPU.  Each (cell, clip) list becomes its predicted list in place
(`sweep_model.predicted_list`), each (cell, clip, tolerance) is scored by `sweep_model.score`, and the counts are
summed over the clips, into the same device arrays the kernel writes."""

from __future__ import annotations

import numpy as np

from tests import clip_twin, sweep_model
from tests.clip_twin import _array


def workspace_bytes(n_cells, n_clips, n_tol, cuts_total, n_gt, n_fades) -> int:
    """include/psd_b200.h's size of the matching bitmaps, restated."""
    words = lambda bits: (bits + 31) // 32  # noqa: E731
    return 4 * (n_tol * (n_cells * n_clips + words(cuts_total))
                + n_cells * n_tol * (2 * n_clips + words(n_gt) + words(n_fades)))


class Lib(clip_twin.Lib):
    def psd_clip_eval(self, cuts, cut_offsets, n_cells, n_clips, cuts_total, max_cuts, ends, gt_offsets, gt_cuts, n_gt,
                      fade_offsets, fades, n_fades, tolerances, n_tol, workspace, workspace_bytes_, out_n_pred,
                      out_hard, out_fades, out_totals_hard, out_totals_fades, out_over, st):
        assert workspace_bytes_ >= workspace_bytes(n_cells, n_clips, n_tol, cuts_total, n_gt, n_fades)
        self._count("psd_clip_eval", 3)
        m = n_cells * n_clips
        off = _array(cut_offsets, np.int64, m + 1)
        assert int(off[-1]) == cuts_total
        c = _array(cuts, np.int64)
        end = _array(ends, np.int64, n_clips)
        go, fo = _array(gt_offsets, np.int64, n_clips + 1), _array(fade_offsets, np.int64, n_clips + 1)
        gt = _array(gt_cuts, np.int64, n_gt) if n_gt else []
        fd = _array(fades, np.int64, 2 * n_fades).reshape(-1, 2) if n_fades else []
        n_pred = _array(out_n_pred, np.int32, m)
        hard = _array(out_hard, np.int64, m * n_tol * 5).reshape(m, n_tol, 5)
        fc = _array(out_fades, np.int64, m * 3).reshape(m, 3)
        over = -1
        for t in range(m):
            j = t % n_clips
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
