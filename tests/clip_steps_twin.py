"""tests/clip_window_twin.py's library with psd_clip_cuts_steps: one frame step per clip.  The twin is the stepped
automata of clip_window_twin run once per clip with that clip's step, which is what the entry promises: clip j's lists
are those of psd_clip_cuts_step over clip j alone with frame_step[j]."""

from __future__ import annotations

import numpy as np

from tests import clip_window_twin
from tests.clip_twin import _array


def clip_cut_lists_steps(cells, n_cells, off, first, n_clips, mf, steps, end) -> list:
    """Every (cell, clip) list, cell-major, from host arrays: clip j through clip_window_twin.clip_cut_lists as a
    one-clip table with step steps[j] (end: the clips' end frames, or None)."""
    per_clip = []
    for j in range(n_clips):
        mf_j = [int(mf[k * n_clips + j]) for k in range(n_cells)]
        per_clip.append(clip_window_twin.clip_cut_lists(cells, n_cells, off[j:j + 2], first[j:j + 1], 1, mf_j,
                                                        int(steps[j]), end[j:j + 1] if end is not None else None))
    return [per_clip[j][k] for k in range(n_cells) for j in range(n_clips)]


class Lib(clip_window_twin.Lib):
    def psd_clip_cuts_steps(self, cells, n_cells, offsets, first, n_clips, min_frames, cuts, cap, cut_offsets, steps,
                            end, st):
        steps = [int(steps[j]) for j in range(n_clips)]  # a HOST array
        assert all(s >= 1 for s in steps)
        self._count("psd_clip_cuts_steps", 3)
        lists = clip_cut_lists_steps(cells, n_cells, _array(offsets, np.int64, n_clips + 1),
                                     _array(first, np.int64, n_clips), n_clips,
                                     _array(min_frames, np.int64, n_cells * n_clips), steps,
                                     _array(end, np.int64, n_clips) if end is not None else None)
        o = _array(cut_offsets, np.int64, n_cells * n_clips + 1)
        o[:] = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        if o[-1] <= cap and o[-1]:
            _array(cuts, np.int64, int(o[-1]))[:] = [c for x in lists for c in x]
        return 0
