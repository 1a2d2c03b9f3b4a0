"""tests/clip_twin.py's library with psd_clip_cuts_step: the five automata of cut_automata.cuh restated with the frame
step (element i is frame first + i * step) and ThresholdDetector's post_process position, so that `detect_clips` with
`frame_skip` runs on a box with no GPU.  With step 1 and no end frames these are clip_twin's automata."""

from __future__ import annotations

import numpy as np

from pyscenedetect_b200 import _capi
from tests import stats_clip_twin
from tests.clip_twin import _array


def flash_filter_cuts(above, n, first, step, min_frames, mode, out):
    if min_frames <= 0:
        out.extend(first + i * step for i in range(n) if above(i))
        return
    last_above, merge_enabled, merge_triggered, merge_start = first, False, False, 0
    for i in range(n):
        t = first + i * step
        a = above(i)
        met = (t - last_above) >= min_frames
        if mode == 1:
            if a and met:
                last_above = t
                out.append(t)
            continue
        if a:
            last_above = t
        if merge_triggered:
            if met and not a and (last_above - merge_start) >= min_frames:
                merge_triggered = False
                out.append(last_above)
            continue
        if not a:
            continue
        if met:
            merge_enabled = True
            out.append(t)
        elif merge_enabled:
            merge_triggered, merge_start = True, t


def adaptive_cuts(ratio, score, n, first, step, w, thr, mcv, min_frames, out):
    last_cut = first
    for i in range(w, n - w):
        met = ratio[i] >= thr and score[i] >= mcv
        if met and (first + (i + w) * step - last_cut) >= min_frames:
            last_cut = first + i * step
            out.append(last_cut)


def histogram_cuts(correl, n, first, step, thr, min_frames, out):
    last_cut = first
    for i in range(1, n):
        t = first + i * step
        if correl[i] <= thr and (t - last_cut) >= min_frames:
            out.append(t)
            last_cut = t


def hash_cuts(dist, n, first, step, thr, min_frames, out):
    last_cut = first
    for i in range(n):
        d = dist[i]
        if d != d:
            continue
        t = first + i * step
        if d >= thr and (t - last_cut) >= min_frames:
            out.append(t)
            last_cut = t


def threshold_cuts(avg, n, first, step, last, thr, ceiling, fade_bias, min_frames, add_final, out):
    if n <= 0:
        return
    last_scene_cut = fade_frame = first
    fade_in = not (avg[0] < thr)
    for i in range(1, n):
        t = first + i * step
        v = avg[i]
        below = (v >= thr) if ceiling else (v < thr)
        if fade_in and below:
            fade_in, fade_frame = False, t
        elif not fade_in and not below:
            if (t - last_scene_cut) >= min_frames:
                out.append(fade_frame + round(((t - fade_frame) * (1.0 + fade_bias)) / 2.0))
                last_scene_cut = t
            fade_in, fade_frame = True, t
    if not fade_in and add_final and (last - last_scene_cut) >= min_frames:
        out.append(fade_frame)


def run_cell(c, base, n, first, step, last, min_frames, out):
    m = _array(c.metric, np.float64)[base:base + n]
    if c.kind == _capi.SWEEP_CONTENT:
        flash_filter_cuts(lambda i: m[i] >= c.threshold, n, first, step, min_frames, c.mode, out)
    elif c.kind == _capi.SWEEP_ADAPTIVE:
        adaptive_cuts(m, _array(c.metric2, np.float64)[base:base + n], n, first, step, c.window, c.threshold,
                      c.min_content_val, min_frames, out)
    elif c.kind == _capi.SWEEP_THRESHOLD:
        threshold_cuts(m, n, first, step, last, c.threshold, c.mode, c.fade_bias, min_frames, c.add_final_scene, out)
    elif c.kind == _capi.SWEEP_HISTOGRAM:
        histogram_cuts(m, n, first, step, c.threshold, min_frames, out)
    else:
        hash_cuts(m, n, first, step, c.threshold, min_frames, out)


def clip_cut_lists(cells, n_cells, off, first, n_clips, mf, step, end) -> list:
    """Every (cell, clip) list, cell-major, from host arrays (end: the clips' end frames, or None)."""
    lists = []
    for k in range(n_cells):
        for j in range(n_clips):
            b = max(int(off[j]), 0)
            e = max(int(off[j + 1]), b)
            f = int(first[j])
            last = int(end[j]) - 1 if end is not None else f + (e - b - 1) * step
            out = []
            run_cell(cells[k], b, e - b, f, step, last, int(mf[k * n_clips + j]), out)
            lists.append(out)
    return lists


class Lib(stats_clip_twin.Lib):
    def psd_clip_cuts_step(self, cells, n_cells, offsets, first, n_clips, min_frames, cuts, cap, cut_offsets, step,
                           end, st):
        assert step >= 1
        self._count("psd_clip_cuts", 3)
        lists = clip_cut_lists(cells, n_cells, _array(offsets, np.int64, n_clips + 1), _array(first, np.int64, n_clips),
                               n_clips, _array(min_frames, np.int64, n_cells * n_clips), step,
                               _array(end, np.int64, n_clips) if end is not None else None)
        o = _array(cut_offsets, np.int64, n_cells * n_clips + 1)
        o[:] = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        if o[-1] <= cap and o[-1]:
            _array(cuts, np.int64, int(o[-1]))[:] = [c for x in lists for c in x]
        return 0
