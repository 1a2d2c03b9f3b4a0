"""tests/clip_twin.py's library with psd_clip_stats_csv and the content scan's components, so that
`detect_clips(stats=True)` runs on a box with no GPU.  The text comes from tests/stats_csv_twin.py."""

from __future__ import annotations

import numpy as np

from tests import clip_twin, stats_csv_twin
from tests.clip_twin import _array


class Lib(clip_twin.Lib):
    def psd_scan_content_edges(self, sums, sads, n, n_pixels, w, wsum, comps, out, st):
        super().psd_scan_content_edges(sums, sads, n, n_pixels, w, wsum, comps, out, st)
        if comps is not None:
            _array(comps, np.float64, 4 * n)[:] = sums.scan_content(list(w))[1].reshape(-1)
        return 0

    def psd_clip_stats_csv(self, columns, n_columns, offsets, first, rates, n_clips, n, row_offsets, out, cap,
                           clip_bytes, st):
        cb = _array(clip_bytes, np.int64, n_clips + 1)
        if n == 0 or n_clips == 0:
            cb[:] = 0
            return 0
        self._count("psd_clip_stats_csv", 3)
        cols = [(_array(c.values, np.float64), c.stride, c.head, c.tail) for c in columns[:n_columns]]
        text, offs = stats_csv_twin.pass_csv(cols, _array(offsets, np.int64, n_clips + 1),
                                             _array(first, np.int64, n_clips), _array(rates, np.float64, n_clips))
        cb[:] = offs
        if len(text) <= cap:
            _array(out, np.uint8, len(text))[:] = np.frombuffer(text, np.uint8)
        return 0
