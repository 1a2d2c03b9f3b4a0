"""Python restatement of the device scorer (psd_sweep_eval, sweep_kernels.cu), in the kernel's own
formulation: fade intervals first (first hit in the order given), then hard cuts with the distance-outer
greedy walk - for d = 0..tol, for each remaining prediction in order, claim g = p - d, else g = p + d.
tests/test_sweep_host.py pins it against the reference evaluator's sort-based matching
(benchmark/evaluator.py:227-331) recorded in tests/golden/sweep_v1.json."""

from __future__ import annotations

import bisect


def predicted_list(cuts, end_frame: int) -> list[int]:
    """benchmark/sweep.py:169: `scene[1]` of every scene = sorted unique cuts, then the end position."""
    u = sorted(set(int(c) for c in cuts))
    return u + [int(end_frame)] if u else []


def score(preds, hard_cuts, fades, tol: int):
    """-> (matched, false_positives, missed, offset_sum, offset_count), (fade matched, fp, missed)."""
    preds = [int(p) for p in preds]
    used_p = [False] * len(preds)
    used_f = [False] * len(fades)
    fm = ffp = 0
    for i, p in enumerate(preds):
        for f, (a, b) in enumerate(fades):
            if a <= p <= b:
                used_p[i] = True
                if used_f[f]:
                    ffp += 1
                else:
                    used_f[f] = True
                    fm += 1
                break
    remaining = len(preds) - sum(used_p)
    used_g = [False] * len(hard_cuts)

    def find(g):
        j = bisect.bisect_left(hard_cuts, g)
        return j if j < len(hard_cuts) and hard_cuts[j] == g and not used_g[j] else -1

    matched = offset = 0
    for d in range(tol + 1):
        for i, p in enumerate(preds):
            if used_p[i]:
                continue
            j = find(p - d)
            if j < 0 and d:
                j = find(p + d)
            if j < 0:
                continue
            used_g[j] = used_p[i] = True
            matched += 1
            offset += d
    return ((matched, remaining - matched, len(hard_cuts) - matched, offset, matched),
            (fm, ffp, len(fades) - fm))
