"""Clip tables for the stepped cut automata (psd_clip_cuts_step), built from the recorded metric arrays of the
adversarial sequences of tests/automata_inputs.py: every sequence of one detector kind (and adaptive window) is one
clip of a pass, and the cells cover thresholds around the data, both modes, every fade_bias edge and several
min_frames."""

from __future__ import annotations

import math

import numpy as np

from tests import automata_inputs as A

MIN_FRAMES = (0, 1, 3, 15)


def _arr(values) -> np.ndarray:
    return np.array([math.nan if x is None else float.fromhex(x) for x in values], np.float64)


def _cases():
    """(group key, metric, metric2) of every recorded metric array."""
    for spec in A.sequences():
        m = A.recording()[spec["name"]]["metrics"]
        det = spec["det"]
        if det == "content":
            for w in spec["weights"]:
                yield ("content", 0), _arr(m[A.metric_key("content_val", w)]), None
        elif det == "adaptive":
            for key in sorted(k for k in m if k.startswith("adaptive_ratio|")):
                _, w, win, _mcv = key.split("|")
                yield ("adaptive", int(win)), _arr(m[key]), _arr(m["content_val|" + w])
        elif det == "threshold":
            yield ("threshold", 0), _arr(m[A.metric_key("average_rgb")]), None
        elif det == "histogram":
            yield ("histogram", 0), _arr(m[sorted(m)[0]]), None
        else:
            yield ("hash", 0), _arr(m[A.metric_key("hash_dist")]), None


def groups() -> list:
    """[(kind, window, clip sizes, metric, metric2 or None, cell parameter dicts)], one per pass."""
    by = {}
    for key, a, b in _cases():
        by.setdefault(key, []).append((a, b))
    out = []
    for (kind, window), items in sorted(by.items()):
        metric = np.concatenate([a for a, _ in items])
        metric2 = np.concatenate([b for _, b in items]) if items[0][1] is not None else None
        finite = metric[np.isfinite(metric)]
        q = (lambda p: float(np.percentile(finite, p))) if finite.size else (lambda p: 0.5)
        if kind == "content":
            params = [dict(threshold=q(p), mode=mode) for p in (50, 80, 95) for mode in (0, 1)]
        elif kind == "adaptive":
            params = [dict(threshold=t, min_content_val=v, window=window) for t in (1.5, 3.0) for v in (0.0, 15.0)]
        elif kind == "threshold":
            params = [dict(threshold=float(t), mode=mode, fade_bias=bias, add_final_scene=1)
                      for t in (12, 40) for mode in (0, 1) for bias in (-1.0, 0.0, 0.5, 1.0, 1.5)]
        elif kind == "histogram":
            params = [dict(threshold=q(p)) for p in (10, 40)]
        else:
            params = [dict(threshold=q(p)) for p in (60, 90)]
        out.append((kind, window, [len(a) for a, _ in items], metric, metric2, params))
    return out


def cells_and_min_frames(kind: str, params: list, metric_ptr: int, metric2_ptr, n_clips: int, seed: int):
    """ctypes cells (one per parameter set and min_frames) and min_frames[n_cells * n_clips]."""
    from pyscenedetect_b200 import _capi
    kinds = dict(content=_capi.SWEEP_CONTENT, adaptive=_capi.SWEEP_ADAPTIVE, threshold=_capi.SWEEP_THRESHOLD,
                 histogram=_capi.SWEEP_HISTOGRAM, hash=_capi.SWEEP_HASH)
    plist = [(p, mf) for p in params for mf in MIN_FRAMES]
    cells = (_capi.PsdSweepCell * len(plist))()
    for i, (p, _) in enumerate(plist):
        cells[i] = _capi.PsdSweepCell(kind=kinds[kind], metric=metric_ptr, metric2=metric2_ptr, **p)
    rng = np.random.default_rng(seed)
    mf = np.array([mf if j % 3 else int(rng.integers(0, 40)) for _, mf in plist for j in range(n_clips)], np.int64)
    return cells, len(plist), mf


def first_and_end(sizes, step: int, seed: int):
    """Each clip's first frame and end frame (its end position + 1: between the last element's frame and up to
    step - 1 frames past it, as skipped reads leave it)."""
    rng = np.random.default_rng(seed)
    first = rng.integers(0, 20000, len(sizes)).astype(np.int64)
    last = first + (np.maximum(np.array(sizes), 1) - 1) * step
    end = last + 1 + rng.integers(0, step, len(sizes))
    return first, end.astype(np.int64)
