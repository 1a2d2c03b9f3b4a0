"""Scripted per-frame integer results for the cut-automata tests: what the engine would hold for a sequence
(psd_frame_sums rows, 256-bin Y histograms, perceptual-hash words), written directly, without pixels, so
that the stage from integer sums to cut list can be driven through its edges - ties with the threshold,
spikes at exactly the minimum spacing, all-zero adaptive windows, fades of odd and even length, degenerate
histograms, hash distances of exactly k/size^2.

Every sequence is built deterministically from its spec.  The inputs are ones the engine can produce:
`has_prev` is 0 on frame 0 only, the hue SAD is at most 179 per pixel and the other SADs at most 255 per
pixel, the edge SAD is 0 unless the sequence's weights give the edge component a positive weight, every
histogram sums to the pixel count and only the low size^2 bits of a hash are set.

tests/golden/make_automata_golden.py records what PySceneDetect 0.7.1 computes from these inputs in
tests/golden/automata_v1.json.gz; tests/test_automata_reference.py (the oracle) and tests/test_gpu_automata.py
(the device scans, automata and sweep) compare against that recording.  The frame builders below give the
reference real frames whose byte sum (ThresholdDetector) or Y histogram (HistogramDetector) is the scripted
one.
"""

from __future__ import annotations

import functools
import gzip
import hashlib
import json
import os
import random
import zlib
from dataclasses import dataclass

import numpy as np

from pyscenedetect_b200._capi import HASH_WORDS, SUMS_DTYPE

FPS = (30.0, 25.0, 24000 / 1001)
FIRST_FRAMES = (0, 1, 12345)
UHD = 3840 * 2160

# weight vectors: sequences with an edge SAD use only the positive-edge-weight ones
PLAIN_WEIGHTS = ((1.0, 1.0, 1.0, 0.0), (0.0, 0.0, 1.0, 0.0), (1.0, 0.0, 1.0, 0.0))
EDGE_WEIGHTS = ((0.5, 0.25, 1.0, 2.0), (1.0, 1.0, 1.0, 1.0))
HIST_BINS = (1, 2, 3, 7, 16, 100, 127, 128, 129, 200, 255, 256)
HASH_SIZES = (1, 4, 8, 12, 16)
FADE_BIASES = (-1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 1.5)


@dataclass
class Inputs:
    sums: np.ndarray                 # (n,) SUMS_DTYPE
    yhist: np.ndarray | None         # (n, 256) uint32
    hashes: np.ndarray | None        # (n, HASH_WORDS) uint64
    n_pixels: int
    hash_size: int = 8

    def sha256(self) -> str:
        h = hashlib.sha256()
        h.update(np.int64(self.n_pixels).tobytes())
        h.update(np.int64(self.hash_size).tobytes())
        for a in (self.sums, self.yhist, self.hashes):
            h.update(b"-" if a is None else np.ascontiguousarray(a).tobytes())
        return h.hexdigest()


def _rng(spec) -> random.Random:
    return random.Random(zlib.crc32(spec["name"].encode()))


def _empty_sums(n: int) -> np.ndarray:
    s = np.zeros(n, dtype=SUMS_DTYPE)
    if n:
        s["has_prev"][1:] = 1
    return s


# --- content / adaptive -------------------------------------------------------------------------------------

def _content_levels(rng: random.Random, n: int, m: int, pattern: str) -> list[float]:
    """Per-frame luma level (mean absolute difference per pixel, 0..255) of one of the scripted patterns."""
    lo = lambda: rng.choice([0.0, 0.5, 2.0, 4.0, 7.5])  # noqa: E731
    heights = [rng.choice([30.0, 40.0, 55.0]), rng.choice([27.0, 60.0, 90.0])]
    lev: list[float] = []
    while len(lev) < n:
        kind = pattern if pattern != "mixed" else rng.choice(["spikes", "bursts", "plateau"])
        if kind in ("spikes", "tie"):
            for _ in range(rng.randint(3, 8)):
                lev += [lo() for _ in range(rng.choice([m - 1, m, m + 1]) - 1)] + [rng.choice(heights)]
        elif kind == "bursts":
            for _ in range(rng.randint(2, 5)):
                lev += [rng.choice(heights)] + [lo() for _ in range(rng.randint(0, max(0, m - 2)))]
            lev += [lo() for _ in range(rng.randint(1, 2 * m + 2))]
        else:
            lev += [rng.choice(heights) + rng.random() for _ in range(rng.randint(1, 3 * m))]
            lev += [lo() for _ in range(rng.randint(1, 2 * m))]
    return lev[:n]


def _sums_from_levels(rng: random.Random, lev, P: int, edges: bool, jitter: float) -> np.ndarray:
    n = len(lev)
    s = _empty_sums(n)
    fh, fs, fe = rng.uniform(0.2, 1.0), rng.uniform(0.2, 1.0), rng.uniform(0.5, 2.0)
    for i in range(1, n):
        L = lev[i]
        j = lambda: 1.0 + jitter * (rng.random() - 0.5)  # noqa: E731
        s["sad_lum"][i] = min(255 * P, round(L * P * j()))
        s["sad_hue"][i] = min(179 * P, round(L * P * fh * j()))
        s["sad_sat"][i] = min(255 * P, round(L * P * fs * j()))
        s["sad_edges"][i] = min(255 * P, round(L * P * fe * j())) if edges else 0
    s["bgr_sum"] = [rng.randint(0, 765 * P) for _ in range(n)]
    return s


def _content(spec) -> Inputs:
    rng = _rng(spec)
    n, P, m, pattern = spec["n"], spec["P"], spec["m"], spec["pattern"]
    lev = _content_levels(rng, n, m, pattern)
    s = _sums_from_levels(rng, lev, P, spec["edges"], 0.0 if pattern == "tie" else 0.1)
    if pattern == "tie":
        # spikes one SAD unit either side of an integer score: about 1.2e-7 from the threshold at 3840x2160
        for i in range(1, n):
            if lev[i] >= 27.0:
                s["sad_lum"][i] = int(s["sad_lum"][i]) + rng.choice([-1, 0, 0, 1])
    return Inputs(s, None, None, P)


def _adaptive(spec) -> Inputs:
    rng = _rng(spec)
    n, P, pattern = spec["n"], spec["P"], spec["pattern"]
    if pattern == "mixed":
        return _content(dict(spec, pattern="mixed", edges=spec["edges"]))
    s = _empty_sums(n)
    heights = [rng.choice([10.0, 14.0]), 15.0, rng.choice([16.0, 40.0])]
    for i in range(1, n):
        if pattern == "zero_windows":
            # isolated targets: sometimes further apart than any window, sometimes inside one
            lum = rng.choice(heights) * P if rng.random() < 0.2 else 0
        elif pattern == "near_zero":
            # 3840x2160: a background of 0..90 SAD units averages just below and just above 1e-5
            lum = rng.choice([20, 40]) * P if rng.random() < 0.15 else rng.choice([0, 1, 80, 83, 84, 90])
        else:  # "clamp": small but non-zero windows, large targets -> ratios clamped at 255
            lum = rng.choice([60, 200]) * P if rng.random() < 0.2 else rng.choice([0, 1, 2])
        s["sad_lum"][i] = min(255 * P, lum)
        s["sad_hue"][i] = 0
        s["sad_sat"][i] = min(255 * P, lum // 3)
    return Inputs(s, None, None, P)


# --- threshold ----------------------------------------------------------------------------------------------

def _threshold(spec) -> Inputs:
    rng = _rng(spec)
    n, P, T = spec["n"], spec["P"], spec["T"]
    s = _empty_sums(n)
    vals = []
    state_in = spec["first_in"]
    while len(vals) < n:
        run = rng.randint(1, 9)
        for _ in range(run):
            r = rng.random()
            if r < 0.2:
                v = T * 3 * P                                   # exactly the threshold
            elif state_in:
                v = T * 3 * P + rng.randint(1, 40 * 3 * P)
            else:
                v = T * 3 * P - rng.randint(1, min(T * 3 * P, 3 * P * 8) or 1)
            vals.append(max(0, min(765 * P, v)))
        state_in = not state_in
    vals = vals[:n]
    if spec.get("end_out") and n >= 3:
        for i in range(max(1, n - rng.randint(1, 4)), n):
            vals[i] = max(0, T * 3 * P - 1 - rng.randint(0, 3 * P))
    s["bgr_sum"] = vals
    return Inputs(s, None, None, P)


def threshold_frame(bgr_sum: int, shape) -> np.ndarray:
    """A (h, w, 3) uint8 frame whose byte sum is `bgr_sum`: bytes q or q + 1."""
    h, w = shape
    total = h * w * 3
    q, r = divmod(int(bgr_sum), total)
    flat = np.full(total, q, dtype=np.uint8)
    flat[:r] += 1
    return flat.reshape(h, w, 3)


# --- histogram ----------------------------------------------------------------------------------------------

def _hist_frame(rng: random.Random, P: int, prev: np.ndarray | None, kind: str) -> np.ndarray:
    h = np.zeros(256, dtype=np.int64)
    if kind == "identical" and prev is not None:
        return prev.copy()
    if kind == "near" and prev is not None:
        h = prev.copy()
        for _ in range(rng.randint(1, 3)):
            src = rng.choice(np.nonzero(h)[0].tolist())
            dst = min(255, max(0, src + rng.choice([-1, 1])))
            k = rng.randint(1, int(h[src]))
            h[src] -= k
            h[dst] += k
        return h
    if kind == "single":
        h[rng.randrange(256)] = P
    elif kind == "uniform":
        q, r = divmod(P, 256)
        h[:] = q
        h[:r] += 1
    elif kind == "disjoint":
        lo = 0 if prev is None or int(np.argmax(prev)) >= 128 else 128
        a = rng.randrange(lo, lo + 120)
        b = rng.randrange(a + 1, lo + 128)
        cuts = sorted(rng.randint(0, P) for _ in range(b - a - 1))
        h[a:b] = np.diff([0, *cuts, P])
    else:  # "random": a random bump plus a floor
        centre, width = rng.randrange(256), rng.uniform(3, 80)
        p = np.exp(-0.5 * ((np.arange(256) - centre) / width) ** 2) + rng.random() * 0.05
        h = np.bincount(np.random.default_rng(rng.randrange(1 << 30)).choice(256, size=P, p=p / p.sum()),
                        minlength=256).astype(np.int64)
    return h


def _histogram(spec) -> Inputs:
    rng = _rng(spec)
    n, (hh, ww) = spec["n"], spec["shape"]
    P = hh * ww
    kinds = spec.get("kinds") or ["single", "uniform", "disjoint", "identical", "near", "random"]
    rows, prev = [], None
    for _ in range(n):
        prev = _hist_frame(rng, P, prev, rng.choice(kinds))
        assert prev.sum() == P
        rows.append(prev)
    yh = np.asarray(rows, dtype=np.uint32).reshape(n, 256)
    return Inputs(_empty_sums(n), yh, None, P)


def _uhd8k_histograms(spec) -> Inputs:
    """7680x4320: single bins of 2^24 + 1 and more pixels, where calcHist's float32 counts round."""
    hh, ww = spec["shape"]
    P = hh * ww
    big = (1 << 24) + 1
    rows = []
    for split in ((7, P), (7, big, 200, P - big), (7, P - big, 9, big), (255, big + 3, 0, P - big - 3),
                  (255, big + 3, 0, P - big - 3)):
        h = np.zeros(256, dtype=np.int64)
        if len(split) == 2:
            h[split[0]] = split[1]
        else:
            h[split[0]], h[split[2]] = split[1], split[3]
        rows.append(h)
    return Inputs(_empty_sums(len(rows)), np.asarray(rows, dtype=np.uint32), None, P)


def gray_frame(hist_row: np.ndarray, shape) -> np.ndarray:
    """A (h, w, 3) gray frame (B = G = R = v, whose Y is v) with the given per-value pixel counts."""
    h, w = shape
    v = np.repeat(np.arange(256, dtype=np.uint8), np.asarray(hist_row, dtype=np.int64))
    return np.repeat(v.reshape(h, w, 1), 3, axis=2)


# --- hash ---------------------------------------------------------------------------------------------------

def _hash(spec) -> Inputs:
    rng = _rng(spec)
    n, size = spec["n"], spec["size"]
    nb = size * size
    ks = sorted({max(1, nb // 8), max(1, nb // 4), max(1, (nb * 35 + 99) // 100), max(1, nb // 2)})
    bits = []
    cur = np.array([rng.random() < 0.5 for _ in range(nb)], dtype=bool)
    for _ in range(n):
        r = rng.random()
        if r < 0.25:
            pass                                           # identical to the previous frame
        elif r < 0.8:
            k = min(nb, rng.choice(ks) + rng.choice([-1, 0, 0, 1]))
            if k > 0:
                idx = rng.sample(range(nb), k)
                cur = cur.copy()
                cur[idx] = ~cur[idx]
        else:
            cur = np.array([rng.random() < 0.5 for _ in range(nb)], dtype=bool)
        bits.append(cur)
    words = np.zeros((n, HASH_WORDS), dtype=np.uint64)
    for i, b in enumerate(bits):
        for j in np.nonzero(b)[0]:
            words[i, j // 64] |= np.uint64(1) << np.uint64(j % 64)
    return Inputs(_empty_sums(n), None, words, 1, hash_size=size)


def hash_bits(words_row: np.ndarray, size: int) -> np.ndarray:
    """The (size, size) bool array whose flattened bit j is bit j % 64 of word j // 64."""
    nb = size * size
    j = np.arange(nb)
    w = np.asarray(words_row, dtype=np.uint64)[j // 64]
    return ((w >> (j % 64).astype(np.uint64)) & np.uint64(1)).astype(bool).reshape(size, size)


# --- the sequences ------------------------------------------------------------------------------------------

def _common(det: str, j: int, rng: random.Random) -> dict:
    return dict(name=f"{det}_{j:02d}", det=det, fps=FPS[j % 3], first_frame=FIRST_FRAMES[(j // 3) % 3])


def sequences() -> list[dict]:
    """Every scripted sequence's spec, in a fixed order."""
    rng = random.Random(20261015)
    out = []
    for j in range(40):
        sp = _common("content", j, rng)
        pattern = ["spikes", "bursts", "plateau", "mixed", "tie"][j % 5]
        edges = pattern != "tie" and j % 2 == 1
        sp.update(pattern=pattern, m=[15, 10, 6, 3][j % 4], edges=edges,
                  P=UHD if pattern == "tie" else [1, 7, 160 * 90, 1000][(j // 5) % 4],
                  n=[1, 2][j] if j < 2 else rng.randint(150, 450))
        sp["weights"] = [list(w) for w in (EDGE_WEIGHTS if edges else
                                           (PLAIN_WEIGHTS[1:2] + PLAIN_WEIGHTS[0:1] if pattern == "tie" else
                                            PLAIN_WEIGHTS))]
        out.append(sp)
    for j in range(40):
        sp = _common("adaptive", j, rng)
        pattern = ["zero_windows", "near_zero", "clamp", "mixed"][j % 4]
        short = j < 12
        sp.update(pattern=pattern, m=[15, 6, 3][j % 3], edges=pattern == "mixed" and j % 8 == 7,
                  P=UHD if pattern == "near_zero" else [1, 5, 1000][j % 3],
                  n=[2, 3, 4, 5, 6, 10, 11, 12, 1, 2, 3, 7][j] if short else rng.randint(120, 400))
        sp["weights"] = [list(w) for w in (EDGE_WEIGHTS[:1] if sp["edges"] else
                                           (PLAIN_WEIGHTS[1:2] if pattern != "mixed" else PLAIN_WEIGHTS[:2]))]
        out.append(sp)
    for j in range(40):
        sp = _common("threshold", j, rng)
        sp.update(P=[1, 5, 16, 14400][j % 4], T=[12, 40, 100, 1][(j // 4) % 4], first_in=j % 2 == 0,
                  end_out=(j // 2) % 2 == 0, n=[1, 2][j] if j < 2 else rng.randint(60, 300))
        sp["shape"] = {1: (1, 1), 5: (1, 5), 16: (4, 4), 14400: (90, 160)}[sp["P"]]
        out.append(sp)
    for j in range(40):
        sp = _common("histogram", j, rng)
        sp.update(shape=[(1, 256), (9, 16), (90, 160), (7, 37), (1, 1)][j % 5],
                  n=[1, 2][j] if j < 2 else rng.randint(30, 90))
        if j % 7 == 3:
            sp["kinds"] = ["single", "uniform", "identical"]
        elif j % 7 == 5:
            sp["kinds"] = ["near", "identical", "random"]
        out.append(sp)
    sp = _common("histogram", 40, rng)
    sp.update(name="histogram_8k", shape=(4320, 7680), n=5, uhd8k=True)
    out.append(sp)
    for j in range(40):
        sp = _common("hash", j, rng)
        sp.update(size=HASH_SIZES[j % 5], n=[1, 2][j] if j < 2 else rng.randint(80, 300))
        out.append(sp)
    # one empty sequence per detector: no frame, no metric, no cut
    for det, extra in (("content", dict(pattern="spikes", m=15, edges=False, P=160 * 90,
                                        weights=[list(w) for w in PLAIN_WEIGHTS])),
                       ("adaptive", dict(pattern="zero_windows", m=15, edges=False, P=1,
                                         weights=[list(PLAIN_WEIGHTS[1])])),
                       ("threshold", dict(P=5, T=12, first_in=True, end_out=False, shape=(1, 5))),
                       ("histogram", dict(shape=(9, 16))),
                       ("hash", dict(size=8))):
        sp = dict(name=f"{det}_empty", det=det, fps=FPS[0], first_frame=FIRST_FRAMES[2], n=0, **extra)
        out.append(sp)
    return out


def build(spec) -> Inputs:
    det = spec["det"]
    if det == "content":
        return _content(spec)
    if det == "adaptive":
        return _adaptive(spec)
    if det == "threshold":
        return _threshold(spec)
    if det == "histogram":
        return _uhd8k_histograms(spec) if spec.get("uhd8k") else _histogram(spec)
    return _hash(spec)


def frame_source(spec, inp: Inputs, i: int) -> np.ndarray:
    """Frame i as the reference is given it: real pixels where the reference computes the metric from them
    (threshold, histogram), otherwise a small dummy frame (content and adaptive read the patched pixel
    distance; hash reads the patched hash, which finds the frame index in the dummy frame's first bytes)."""
    det = spec["det"]
    if det == "threshold":
        return threshold_frame(int(inp.sums["bgr_sum"][i]), spec["shape"])
    if det == "histogram":
        return gray_frame(inp.yhist[i], spec["shape"])
    return index_frame(i)


def index_frame(i: int) -> np.ndarray:
    """A 1x1 BGR frame that carries frame index i (< 2^24) in its three bytes; `frame_index` reads it back."""
    return np.frombuffer(np.int64(i).tobytes()[:3], dtype=np.uint8).reshape(1, 1, 3).copy()


def frame_index(frame: np.ndarray) -> int:
    b = np.asarray(frame, dtype=np.uint8).reshape(-1)[:3]
    return int(b[0]) | int(b[1]) << 8 | int(b[2]) << 16


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "automata_v1.json.gz")


@functools.lru_cache(maxsize=1)
def recording() -> dict:
    """The recorded reference results, by sequence name."""
    with gzip.open(GOLDEN, "rt") as f:
        doc = json.load(f)
    return {s["spec"]["name"]: s for s in doc["sequences"]}


def recorded(spec) -> tuple[dict, Inputs]:
    """The recorded entry of `spec` and its inputs, after checking that this module still builds the inputs
    the recording was made from."""
    rec = recording()[spec["name"]]
    assert json.loads(json.dumps(spec)) == rec["spec"], "sequence spec drifted from the recording"
    inp = build(spec)
    assert inp.sha256() == rec["sha256"], "scripted inputs drifted from the recording"
    return rec, inp


def metric_key(name: str, *params) -> str:
    """The recording's key of one per-frame metric array, e.g. `content_val|[1.0, 1.0, 1.0, 0.0]`."""
    def text(p):
        if isinstance(p, (list, tuple)):
            return repr([float(x) for x in p])
        return repr(float(p)) if isinstance(p, float) else repr(int(p))
    return "|".join([name, *(text(p) for p in params)])


def components(inp: Inputs, i: int) -> list[float]:
    """The four per-pixel mean differences of frame i, as content_detector._mean_pixel_distance returns them
    (numpy integer sum / float(num_pixels))."""
    s = inp.sums[i]
    return [np.int64(s[k]) / float(inp.n_pixels) for k in ("sad_hue", "sad_sat", "sad_lum", "sad_edges")]
