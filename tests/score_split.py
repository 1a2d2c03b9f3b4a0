"""Python twin of the fused score pass's work split (csrc/score_kernel.cu: `pick_chunks`, `chunk_first`,
`ws_item`, `launch_ws`).  The GPU tests use it only to CHOOSE frame counts that reach every decomposition case
and to assert that they did; no pass/fail comparison of a result depends on it.  test_score_split.py pins the
constants below to the kernel source, so a change of the split there fails loudly instead of silently thinning
the coverage."""

from __future__ import annotations

from dataclasses import dataclass

WS_CONSUMER_WARPS = 24   # kWsConsumerWarps
PX_PER_THREAD = 16       # kPxPerThread
WS_UNROLL = 4            # kWsUnroll
WS_STAGES = 4            # kWsStages
SHORT_WALK = 8           # pick_chunks: `longest < 8 && c > 1` ends the search
CHUNK_CAP = 4096         # pick_chunks: at most 4 096 chunks
STRIP_PX = WS_CONSUMER_WARPS * 32 * PX_PER_THREAD   # kWsStripPx = 12 288


def pick_chunks(n_frames: int, n_strips: int, grid: int) -> int:
    best_cost, best = -1, 1
    for c in range(1, min(n_frames, CHUNK_CAP) + 1):
        longest = (n_frames + c - 1) // c
        if longest < SHORT_WALK and c > 1:
            break
        per_cta = (n_strips * c + grid - 1) // grid
        cost = per_cta * (longest + 1)
        if best_cost < 0 or cost < best_cost:
            best_cost, best = cost, c
    return best


def chunk_first(c: int, n_frames: int, n_chunks: int) -> int:
    return c * n_frames // n_chunks


@dataclass(frozen=True)
class Item:
    strip: int
    chunk: int
    f0: int
    nf: int
    halo: bool
    walked: int
    slots: int


@dataclass(frozen=True)
class Split:
    """One launch of psd_score_ws_kernel<F> (None when P < 16: only the tail kernel runs)."""
    n_strips: int
    n_chunks: int
    grid: int
    items: tuple

    def cta_items(self, b: int) -> list:
        return list(self.items[b::self.grid])

    @property
    def remainders(self) -> set:
        """(walked mod 4, halo) of every item."""
        return {(it.walked % WS_UNROLL, it.halo) for it in self.items}

    @property
    def mixed_slot_cta(self) -> bool:
        """Some CTA walks items with different slot counts."""
        return any(len({it.slots for it in self.cta_items(b)}) > 1 for b in range(self.grid))


def split(n_pixels: int, n_frames: int, hsv: bool, has_prev: bool, sm_count: int) -> Split | None:
    """The launch `launch_score` makes for one batch of `n_frames` frames of `n_pixels` pixels.  `hsv`: the mask
    contains F_HSV (or F_EDGES, which implies it); `has_prev`: the batch has a predecessor frame (carried or
    halo)."""
    p16 = n_pixels & ~15
    if p16 == 0:
        return None
    strips = (p16 + STRIP_PX - 1) // STRIP_PX
    chunks = min(pick_chunks(n_frames, strips, sm_count), n_frames)
    n_items = chunks * strips
    items = []
    for i in range(n_items):
        chunk, strip = i % chunks, i // chunks
        f0 = chunk_first(chunk, n_frames, chunks)
        nf = chunk_first(chunk + 1, n_frames, chunks) - f0
        halo = hsv and (f0 > 0 or has_prev)
        walked = nf + (1 if halo else 0)
        slots = (walked + WS_UNROLL - 1) // WS_UNROLL * WS_UNROLL
        items.append(Item(strip, chunk, f0, nf, halo, walked, slots))
    return Split(strips, chunks, min(n_items, sm_count), tuple(items))


def coverage(n_pixels: int, launches, sm_count: int) -> set:
    """Decomposition cases reached by a list of launches (n_frames, has_prev):
    ("hsv", walked mod 4, halo) for the masks with HSV, ("plain", walked mod 4) for the others, "few" (a launch
    with fewer items than SMs) and "mixed" (a CTA whose items have different slot counts)."""
    got = set()
    for n, has_prev in launches:
        for hsv in (True, False):
            s = split(n_pixels, n, hsv, has_prev, sm_count)
            if s is None:
                continue
            for r, halo in s.remainders:
                got.add(("hsv", r, halo) if hsv else ("plain", r))
            if len(s.items) < sm_count:
                got.add("few")
            if s.mixed_slot_cta:
                got.add("mixed")
    return got


def required_cases() -> set:
    """What the launches of every scored geometry must reach: each `walked mod 4`, with and without a halo frame
    for the masks with HSV."""
    return {("hsv", r, h) for r in range(WS_UNROLL) for h in (False, True)} | {("plain", r) for r in range(WS_UNROLL)}


def choose_launches(n_pixels: int, sm_count: int, n_max: int = 24) -> list:
    """A short list of launches (n_frames, has_prev) that reaches every case of `required_cases`: greedy, the
    launch that adds the most missing cases per frame first."""
    want = required_cases()
    got, out = set(), []
    cands = [(n, p) for n in range(1, n_max + 1) for p in (False, True)]
    while not want <= got:
        best = max(cands, key=lambda c: (len((coverage(n_pixels, [c], sm_count) & want) - got) / c[0], -c[0]))
        new = (coverage(n_pixels, [best], sm_count) & want) - got
        if not new:
            raise AssertionError(f"no launch of <= {n_max} frames reaches {sorted(map(str, want - got))}")
        got |= new
        out.append(best)
    return out


def find_mixed_launch(n_pixels: int, sm_count: int, n_max: int) -> tuple | None:
    """The smallest launch (n_frames, has_prev) in which some CTA walks items with different slot counts."""
    for n in range(1, n_max + 1):
        for p in (False, True):
            if "mixed" in coverage(n_pixels, [(n, p)], sm_count):
                return n, p
    return None
