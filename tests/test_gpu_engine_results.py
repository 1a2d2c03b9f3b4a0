"""An engine's per-frame result arrays across growth (csrc/engine.cu: FrameRows, ensure_capacity).

The result arrays start at 4 096 rows and double when a submission needs more; the rows already scored are copied
into the new array.  One engine with three edge slots (k = 19 uses the separable dilation) and two hash slots
((17, 1) needs 5 words a frame) scores a halo and 9 000 frames in host and device submissions of 1 000, so its arrays
grow at 4 096 and 8 192 rows with results in place.  Every slot's results must equal, byte for byte, those of an
engine with one slot of each kind that scored the same frames, and the rows scored before each growth must read back
unchanged after it.  Then reset() and a second, shorter video without a halo."""

import pytest

pytestmark = pytest.mark.gpu

W, H = 64, 36
CALL = 1000
WEIGHTS = (1.0, 0.5, 1.0, 0.25)
EDGE_KS = (3, 5, 19)
HASH_GEOS = ((8, 2), (17, 1))


def _video(n, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    return render_frames(ScenePlan(n, seed=seed, min_len=10, max_len=400).params, W, H)


def _engines():
    """The engine under test, and one-slot engines: refs[i] has edge slot EDGE_KS[i] and hash geometry
    HASH_GEOS[min(i, 1)]."""
    from pyscenedetect_b200.engine import F_BGRSUM, F_EDGES, F_HASH, F_HSV, F_YHIST, Engine
    feats = F_HSV | F_EDGES | F_BGRSUM | F_YHIST | F_HASH

    def make(k, geo):
        return Engine(W, H, feats, edge_kernel_size=k, hash_size=geo[0], hash_lowpass=geo[1])

    eng = make(EDGE_KS[0], HASH_GEOS[0])
    assert [eng.add_edge_kernel_size(k) for k in EDGE_KS[1:]] == [1, 2]
    assert eng.add_hash_geometry(*HASH_GEOS[1]) == 1
    refs = [make(k, HASH_GEOS[min(i, 1)]) for i, k in enumerate(EDGE_KS)]
    return eng, refs


def _feed(engines, frames, buf, halo):
    """Submit `frames` to every engine in calls of CALL frames, host and device alternately; after each call, the
    engine under test's raw results (halo row first) for the checks across growth."""
    stride = W * H * 3
    buf.upload(frames)
    for e in engines:
        e.reset()
        if halo is not None:
            e.set_halo(halo)
    snapshots = []
    for c, first in enumerate(range(0, len(frames), CALL)):
        n = min(CALL, len(frames) - first)
        for e in engines:
            if c % 2:
                e.submit_device(buf.ptr + first * stride, n, stride)
            else:
                e.submit(frames[first:first + n])
        snapshots.append(_raw(engines[0], -1 if halo is not None else 0))
    return snapshots


def _raw(eng, start):
    """The integer results of stream frames start.. (start = -1: from the halo frame's row)."""
    out = {"sums": eng.read_sums(start), "yhist": eng.read_yhist(start)}
    for s in range(len(HASH_GEOS)):
        out[f"hash{s}"] = eng.read_hash(start, hash_slot=s)
    return out


def _check(eng, refs, n, halo):
    start = -1 if halo else 0
    a = refs[0]
    assert eng.frame_count == n and all(r.frame_count == n for r in refs)
    assert eng.read_sums(start).tobytes() == a.read_sums(start).tobytes()
    assert eng.read_yhist(start).tobytes() == a.read_yhist(start).tobytes()
    for s in range(len(HASH_GEOS)):
        assert eng.read_hash(start, hash_slot=s).tobytes() == refs[s].read_hash(start).tobytes(), s
    for first in (0, n // 2 + 321):   # 4 821 of 9 000 frames: past the first growth
        for s, r in enumerate(refs):
            got, want = eng.scan_content(WEIGHTS, first, edge_slot=s), r.scan_content(WEIGHTS, first)
            assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), (first, s)
        for s in range(len(HASH_GEOS)):
            got, want = eng.scan_hash_dist(first, hash_slot=s), refs[s].scan_hash_dist(first)
            assert got.tobytes() == want.tobytes(), (first, s)
        assert eng.scan_hist_correl(256, first).tobytes() == a.scan_hist_correl(256, first).tobytes(), first
    # the video has cuts: none of the compared integers is trivially zero
    sums = eng.read_sums()
    for key in ("sad_hue", "sad_sat", "sad_lum", "sad_edges"):
        assert sums[key].any(), key
    for s in range(1, len(EDGE_KS)):
        _, comps = eng.scan_content(WEIGHTS, 0, edge_slot=s)
        assert comps[:, 3].any(), s


def _check_rows_kept(snapshots, final):
    """The rows each snapshot held are the first rows of the final arrays: growth kept them in place."""
    for snap in snapshots:
        for key, rows in snap.items():
            assert final[key][:len(rows)].tobytes() == rows.tobytes(), key


def test_results_survive_growth_and_match_one_slot_engines():
    from pyscenedetect_b200.engine import DeviceBuffer
    eng, refs = _engines()
    engines = [eng] + refs
    n1, n2 = 9000, 1500
    frames = _video(n1 + 1, seed=11)
    buf = DeviceBuffer(n1 * W * H * 3)
    try:
        snapshots = _feed(engines, frames[1:], buf, halo=frames[0])
        _check(eng, refs, n1, halo=True)
        # before the growth at 4 096 rows (4 000 frames + the halo) and before the one at 8 192 (8 000 frames)
        _check_rows_kept([snapshots[3], snapshots[7]], _raw(eng, -1))

        second = _video(n2, seed=12)
        snapshots = _feed(engines, second, buf, halo=None)
        _check(eng, refs, n2, halo=False)
        _check_rows_kept(snapshots, _raw(eng, 0))
    finally:
        buf.close()
        for e in engines:
            e.close()
