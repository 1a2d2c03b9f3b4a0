"""Device-resident submissions larger than the engine's max_batch (csrc/engine.cu psd_engine_submit_device).

Frames the fused pass can read in place (no resize, no edge or hash features, 16-byte aligned base and frame
stride) are scored with one launch however many there are; every other submission is still cut into max_batch
batches.  Either way the per-frame integers are the ones the same frames give when submitted max_batch at a time,
with and without a device halo frame, and psd_launch_count() shows which of the two paths ran."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F_HSV, F_BGRSUM, F_YHIST, F_EDGES = 1, 2, 4, 8
MAX_BATCH = 16


def _launches(lib, run):
    before = lib.psd_launch_count()
    run()
    return lib.psd_launch_count() - before


def _results(eng):
    yh = eng.read_yhist().tobytes() if eng.features & F_YHIST else b""
    return eng.read_sums().tobytes(), yh


# (width, height, frame stride): 640x360 is 16-byte aligned; 131x97 (38 121 bytes, a 3-pixel tail) packed tight is
# not, so it goes through the aligned copy in max_batch batches; at a 38 128-byte stride it is read in place.
CASES = [(640, 360, 640 * 360 * 3), (131, 97, 131 * 97 * 3), (131, 97, 38128)]


@pytest.mark.parametrize("halo", [False, True], ids=["no_halo", "device_halo"])
@pytest.mark.parametrize("w,h,stride", CASES, ids=["640x360", "131x97_copy", "131x97_in_place"])
def test_one_submission_equals_max_batch_submissions(w, h, stride, halo):
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import DeviceBuffer, Engine
    lib = _capi.load()
    n = 3 * MAX_BATCH + 5
    rng = np.random.default_rng(w * 7 + h + stride)
    frames = rng.integers(0, 256, size=(n + 1, h, w, 3), dtype=np.uint8)
    frames[n // 2:n // 2 + 3] = frames[n // 2 - 1]     # a few unchanged frames: zero SADs among the large ones
    buf = DeviceBuffer((n + 1) * stride)
    try:
        for i in range(n + 1):
            buf.upload(frames[i], offset=i * stride)
        halo_ptr, first = (buf.ptr, buf.ptr + stride) if halo else (None, buf.ptr)
        feats = F_HSV | F_BGRSUM | F_YHIST

        def run(submit_sizes):
            eng = Engine(w, h, feats, max_batch=MAX_BATCH)
            if halo_ptr is not None:
                eng.set_halo_device(halo_ptr)
            eng.sync()

            def submit():
                done = 0
                for k in submit_sizes:
                    eng.submit_device(first + done * stride, k, stride)
                    done += k
                eng.sync()
            launches = _launches(lib, submit)
            assert eng.frame_count == n
            out = _results(eng)
            eng.close()
            return out, launches

        want, batched_launches = run([MAX_BATCH] * 3 + [5])
        got, launches = run([n])
        assert got == want
        per_launch = 1 + ((w * h) % 16 != 0)   # the warp-specialised kernel, plus the tail kernel for P mod 16 pixels
        assert batched_launches == 4 * per_launch
        in_place = stride % 16 == 0
        assert launches == (per_launch if in_place else 4 * per_launch)
    finally:
        buf.close()


def test_edge_features_keep_max_batch_batches():
    """With F_EDGES the per-batch edge scratch is sized by max_batch: a large device submission launches exactly
    what the same frames submitted max_batch at a time launch, and gives the same integers."""
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import DeviceBuffer, Engine
    lib = _capi.load()
    w, h, n = 640, 360, 3 * MAX_BATCH + 5
    fb = w * h * 3
    frames = np.random.default_rng(5).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)
    buf = DeviceBuffer(n * fb)
    try:
        buf.upload(frames)
        got = []
        for sizes in ([MAX_BATCH] * 3 + [5], [n]):
            eng = Engine(w, h, F_EDGES, max_batch=MAX_BATCH)

            def submit():
                done = 0
                for k in sizes:
                    eng.submit_device(buf.ptr + done * fb, k, fb)
                    done += k
                eng.sync()
            launches = _launches(lib, submit)
            got.append((eng.read_sums().tobytes(), launches))
            eng.close()
        assert got[0] == got[1]
    finally:
        buf.close()


def test_1080p_one_launch_equals_max_batch_launches():
    """bench.py's flagship shape at a smaller frame count: one in-place launch of 2 x 256 + 5 resident 1080p frames
    against the same frames submitted 256 at a time."""
    from pyscenedetect_b200 import _capi
    from pyscenedetect_b200.engine import DeviceBuffer, Engine, synth_frames_device
    from pyscenedetect_b200.synth import ScenePlan
    lib = _capi.load()
    w, h, mb = 1920, 1080, 256
    n = 2 * mb + 5
    fb = w * h * 3
    buf = DeviceBuffer(n * fb)
    try:
        synth_frames_device(buf.ptr, ScenePlan(n, seed=4, min_len=3, max_len=40).params, w, h)
        out = []
        for sizes in ([mb, mb, 5], [n]):
            eng = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, max_batch=mb)

            def submit():
                done = 0
                for k in sizes:
                    eng.submit_device(buf.ptr + done * fb, k, fb)
                    done += k
                eng.sync()
            launches = _launches(lib, submit)
            out.append((_results(eng), launches, eng.timing_ms()[2]))
            eng.close()
        assert out[1][0] == out[0][0]
        assert (out[0][1], out[0][2]) == (3, 3)
        assert (out[1][1], out[1][2]) == (1, 1)   # one score launch, and the engine's timing counts one
    finally:
        buf.close()
