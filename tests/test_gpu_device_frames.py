"""Frames already on the GPU, in any layout (include/psd_b200.h psd_frame_layout): psd_gather_bgr byte for byte
against its numpy twin, Engine.submit of each layout against the same frames submitted as packed host BGR, and
SceneManager / strict process_frame over CUDA tensors against the same frames in numpy, with the producer's stream
ordering and the errors a device submission raises."""

import ctypes as C
import io

import numpy as np
import pytest
import torch

from tests.layout_twin import gather_twin

pytestmark = pytest.mark.gpu

F_HSV, F_BGRSUM, F_YHIST, F_EDGES, F_HASH = 1, 2, 4, 8, 16


def _synth(n, w, h, seed):
    from pyscenedetect_b200.synth import ScenePlan, render_frames
    return render_frames(ScenePlan(n, seed=seed, min_len=4, max_len=15).params, w, h)


def _gather_layouts(w, h, n):
    """name -> (view of one uint8 CUDA buffer, channel_order); every view is n frames of w x h."""
    rng = np.random.default_rng(w * 31 + h)
    fb = w * h * 3
    buf = torch.from_numpy(rng.integers(0, 256, size=4 * n * fb + 4 * (w + 8) * 3 * (h + 4) * n + 64,
                                        dtype=np.uint8)).cuda()
    packed = buf[:n * fb].view(n, h, w, 3)
    planar = buf[:n * fb].view(n, 3, h, w).permute(0, 2, 3, 1)
    wide = buf[:n * (h + 2) * (w + 5) * 3].view(n, h + 2, w + 5, 3)
    rs, fs = (w + 8) * 3 + 4, ((w + 8) * 3 + 4) * (h + 3) + 16
    return {
        "packed_bgr": (packed, "bgr"),
        "packed_rgb": (packed, "rgb"),
        "nchw_bgr": (planar, "bgr"),
        "nchw_rgb": (planar, "rgb"),
        "crop_odd_x": (wide[:, 1:1 + h, 3:3 + w], "bgr"),
        "crop_odd_x_rgb": (wide[:, 2:2 + h, 1:1 + w], "rgb"),
        "unaligned_base": (torch.as_strided(buf, (n, h, w, 3), (fb, w * 3, 3, 1), 1), "bgr"),
        "padded_strides": (torch.as_strided(buf, (n, h, w, 3), (fs, rs, 3, 1), 4), "rgb"),
        "padded_strides_bgr": (torch.as_strided(buf, (n, h, w, 3), (fs, rs, 3, 1), 8), "bgr"),
        "zero_frame_stride": (packed[1:2].expand(n, h, w, 3), "bgr"),
    }, buf


@pytest.mark.parametrize("w,h", [(1920, 1080), (131, 37), (1, 17)], ids=["1080p", "131x37", "1x17"])
def test_gather_bgr_equals_numpy_twin(w, h):
    from pyscenedetect_b200 import _dlpack
    from pyscenedetect_b200.engine import gather_bgr
    n = 3
    layouts, buf = _gather_layouts(w, h, n)
    host = buf.cpu().numpy()
    for name, (view, order) in layouts.items():
        dst = torch.full((n, h, w, 3), 7, dtype=torch.uint8, device="cuda")
        gather_bgr(view, dst.data_ptr(), w * h * 3, channel_order=order)
        torch.cuda.synchronize()
        v = _dlpack.import_frames(view, channel_order=order)
        want = gather_twin(host, v.base - buf.data_ptr(), v.layout, n, w, h)
        assert np.array_equal(dst.cpu().numpy(), want), name


def _device_variants(frames: np.ndarray) -> dict:
    """name -> (CUDA view of `frames`' pixels in another layout, channel_order)."""
    n, h, w, _ = frames.shape
    rgb = np.ascontiguousarray(frames[..., ::-1])
    big = np.zeros((n, h + 3, w + 5, 3), dtype=np.uint8)
    big[:, 1:1 + h, 3:3 + w] = frames
    return {
        "packed_bgr": (torch.from_numpy(frames).cuda(), "bgr"),
        "packed_rgb": (torch.from_numpy(rgb).cuda(), "rgb"),
        "nchw_bgr": (torch.from_numpy(np.ascontiguousarray(frames.transpose(0, 3, 1, 2))).cuda().permute(0, 2, 3, 1),
                     "bgr"),
        "nchw_rgb": (torch.from_numpy(np.ascontiguousarray(rgb.transpose(0, 3, 1, 2))).cuda().permute(0, 2, 3, 1),
                     "rgb"),
        "crop_odd_x": (torch.from_numpy(big).cuda()[:, 1:1 + h, 3:3 + w], "bgr"),
    }


def _engine_results(eng, n, edge_slots, hash_slots):
    from pyscenedetect_b200 import _capi
    out = [eng.read_sums().tobytes()]
    if eng.features & F_YHIST:
        out.append(eng.read_yhist().tobytes())
    for s in hash_slots:
        out.append(eng.read_hash(hash_slot=s).tobytes())
    eng.sync()
    for s in edge_slots[1:]:
        sads = np.zeros(n, dtype=np.uint64)
        _capi.check(_capi.load().psd_memcpy_d2h(eng.device, sads.ctypes.data, eng.device_edge_sads(s), n * 8))
        out.append(sads.tobytes())
    return out


def _run_engine(frames_for_submit, w, h, size, feats, max_batch, chunks):
    from pyscenedetect_b200.engine import Engine
    eng = Engine(w, h, feats, width=size[0], height=size[1], max_batch=max_batch)
    edge_slots = [0] + ([eng.add_edge_kernel_size(k) for k in (3, 7)] if feats & F_EDGES else [])
    hash_slots = [0, eng.add_hash_geometry(4, 2)] if feats & F_HASH else []
    done = 0
    for k, submit in zip(chunks, frames_for_submit):
        submit(eng, done, k)
        done += k
    n = eng.frame_count
    out = _engine_results(eng, n, edge_slots, hash_slots)
    eng.close()
    return out


FEATURES = {"hsv": F_HSV, "bgrsum": F_BGRSUM, "yhist": F_YHIST, "edges": F_EDGES, "hash": F_HASH,
            "all": F_HSV | F_BGRSUM | F_YHIST | F_EDGES | F_HASH}


@pytest.mark.parametrize("feat", list(FEATURES))
@pytest.mark.parametrize("geometry", ["full_res", "resized_1080p", "odd_crop_resized"])
def test_engine_submit_of_each_layout_equals_host_bgr(feat, geometry):
    feats = FEATURES[feat]
    if geometry == "full_res":
        w, h, size, n, mb = 320, 180, (320, 180), 21, 8
    elif geometry == "resized_1080p":
        w, h, size, n, mb = 1920, 1080, (256, 144), 11, 4
    else:
        w, h, size, n, mb = 333, 187, (111, 62), 13, 4
    frames = _synth(n, w, h, seed=len(feat) + w)
    chunks = [mb + 3, 1, n - mb - 4]   # one submission larger than max_batch, a single frame, the rest
    host = [lambda e, d, k: e.submit(frames[d:d + k])] * 3
    want = _run_engine(host, w, h, size, feats, mb, chunks)
    for name, (view, order) in _device_variants(frames).items():
        dev = [lambda e, d, k, v=view, o=order: e.submit(v[d:d + k], channel_order=o)] * 3
        assert _run_engine(dev, w, h, size, feats, mb, chunks) == want, name
        # host and device batches alternating in one engine: the carried frame crosses both ways
        mixed = [dev[0], host[0], dev[0]]
        assert _run_engine(mixed, w, h, size, feats, mb, chunks) == want, name + " mixed"
        one = [lambda e, d, k, v=view, o=order: [e.submit(v[i], channel_order=o) for i in range(d, d + k)]] * 3
        assert _run_engine(one, w, h, size, feats, mb, chunks) == want, name + " frame by frame"


class _ReadOnlyStream:
    """A device stream with `read()` only (no read_batch)."""

    def __init__(self, frames, fps=30.0, channel_order="bgr"):
        from pyscenedetect_b200.video import ArrayVideoStream
        self._inner = ArrayVideoStream(frames, fps, channel_order=channel_order)

    frame_rate = property(lambda self: self._inner.frame_rate)
    frame_size = property(lambda self: self._inner.frame_size)
    frame_number = property(lambda self: self._inner.frame_number)
    position = property(lambda self: self._inner.position)
    base_timecode = property(lambda self: self._inner.base_timecode)
    channel_order = property(lambda self: self._inner.channel_order)

    def read(self, decode=True):
        return self._inner.read(decode)


def _detectors(which):
    from pyscenedetect_b200.detectors import (AdaptiveDetector, ContentDetector, HashDetector, HistogramDetector,
                                              ThresholdDetector)
    make = {"content": lambda: ContentDetector(threshold=20.0, min_scene_len=3),
            "content_edges": lambda: ContentDetector(threshold=20.0, min_scene_len=3,
                                                     weights=ContentDetector.Components(1.0, 1.0, 1.0, 1.0)),
            "adaptive": lambda: AdaptiveDetector(min_scene_len=3),
            "threshold": lambda: ThresholdDetector(threshold=40, min_scene_len=3),
            "histogram": lambda: HistogramDetector(min_scene_len=3),
            "hash": lambda: HashDetector(min_scene_len=3)}
    names = list(make)[:1] + list(make)[2:] + ["content_edges"] if which == "mix" else [which]
    return [make[k]() for k in names]


def _detect(video, which, stats, callback, config):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager() if stats else None, batch_size=config.get("batch", 8))
    for d in _detectors(which):
        sm.add_detector(d)
    if "auto_downscale" in config:
        sm.auto_downscale = config["auto_downscale"]
    if "downscale" in config:
        sm.auto_downscale = False
        sm.downscale = config["downscale"]
    if "crop" in config:
        sm.crop = config["crop"]
    calls = []
    cb = (lambda frame, tc: calls.append((tc.frame_num, np.asarray(frame).tobytes()))) if callback else None
    n = sm.detect_scenes(video, duration=config.get("duration"), end_time=config.get("end_time"),
                         frame_skip=config.get("frame_skip", 0), callback=cb)
    csv = None
    if stats:
        f = io.StringIO()
        sm.stats_manager.save_to_csv(f)
        csv = f.getvalue()
    return (n, [c.frame_num for c in sm.get_cut_list()],
            [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list()], csv, calls, video.position.frame_num)


CONFIGS = {
    "default": {},
    "no_auto_downscale": {"auto_downscale": False},
    "downscale_3": {"downscale": 3},
    "crop": {"crop": (13, 9, 300, 170)},
    "frame_skip_2": {"frame_skip": 2},
    "duration": {"duration": 37},
    "end_time": {"end_time": 41},
    "batch_64": {"batch": 64},
}


def _scene_frames():
    return _synth(90, 320, 180, seed=11)


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("which", ["content", "adaptive", "threshold", "histogram", "hash", "mix"])
def test_scene_manager_over_cuda_frames_equals_numpy(which, config):
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = _scene_frames()
    cfg = CONFIGS[config]
    stats = "frame_skip" not in cfg
    want = _detect(ArrayVideoStream(frames), which, stats, True, cfg)
    got = _detect(ArrayVideoStream(torch.from_numpy(frames).cuda()), which, stats, True, cfg)
    assert got == want


@pytest.mark.parametrize("layout", ["rgb", "nchw", "nchw_rgb", "read_only", "read_only_rgb"])
@pytest.mark.parametrize("config", ["default", "crop", "frame_skip_2", "end_time"])
def test_scene_manager_layouts_and_read_only_streams(layout, config):
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = _scene_frames()
    cfg = CONFIGS[config]
    stats = "frame_skip" not in cfg
    want = _detect(ArrayVideoStream(frames), "mix", stats, True, cfg)
    order = "rgb" if layout.endswith("rgb") else "bgr"
    src = np.ascontiguousarray(frames[..., ::-1]) if order == "rgb" else frames
    if layout.startswith("nchw"):
        t = torch.from_numpy(np.ascontiguousarray(src.transpose(0, 3, 1, 2))).cuda().permute(0, 2, 3, 1)
    else:
        t = torch.from_numpy(src).cuda()
    stream = (_ReadOnlyStream if layout.startswith("read_only") else ArrayVideoStream)(t, channel_order=order)
    assert _detect(stream, "mix", stats, True, cfg) == want


def test_numpy_rgb_stream_equals_bgr():
    from pyscenedetect_b200.video import ArrayVideoStream
    frames = _scene_frames()
    want = _detect(ArrayVideoStream(frames), "mix", True, True, {})
    got = _detect(ArrayVideoStream(np.ascontiguousarray(frames[..., ::-1]), channel_order="rgb"), "mix", True, True, {})
    assert got == want


@pytest.mark.parametrize("which", ["content_edges", "adaptive", "threshold", "histogram", "hash"])
def test_strict_process_frame_with_cuda_frames(which):
    from pyscenedetect_b200 import FrameTimecode, StatsManager
    frames = _synth(40, 160, 90, seed=3)
    dev = torch.from_numpy(frames).cuda()
    results = []
    for src in (frames, dev):
        det = _detectors(which)[0]
        det.stats_manager = StatsManager()
        cuts = []
        for i in range(len(frames)):
            cuts += [c.frame_num for c in det.process_frame(FrameTimecode(i, 30.0), src[i])]
        f = io.StringIO()
        det.stats_manager.save_to_csv(f)
        results.append((cuts, f.getvalue()))
    assert results[1] == results[0]


@pytest.mark.parametrize("where", ["current_stream", "side_stream"])
def test_frames_written_by_a_queued_op_are_read_after_it(where):
    from pyscenedetect_b200.engine import Engine
    w, h, n = 640, 360, 24
    frames = _synth(n, w, h, seed=9)
    want_eng = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST)
    want_eng.submit(frames)
    want = (want_eng.read_sums().tobytes(), want_eng.read_yhist().tobytes())
    want_eng.close()
    src = torch.from_numpy(frames).cuda()
    layouts = {"packed": lambda d: d, "nchw": lambda d: d.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)}
    for name, shape in layouts.items():
        for size in [(w, h), (256, 144)]:
            eng = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, width=size[0], height=size[1])
            torch.cuda.synchronize()
            stream = torch.cuda.Stream() if where == "side_stream" else torch.cuda.current_stream()
            with torch.cuda.stream(stream):
                dst = shape(torch.zeros_like(src))
                torch.cuda._sleep(200_000_000)   # the copy below starts long after submit() returns
                dst.copy_(src)
                eng.submit(dst)
                got = (eng.read_sums().tobytes(), eng.read_yhist().tobytes())
            eng.close()
            if size == (w, h):
                assert got == want, (name, where)
            else:
                ref = Engine(w, h, F_HSV | F_BGRSUM | F_YHIST, width=size[0], height=size[1])
                ref.submit(frames)
                assert got == (ref.read_sums().tobytes(), ref.read_yhist().tobytes()), (name, where, size)
                ref.close()


def test_device_submission_errors():
    from pyscenedetect_b200.engine import Engine
    eng = Engine(64, 36, F_HSV)
    ok = torch.zeros(2, 36, 64, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="uint8"):
        eng.submit(ok.float())
    with pytest.raises(ValueError, match="shape"):
        eng.submit(torch.zeros(2, 36, 64, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="does not match"):
        eng.submit(torch.zeros(2, 36, 63, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="CUDA memory"):
        eng.submit(ok.cpu())  # a CPU tensor as device input
    eng.submit(ok)
    assert eng.frame_count == 2
    eng.submit(torch.empty(0, 36, 64, 3, dtype=torch.uint8, device="cuda"))   # an empty batch: nothing to score
    assert eng.frame_count == 2
    # the raw entry refuses host memory
    from pyscenedetect_b200 import _capi
    host = np.zeros((2, 36, 64, 3), dtype=np.uint8)
    layout = _capi.PsdFrameLayout(36 * 64 * 3, 64 * 3, 3, 1)
    assert _capi.load().psd_engine_submit_device_layout(eng._h, host.ctypes.data, 2, C.byref(layout)) == \
        _capi.PSD_ERR_INVALID
    eng.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_frames_on_another_device_are_refused():
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.engine import Engine
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    t = torch.zeros(4, 36, 64, 3, dtype=torch.uint8, device="cuda:1")
    with pytest.raises(ValueError, match="device 0"):
        Engine(64, 36, F_HSV, device=0).submit(t)
    # torch exports a tensor only while its device is torch's current device: the refusal is a ValueError too
    with pytest.raises(ValueError, match="current device"):
        ArrayVideoStream(t)
    with torch.cuda.device(1):
        stream = ArrayVideoStream(t)
    sm = SceneManager(device=0)
    sm.add_detector(ContentDetector())
    with pytest.raises(ValueError, match="device 0"):
        sm.detect_scenes(stream)
    # frames on the engine's device are scored there once it is torch's current device
    frames = _synth(6, 64, 36, seed=1)
    ref = Engine(64, 36, F_HSV | F_BGRSUM, device=0)
    ref.submit(frames)
    with torch.cuda.device(1):
        eng = Engine(64, 36, F_HSV | F_BGRSUM, device=1)
        eng.submit(torch.from_numpy(frames).to("cuda:1"))
        assert eng.read_sums().tobytes() == ref.read_sums().tobytes()
        eng.close()
    ref.close()
