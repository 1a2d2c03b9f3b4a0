"""DLPack import (pyscenedetect_b200/_dlpack.py) on CPU torch tensors: the psd_frame_layout it builds names the
tensor's own bytes for contiguous, NCHW-permuted, cropped, stepped and expanded views, in both channel orders; the
inputs a device submission refuses; and the crop / frame-skip views FrameBatches reads CUDA streams through."""

import ctypes as C

import numpy as np
import pytest
import torch

from pyscenedetect_b200 import _dlpack
from pyscenedetect_b200.scene_manager import FrameBatches
from pyscenedetect_b200.video import ArrayVideoStream
from tests.layout_twin import gather_twin

N, H, W = 5, 7, 11


def _storage_bytes(t: torch.Tensor) -> tuple[np.ndarray, int]:
    st = t.untyped_storage()
    arr = np.ctypeslib.as_array((C.c_uint8 * st.nbytes()).from_address(st.data_ptr()))
    return arr, st.data_ptr()


def _bgr_frames(seed=0) -> torch.Tensor:
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, size=(N, H, W, 3), dtype=np.uint8))


def _views():
    bgr = _bgr_frames()
    nchw = bgr.permute(0, 3, 1, 2).contiguous()
    big = torch.from_numpy(np.random.default_rng(1).integers(0, 256, size=(2 * N, H + 3, W + 4, 3), dtype=np.uint8))
    return {
        "contiguous": bgr,
        "nchw_permuted": nchw.permute(0, 2, 3, 1),
        "cropped": big[:N, 1:1 + H, 3:3 + W],
        "stepped": big[::2, 2:2 + H, 1:1 + W],
        "expanded": bgr[2:3].expand(N, H, W, 3),
        "one_frame": bgr[3],
    }


@pytest.mark.parametrize("order", ["bgr", "rgb"])
@pytest.mark.parametrize("name", list(_views()))
def test_layout_reproduces_the_tensor(name, order):
    t = _views()[name]
    v = _dlpack.import_frames(t, channel_order=order)
    batch = t if t.dim() == 4 else t[None]
    assert (v.n, v.height, v.width) == tuple(batch.shape[:3])
    assert v.ndim == t.dim()
    buf, origin = _storage_bytes(t)
    got = gather_twin(buf, v.base - origin, v.layout, v.n, v.width, v.height)
    want = batch.numpy()
    np.testing.assert_array_equal(got, want if order == "bgr" else want[..., ::-1])


def test_layout_strides():
    bgr = _bgr_frames()
    assert _dlpack.import_frames(bgr).layout == (H * W * 3, W * 3, 3, 1)
    rgb = _dlpack.import_frames(bgr, channel_order="rgb")
    assert rgb.layout == (H * W * 3, W * 3, 3, -1) and rgb.base == bgr.data_ptr() + 2
    nchw = bgr.permute(0, 3, 1, 2).contiguous()
    v = _dlpack.import_frames(nchw.permute(0, 2, 3, 1), channel_order="rgb")
    assert v.layout == (3 * H * W, W, 1, -H * W) and v.base == nchw.data_ptr() + 2 * H * W
    assert _dlpack.import_frames(bgr[0:1].expand(N, H, W, 3)).layout[0] == 0


def test_rejects_what_a_device_submission_cannot_take():
    bgr = _bgr_frames()
    with pytest.raises(ValueError, match="uint8"):
        _dlpack.import_frames(bgr.float())
    with pytest.raises(ValueError, match="shape"):
        _dlpack.import_frames(torch.zeros(N, H, W, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match="shape"):
        _dlpack.import_frames(torch.zeros(H, W, dtype=torch.uint8))
    with pytest.raises(ValueError, match="CUDA memory of device 0"):
        _dlpack.import_frames(bgr, device=0)
    with pytest.raises(ValueError, match="channel_order"):
        _dlpack.import_frames(bgr, channel_order="bgra")
    assert _dlpack.is_dlpack(bgr) and not _dlpack.is_dlpack(bgr.numpy())
    assert not _dlpack.on_cuda(bgr)


def test_engine_and_stream_refuse_cpu_tensors_as_device_input():
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.compat import FrameTimecode
    with pytest.raises(ValueError, match="CUDA memory"):
        ContentDetector().process_frame(FrameTimecode(0, 30.0), _bgr_frames()[0])
    with pytest.raises(ValueError):
        ArrayVideoStream(_bgr_frames().float())


class _RefusingExporter:
    """A CUDA array whose exporter refuses to export, as torch does for a tensor off its current device."""

    def __dlpack_device__(self):
        return (_dlpack.KDL_CUDA, 1)

    def __dlpack__(self, stream=None):
        raise BufferError("Can't export tensors on a different CUDA device index")


def test_an_exporter_refusal_is_a_value_error():
    with pytest.raises(ValueError, match="current device"):
        _dlpack.frame_format(_RefusingExporter())
    with pytest.raises(ValueError, match="current device"):
        _dlpack.import_frames(_RefusingExporter(), stream=7, device=1)
    with pytest.raises(ValueError, match="current device"):
        ArrayVideoStream(_RefusingExporter())
    with pytest.raises(ValueError, match="device 0"):   # another device than the engine's: refused before export
        _dlpack.import_frames(_RefusingExporter(), device=0)


def test_stream_refuses_host_dlpack_frames_and_reads_sizes_from_the_view():
    with pytest.raises(ValueError, match="CUDA memory"):
        ArrayVideoStream(_bgr_frames())
    s = _CudaLikeStream(_bgr_frames().numpy(), repeat=2)
    assert s.frame_size == (W, H) and s.duration.frame_num == 2 * N


class _CudaLikeStream(ArrayVideoStream):
    """A numpy stream that says its frames are on the GPU: FrameBatches then reads it through views."""

    def __dlpack_device__(self):
        return (_dlpack.KDL_CUDA, 0)


def _drain(video, box, size, batch, cropped, skip, end):
    fb = FrameBatches(video, box, size, batch, cropped=cropped, frame_skip=skip, end_frame=end)
    tcs, frames = [], []
    while True:
        got = fb.next()
        if got is None:
            break
        tcs += [tc.frame_num for tc in got[0]]
        frames += [np.array(f) for f in got[1]]
        assert len(got[0]) <= batch
    fb.close()
    return tcs, frames, video.position.frame_num, video.frame_number


@pytest.mark.parametrize("batch", [1, 4, 64])
@pytest.mark.parametrize("end", [None, 1, 7, 8, 9, 23, 40])
@pytest.mark.parametrize("skip", [0, 1, 2, 5])
@pytest.mark.parametrize("cropped", [False, True])
def test_device_views_read_what_the_host_loop_reads(cropped, skip, end, batch, monkeypatch):
    """Positions, frames, the final position and the frames consumed of the view path equal the host path's."""
    from pyscenedetect_b200 import scene_manager

    class _NoPinned:  # the host loop's page-locked buffer, in pageable memory
        def __init__(self, nbytes):
            self.array = np.empty(nbytes, dtype=np.uint8)

        def close(self):
            pass

    monkeypatch.setattr(scene_manager, "PinnedBuffer", _NoPinned)
    frames = np.random.default_rng(skip).integers(0, 256, size=(23, 6, 9, 3), dtype=np.uint8)
    box = (2, 1, 7, 5) if cropped else (0, 0, 9, 6)
    size = (box[2] - box[0], box[3] - box[1])
    host = _drain(ArrayVideoStream(frames), box, size, batch, cropped, skip, end)
    dev = _drain(_CudaLikeStream(frames), box, size, batch, cropped, skip, end)
    assert dev[0] == host[0] and dev[2:] == host[2:]
    assert all(np.array_equal(a, b) for a, b in zip(dev[1], host[1])) and len(dev[1]) == len(host[1])
