"""Frames from any DLPack exporter (torch, CuPy, JAX, DALI): shape, dtype and strides read from the exporter's
legacy "dltensor" capsule and turned into a `psd_frame_layout` (include/psd_b200.h).  No array library is imported:
the protocol is all this needs."""

from __future__ import annotations

import ctypes as C

import numpy as np

KDL_CPU = 1
KDL_CUDA = 2
_KDL_UINT = 1


class _DLDevice(C.Structure):
    _fields_ = [("device_type", C.c_int32), ("device_id", C.c_int32)]


class _DLDataType(C.Structure):
    _fields_ = [("code", C.c_uint8), ("bits", C.c_uint8), ("lanes", C.c_uint16)]


class _DLTensor(C.Structure):
    _fields_ = [
        ("data", C.c_void_p),
        ("device", _DLDevice),
        ("ndim", C.c_int32),
        ("dtype", _DLDataType),
        ("shape", C.POINTER(C.c_int64)),
        ("strides", C.POINTER(C.c_int64)),  # in elements; NULL = compact row-major
        ("byte_offset", C.c_uint64),
    ]


_capsule_pointer = C.pythonapi.PyCapsule_GetPointer
_capsule_pointer.restype = C.c_void_p
_capsule_pointer.argtypes = [C.py_object, C.c_char_p]


def is_dlpack(obj) -> bool:
    """An array that is not numpy and exports DLPack: the device input of Engine.submit and the detectors."""
    return not isinstance(obj, np.ndarray) and hasattr(obj, "__dlpack__")


def on_cuda(obj) -> bool:
    """`obj.__dlpack_device__()` names a CUDA device."""
    dev = getattr(obj, "__dlpack_device__", None)
    return dev is not None and int(dev()[0]) == KDL_CUDA


class FrameView:
    """n frames of height x width imported through DLPack.  `base` addresses channel B of pixel (0,0) of frame 0
    and `layout` = (frame, row, pixel, channel) byte strides, as psd_frame_layout takes them.  `capsule` keeps the
    exporter's memory alive: hold it until the work that reads the frames has finished."""

    __slots__ = ("capsule", "ndim", "n", "height", "width", "base", "layout")

    def __init__(self, capsule, ndim, n, height, width, base, layout):
        self.capsule, self.ndim, self.n, self.height, self.width = capsule, ndim, n, height, width
        self.base, self.layout = base, layout


def _export(obj, stream, device):
    dev_type, dev_id = (int(x) for x in obj.__dlpack_device__())
    if device is not None and (dev_type, dev_id) != (KDL_CUDA, int(device)):
        raise ValueError(f"frames must be CUDA memory of device {device}; they are DLPack device "
                         f"(type {dev_type}, id {dev_id})")
    # on CUDA, `stream` is the consumer's stream: the exporter makes it wait for the work that produced the frames
    # (-1: no ordering, for reading the metadata only)
    try:
        capsule = obj.__dlpack__(stream=-1 if stream is None else stream) if dev_type == KDL_CUDA else obj.__dlpack__()
    except BufferError as err:
        # torch exports a CUDA tensor only while its device is torch's current device (torch.cuda.set_device)
        raise ValueError(f"the exporter refused to export frames on DLPack device (type {dev_type}, id {dev_id}): "
                         f"{err}; make that device the exporter's current device first") from err
    return capsule, _DLTensor.from_address(_capsule_pointer(capsule, b"dltensor"))


def frame_format(obj, device=None) -> tuple[tuple, bool]:
    """(shape, whether the elements are uint8) of a DLPack array, without ordering against its producer."""
    _capsule, t = _export(obj, None, device)
    shape = tuple(t.shape[i] for i in range(t.ndim))
    return shape, (t.dtype.code, t.dtype.bits, t.dtype.lanes) == (_KDL_UINT, 8, 1)


def import_frames(obj, stream=None, device=None, channel_order: str = "bgr") -> FrameView:
    """(N,H,W,3) or (H,W,3) uint8 frames of a DLPack exporter -> FrameView.  `device`: the CUDA ordinal the frames
    must be on (None: any device, CPU included).  `stream`: the cudaStream_t (int) that will read them.
    `channel_order` "rgb": the last axis is R, G, B.  ValueError for anything else."""
    if channel_order not in ("bgr", "rgb"):
        raise ValueError(f"channel_order must be 'bgr' or 'rgb', not {channel_order!r}")
    capsule, t = _export(obj, stream, device)
    if (t.dtype.code, t.dtype.bits, t.dtype.lanes) != (_KDL_UINT, 8, 1):
        raise ValueError("frames must be uint8 (8-bit unsigned, one lane)")
    ndim = t.ndim
    shape = [t.shape[i] for i in range(ndim)]
    if ndim not in (3, 4) or shape[-1] != 3:
        raise ValueError(f"frames must have shape (N, H, W, 3) or (H, W, 3), not {tuple(shape)}")
    if t.strides:
        strides = [t.strides[i] for i in range(ndim)]
    else:
        strides, s = [], 1
        for d in reversed(shape):
            strides.insert(0, s)
            s *= d
    if ndim == 3:  # one frame: its stride only has to say how far apart frames would be
        shape, strides = [1] + shape, [shape[0] * strides[0]] + strides
    n, h, w, _ = shape
    fs, rs, ps, cs = strides
    base = (t.data or 0) + t.byte_offset
    if channel_order == "rgb":
        base, cs = base + 2 * cs, -cs
    return FrameView(capsule, ndim, n, h, w, base, (fs, rs, ps, cs))
