"""Python handle on a `psd_engine` (include/psd_b200.h): the batched, device-resident
replacement for the per-frame cv2/numpy work inside the reference detectors."""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi, _dlpack
from ._capi import F_BGRSUM, F_EDGES, F_HASH, F_HSV, F_YHIST, SUMS_DTYPE, check, hash_words


class PinnedBuffer:
    """Page-locked host memory exposed as a numpy uint8 array (for zero-staging submits)."""

    def __init__(self, nbytes: int):
        lib = _capi.load()
        p = C.c_void_p()
        check(lib.psd_host_alloc(int(nbytes), C.byref(p)), "psd_host_alloc")
        self._p = p
        self.nbytes = int(nbytes)
        self.array = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(self.nbytes,))

    def close(self):
        if self._p is not None and self._p.value:
            _capi.load().psd_host_free(self._p)
            self._p = None
            self.array = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceBuffer:
    """Plain device allocation owned through the C-ABI (torch-free HBM residency)."""

    def __init__(self, nbytes: int, device: int = 0):
        lib = _capi.load()
        p = C.c_void_p()
        check(lib.psd_device_alloc(device, int(nbytes), C.byref(p)), "psd_device_alloc")
        self.ptr = p.value
        self.nbytes = int(nbytes)
        self.device = device

    def upload(self, arr: np.ndarray, offset: int = 0):
        arr = np.ascontiguousarray(arr)
        assert offset + arr.nbytes <= self.nbytes
        check(_capi.load().psd_memcpy_h2d(self.device, self.ptr + offset, arr.ctypes.data, arr.nbytes))

    def download(self, nbytes: int, offset: int = 0) -> np.ndarray:
        out = np.empty(nbytes, dtype=np.uint8)
        check(_capi.load().psd_memcpy_d2h(self.device, out.ctypes.data, self.ptr + offset, nbytes))
        return out

    def close(self):
        if self.ptr:
            _capi.load().psd_device_free(self.device, self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One streaming scorer.  Frames go in (host ndarray batches or device pointers); per-frame
    integer sums / histograms stay in HBM; `scan_*` run the trailing device scans that turn
    them into the detectors' float64 metrics."""

    def __init__(self, src_width: int, src_height: int, features: int, width: int | None = None,
                 height: int | None = None, device: int = 0, max_batch: int = 64,
                 edge_kernel_size: int = 0, hash_size: int = 8, hash_lowpass: int = 2):
        self._lib = _capi.load()
        cfg = _capi.PsdConfig()
        cfg.struct_size = C.sizeof(_capi.PsdConfig)
        cfg.device = device
        cfg.src_width, cfg.src_height = int(src_width), int(src_height)
        cfg.width = int(width if width is not None else src_width)
        cfg.height = int(height if height is not None else src_height)
        cfg.features = int(features)
        cfg.edge_kernel_size = int(edge_kernel_size)
        cfg.max_batch = int(max_batch)
        cfg.hash_size, cfg.hash_lowpass = int(hash_size), int(hash_lowpass)
        self.hash_size = int(hash_size)
        self._hash_sizes = [self.hash_size]  # per hash slot
        h = C.c_void_p()
        check(self._lib.psd_engine_create(C.byref(cfg), C.byref(h)), "psd_engine_create")
        self._h = h
        self.device = device
        self.src_width, self.src_height = cfg.src_width, cfg.src_height
        self.width, self.height = cfg.width, cfg.height
        self.features = int(features) | (F_HSV if features & F_EDGES else 0)
        self.max_batch = int(max_batch)
        self.n_pixels = self.width * self.height
        self.src_frame_bytes = self.src_width * self.src_height * 3
        self._held = []  # DLPack capsules of submitted device frames, released once the engine has synchronised

    def _synced(self):
        """The compute stream has finished everything queued so far: the device frames submitted can go."""
        self._held.clear()

    # -- lifetime --
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.psd_engine_destroy(self._h)
            self._h = None
            self._synced()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        check(self._lib.psd_engine_reset(self._h), "psd_engine_reset")
        self._synced()

    # -- input --
    def _check_frames(self, frames: np.ndarray) -> np.ndarray:
        if frames.dtype != np.uint8:
            raise ValueError("frames must be uint8 BGR24")
        if frames.ndim == 3:
            frames = frames[None]
        if frames.ndim != 4 or frames.shape[3] != 3:
            raise ValueError("frames must have shape (N, H, W, 3)")
        if frames.shape[1] != self.src_height or frames.shape[2] != self.src_width:
            raise ValueError(
                f"frame size {frames.shape[2]}x{frames.shape[1]} does not match engine "
                f"{self.src_width}x{self.src_height}")
        if frames.strides[3] != 1 or frames.strides[2] != 3:
            frames = np.ascontiguousarray(frames)
        return frames

    def set_halo(self, frame: np.ndarray):
        f = self._check_frames(frame)
        check(self._lib.psd_engine_set_halo_host(self._h, f.ctypes.data, f.strides[1]),
              "psd_engine_set_halo_host")

    def set_halo_device(self, dptr: int):
        check(self._lib.psd_engine_set_halo_device(self._h, dptr), "psd_engine_set_halo_device")

    def submit(self, frames, pinned: bool = False, channel_order: str = "bgr"):
        """Score a batch of frames (N,H,W,3) or one frame (H,W,3), uint8: a numpy array in host memory, or CUDA
        memory of this engine's device from any DLPack exporter (a torch tensor, say), of any strides (a crop, a
        frame step, `nchw.permute(0, 2, 3, 1)`).  `channel_order` "rgb": the last axis is R, G, B.

        Device frames are read on the engine's compute stream after the exporter's current stream has reached
        this call (the DLPack stream handshake), and must not be overwritten until the engine has synchronised
        (`sync()` or any read or host scan): the engine keeps a reference until then.  torch exports a CUDA tensor
        only while its device is torch's current device (`torch.cuda.set_device`); any refusal of the exporter
        raises ValueError, as do frames on another device than the engine's."""
        if _dlpack.is_dlpack(frames):
            v = _dlpack.import_frames(frames, stream=self.compute_stream, device=self.device,
                                      channel_order=channel_order)
            if (v.width, v.height) != (self.src_width, self.src_height):
                raise ValueError(f"frame size {v.width}x{v.height} does not match engine "
                                 f"{self.src_width}x{self.src_height}")
            layout = _capi.PsdFrameLayout(*v.layout)
            check(self._lib.psd_engine_submit_device_layout(self._h, v.base, v.n, C.byref(layout)),
                  "psd_engine_submit_device_layout")
            self._held.append(v.capsule)
            return
        if channel_order not in ("bgr", "rgb"):
            raise ValueError(f"channel_order must be 'bgr' or 'rgb', not {channel_order!r}")
        if channel_order == "rgb" and isinstance(frames, np.ndarray):
            frames = frames[..., ::-1]
        f = self._check_frames(frames)
        n = f.shape[0]
        fs = f.strides[0] if n > 1 else f.strides[1] * self.src_height
        check(self._lib.psd_engine_submit_host(self._h, f.ctypes.data, n, fs, f.strides[1],
                                               _capi.SUBMIT_PINNED if pinned else 0),
              "psd_engine_submit_host")

    def submit_layout(self, base: int, n_frames: int, layout: tuple):
        """Score n_frames BGR frames at device pointer `base` (channel B of pixel (0, 0) of the first), laid out as
        `layout` = (frame, row, pixel, channel) byte strides, of this engine's source size.  The memory is the
        caller's: it must stay unchanged until the engine has synchronised."""
        lay = _capi.PsdFrameLayout(*layout)
        check(self._lib.psd_engine_submit_device_layout(self._h, int(base), int(n_frames), C.byref(lay)),
              "psd_engine_submit_device_layout")

    def submit_device(self, dptr: int, n_frames: int, frame_stride: int | None = None):
        check(self._lib.psd_engine_submit_device(self._h, dptr, int(n_frames),
                                                 int(frame_stride or self.src_frame_bytes)),
              "psd_engine_submit_device")

    def sync(self):
        check(self._lib.psd_engine_sync(self._h), "psd_engine_sync")
        self._synced()

    @property
    def compute_stream(self) -> int:
        """cudaStream_t handle of the engine's compute stream."""
        return int(self._lib.psd_engine_compute_stream(self._h) or 0)

    @property
    def frame_count(self) -> int:
        return int(self._lib.psd_engine_frame_count(self._h))

    @property
    def edge_kernel_size(self) -> int:
        return int(self._lib.psd_engine_edge_kernel_size(self._h))

    # -- slots: more kernel sizes / hash geometries scored from the same pass (before the first frame) --
    def add_edge_kernel_size(self, kernel_size: int) -> int:
        """Edge slot of a ContentDetector(kernel_size=...) (0 = automatic) next to the configured one; the slot
        already holding that effective size if there is one.  RuntimeError once the engine holds frames."""
        slot = C.c_int32()
        check(self._lib.psd_engine_add_edge_kernel_size(self._h, int(kernel_size), C.byref(slot)),
              "psd_engine_add_edge_kernel_size")
        return slot.value

    def add_hash_geometry(self, size: int, lowpass: int) -> int:
        """Hash slot of a HashDetector(size=..., lowpass=...); the existing slot if that geometry is present."""
        slot = C.c_int32()
        check(self._lib.psd_engine_add_hash_geometry(self._h, int(size), int(lowpass), C.byref(slot)),
              "psd_engine_add_hash_geometry")
        if slot.value == len(self._hash_sizes):
            self._hash_sizes.append(int(size) or 8)
        return slot.value

    def edge_kernel_size_at(self, slot: int) -> int:
        return int(self._lib.psd_engine_edge_kernel_size_at(self._h, int(slot)))

    def hash_size_at(self, slot: int) -> int:
        return self._hash_sizes[slot]

    def device_edge_sads(self, edge_slot: int = 0) -> int | None:
        """Device array of an edge slot's sad_edges (stream frame i at index i); None for slot 0, whose SADs are
        the sums' sad_edges."""
        p = C.c_void_p()
        check(self._lib.psd_engine_device_edge_sads(self._h, int(edge_slot), C.byref(p)),
              "psd_engine_device_edge_sads")
        return p.value

    def view(self, edge_slot: int = 0, hash_slot: int = 0) -> "Engine | SlotView":
        """The results of the given slots: the engine itself for slots 0 / 0, else a `SlotView`."""
        return SlotView(self, edge_slot, hash_slot) if edge_slot or hash_slot else self

    # -- raw integer results --
    def read_sums(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self.frame_count - first if n is None else n
        out = np.zeros(n, dtype=SUMS_DTYPE)
        check(self._lib.psd_engine_read_sums(self._h, first, n, out.ctypes.data), "psd_engine_read_sums")
        self._synced()
        return out

    def read_yhist(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self.frame_count - first if n is None else n
        out = np.zeros((n, 256), dtype=np.uint32)
        check(self._lib.psd_engine_read_yhist(self._h, first, n, out.ctypes.data), "psd_engine_read_yhist")
        self._synced()
        return out

    def read_hash(self, first: int = 0, n: int | None = None, hash_slot: int = 0) -> np.ndarray:
        """-> (n, hash_words(size)) uint64: bit u*size+v of the row (word k // 64, bit k % 64) = DCT[u][v] > median
        (hash_detector.py:156); 4 words for size <= 16."""
        n = self.frame_count - first if n is None else n
        out = np.zeros((n, hash_words(self.hash_size_at(hash_slot))), dtype=np.uint64)
        check(self._lib.psd_engine_read_hash_at(self._h, int(hash_slot), first, n, out.ctypes.data),
              "psd_engine_read_hash")
        self._synced()
        return out

    def device_hash(self, hash_slot: int = 0) -> int | None:
        p = C.c_void_p()
        check(self._lib.psd_engine_device_hash_at(self._h, int(hash_slot), C.byref(p)))
        return p.value

    def device_results(self) -> tuple[int, int | None]:
        s, h = C.c_void_p(), C.c_void_p()
        check(self._lib.psd_engine_device_results(self._h, C.byref(s), C.byref(h)))
        return s.value, h.value

    # -- trailing device scans (host-array convenience forms) --
    def scan_content(self, weights, first: int = 0, n: int | None = None, edge_slot: int = 0):
        """-> (content_val[n], components[n,4]) as float64; bit-identical to
        content_detector.py:166-180 (the edge component of edge slot `edge_slot`)."""
        n = self.frame_count - first if n is None else n
        w = (C.c_double * 4)(*[float(x) for x in weights])
        wsum = float(sum(abs(x) for x in weights))  # same expression as content_detector.py:180
        val = np.zeros(n, dtype=np.float64)
        comps = np.zeros((n, 4), dtype=np.float64)
        check(self._lib.psd_engine_scan_content_host_at(self._h, int(edge_slot), first, n, w, wsum,
                                                        comps.ctypes.data, val.ctypes.data),
              "psd_engine_scan_content_host")
        if n:
            self._synced()
        return val, comps

    def scan_adaptive(self, scores: np.ndarray, window_width: int, min_content_val: float) -> np.ndarray:
        s = np.ascontiguousarray(scores, dtype=np.float64)
        out = np.zeros(s.shape[0], dtype=np.float64)
        check(self._lib.psd_engine_scan_adaptive_host(self._h, s.ctypes.data, s.shape[0],
                                                      int(window_width), float(min_content_val),
                                                      out.ctypes.data), "psd_engine_scan_adaptive_host")
        if out.shape[0]:
            self._synced()
        return out

    def scan_average(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self.frame_count - first if n is None else n
        out = np.zeros(n, dtype=np.float64)
        check(self._lib.psd_engine_scan_average_host(self._h, first, n, out.ctypes.data),
              "psd_engine_scan_average_host")
        if out.shape[0]:
            self._synced()
        return out

    def scan_hist_correl(self, bins: int, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self.frame_count - first if n is None else n
        out = np.zeros(n, dtype=np.float64)
        check(self._lib.psd_engine_scan_hist_correl_host(self._h, first, n, int(bins), out.ctypes.data),
              "psd_engine_scan_hist_correl_host")
        if out.shape[0]:
            self._synced()
        return out

    def scan_hash_dist(self, first: int = 0, n: int | None = None, hash_slot: int = 0) -> np.ndarray:
        """hash_dist of frames [first, first+n) against their predecessors; NaN where there is none."""
        n = self.frame_count - first if n is None else n
        out = np.zeros(n, dtype=np.float64)
        check(self._lib.psd_engine_scan_hash_dist_host_at(self._h, int(hash_slot), first, n, out.ctypes.data),
              "psd_engine_scan_hash_dist_host")
        if out.shape[0]:
            self._synced()
        return out

    # -- instrumentation --
    def timing_reset(self):
        check(self._lib.psd_engine_timing_reset(self._h))

    def timing_ms(self) -> tuple[float, float, int]:
        t, s, k = C.c_float(), C.c_float(), C.c_uint64()
        check(self._lib.psd_engine_timing_ms(self._h, C.byref(t), C.byref(s), C.byref(k)))
        return t.value, s.value, k.value

    def debug_plane(self, which: int, index: int) -> np.ndarray:
        if which == 0:
            out = np.zeros((self.height, self.width, 3), dtype=np.uint8)
        else:
            out = np.zeros((self.height, self.width), dtype=np.uint8)
        check(self._lib.psd_engine_debug_plane(self._h, which, index, out.ctypes.data, out.nbytes),
              "psd_engine_debug_plane")
        return out


class SlotView:
    """An Engine with one edge slot and one hash slot selected: what a detector (or a sweep's pixel group) that
    shares the engine reads.  Everything else is the engine's own."""

    def __init__(self, engine: Engine, edge_slot: int = 0, hash_slot: int = 0):
        self._engine = engine
        self.edge_slot, self.hash_slot = int(edge_slot), int(hash_slot)

    def __getattr__(self, name):
        return getattr(self._engine, name)

    @property
    def hash_size(self) -> int:
        return self._engine.hash_size_at(self.hash_slot)

    def device_edge_sads(self) -> int | None:
        return self._engine.device_edge_sads(self.edge_slot)

    def device_hash(self) -> int | None:
        return self._engine.device_hash(hash_slot=self.hash_slot)

    def read_hash(self, first: int = 0, n: int | None = None) -> np.ndarray:
        return self._engine.read_hash(first, n, hash_slot=self.hash_slot)

    def scan_content(self, weights, first: int = 0, n: int | None = None):
        return self._engine.scan_content(weights, first, n, edge_slot=self.edge_slot)

    def scan_hash_dist(self, first: int = 0, n: int | None = None) -> np.ndarray:
        return self._engine.scan_hash_dist(first, n, hash_slot=self.hash_slot)


def bind_host_to_gpu_numa_node(device: int = 0) -> dict:
    """Pin the calling process to the CPUs of the GPU's NUMA node so that page-locked staging
    buffers allocated afterwards are local to the GPU's PCIe root (first-touch placement).  Returns
    what was found; a no-op when the topology is not exposed."""
    import os
    lib = _capi.load()
    buf = C.create_string_buffer(32)
    check(lib.psd_device_pci_bus_id(device, buf, 32), "psd_device_pci_bus_id")
    bdf = buf.value.decode().lower()
    info = {"pci": bdf, "numa_node": None, "cpus": None}
    base = f"/sys/bus/pci/devices/{bdf}"
    try:
        node = int(open(f"{base}/numa_node").read().strip())
        info["numa_node"] = node
        cpulist = open(f"{base}/local_cpulist").read().strip()
        cpus = set()
        for part in cpulist.split(","):
            if "-" in part:
                a, b = part.split("-")
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        allowed = cpus & set(os.sched_getaffinity(0))
        if node >= 0 and allowed:
            os.sched_setaffinity(0, allowed)
            info["cpus"] = len(allowed)
    except (OSError, ValueError):
        pass
    return info


def synth_frames_device(dptr: int, params: np.ndarray, width: int, height: int,
                        frame_stride: int | None = None, device: int = 0):
    """Render ScenePlan rows straight into HBM (bit-exact twin of synth.render_frames)."""
    p = np.ascontiguousarray(params, dtype=np.int32)
    check(_capi.load().psd_synth_frames(device, dptr, p.ctypes.data, p.shape[0], width, height,
                                        int(frame_stride or width * height * 3), None),
          "psd_synth_frames")


def gather_bgr(frames, dst: int, dst_frame_stride: int | None = None, channel_order: str = "bgr", device: int = 0,
               stream: int | None = None):
    """Copy CUDA frames of any layout (a DLPack exporter, as `Engine.submit` takes them) to packed BGR24 at device
    pointer `dst`, `dst_frame_stride` bytes apart (default: packed).  Queued on `stream` (cudaStream_t, default
    the legacy default stream) after the exporter's current stream; returns the imported view, whose capsule must
    outlive the copy."""
    v = _dlpack.import_frames(frames, stream=stream or 1, device=device, channel_order=channel_order)
    layout = _capi.PsdFrameLayout(*v.layout)
    check(_capi.load().psd_gather_bgr(device, v.base, C.byref(layout), v.n, v.width, v.height, dst,
                                      int(dst_frame_stride or v.width * v.height * 3), stream),
          "psd_gather_bgr")
    return v


def download_bgr(frames, channel_order: str = "bgr", device: int = 0,
                 scratch: DeviceBuffer | None = None) -> np.ndarray:
    """CUDA frames of any layout -> a host numpy BGR24 array of the same (N,H,W,3) or (H,W,3) shape.  `scratch`: a
    device buffer of at least the frames' packed size to gather into (default: one allocated and freed here; a
    reused one spares the cudaFree, which waits for the whole device)."""
    meta = _dlpack.import_frames(frames, device=device)
    fb = meta.width * meta.height * 3
    own = scratch is None or scratch.nbytes < meta.n * fb
    buf = DeviceBuffer(max(1, meta.n * fb), device) if own else scratch
    try:
        gather_bgr(frames, buf.ptr, fb, channel_order, device)
        out = buf.download(meta.n * fb)   # cudaMemcpy: ordered after the gather on the legacy default stream
    finally:
        if own:
            buf.close()
    shape = (meta.n, meta.height, meta.width, 3) if meta.ndim == 4 else (meta.height, meta.width, 3)
    return out.reshape(shape)


__all__ = ["Engine", "SlotView", "PinnedBuffer", "DeviceBuffer", "synth_frames_device", "gather_bgr", "download_bgr",
           "bind_host_to_gpu_numa_node", "F_HSV", "F_BGRSUM", "F_YHIST", "F_EDGES", "F_HASH"]
