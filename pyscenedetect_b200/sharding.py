"""Multi-GPU time sharding: one process per GPU, contiguous frame ranges, one-frame halo.

Score(t) depends only on frames t and t-1 (content_detector.py:166-175,
histogram_detector.py:98), so rank r scores frames [bounds[r], bounds[r+1]) after receiving
frame bounds[r]-1 from rank r-1 (a ring shift over NCCL/NVLink with the `nccl` backend, `gloo`
in the CPU tests).  The per-frame INTEGER results are then gathered on rank 0, where the
trailing device scans and the cut state machines run once over the whole sequence - so the
cut list, metrics and CSV equal the serial run by construction (integer sums are
order-independent; the float64 math happens once, in the reference's order).

There is no data-path collective besides the halo send/recv and the small result gather.
"""

from __future__ import annotations

import numpy as np

from ._capi import F_HASH, F_YHIST, SUMS_DTYPE, hash_words


def shard_bounds(n_frames: int, world: int) -> list[int]:
    """Contiguous, near-equal time ranges: rank r owns [b[r], b[r+1])."""
    return [(r * n_frames) // world for r in range(world + 1)]


class TorchComm:
    """torch.distributed plumbing (nccl on GPUs, gloo on CPU).  Frames travel as uint8 tensors;
    with the nccl backend they are staged through `device` memory."""

    def __init__(self, device=None):
        import torch
        import torch.distributed as dist
        self.torch, self.dist = torch, dist
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.device = device if device is not None else torch.device("cpu")

    def _t(self, arr: np.ndarray):
        return self.torch.from_numpy(np.array(arr, copy=True, order="C")).to(self.device)

    def exchange_halo(self, last_frame: np.ndarray | None, shape) -> np.ndarray | None:
        """Send my last frame to rank+1, receive rank-1's last frame (None on rank 0)."""
        dist, torch = self.dist, self.torch
        ops, recv = [], None
        if self.rank + 1 < self.world:
            assert last_frame is not None
            ops.append(dist.P2POp(dist.isend, self._t(last_frame), self.rank + 1))
        if self.rank > 0:
            recv = torch.empty(tuple(shape), dtype=torch.uint8, device=self.device)
            ops.append(dist.P2POp(dist.irecv, recv, self.rank - 1))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        if recv is None:
            return None
        if recv.is_cuda:
            # the halo stays in HBM: the engine copies it device-to-device (psd_engine_set_halo_device)
            torch.cuda.current_stream().synchronize()
            self._halo_keepalive = recv
            return recv
        return recv.cpu().numpy()

    def gather_rows(self, rows: np.ndarray, counts: list[int]) -> np.ndarray | None:
        """Concatenate per-rank row blocks (raw bytes) on rank 0; other ranks get None.  One `gather`
        (only rank 0 receives), blocks padded to the longest shard (shards differ by at most one row)."""
        dist, torch = self.dist, self.torch
        if self.world == 1:
            return rows
        row_bytes = rows.dtype.itemsize * int(np.prod(rows.shape[1:], dtype=np.int64))
        cap = max(counts) * row_bytes
        raw = np.zeros(cap, dtype=np.uint8)
        flat = np.ascontiguousarray(rows).view(np.uint8).reshape(-1)
        raw[: flat.size] = flat
        buf = torch.from_numpy(raw).to(self.device)
        outs = [torch.empty_like(buf) for _ in range(self.world)] if self.rank == 0 else None
        dist.gather(buf, outs, dst=0)
        if self.rank != 0:
            return None
        host = torch.stack(outs).cpu().numpy()  # one device->host copy of all blocks
        parts = [np.frombuffer(host[r, : counts[r] * row_bytes].tobytes(), dtype=rows.dtype)
                 .reshape((counts[r],) + rows.shape[1:]) for r in range(self.world)]
        return np.concatenate(parts)


class GatheredResults:
    """Scan provider over gathered integer results: presents the `Engine.scan_*` interface the
    detectors consume, backed by the stateless device scans of the C-ABI (psd_scan_*)."""

    def __init__(self, sums: np.ndarray, yhist: np.ndarray | None, n_pixels: int, device: int = 0,
                 hashes: np.ndarray | None = None, hash_size: int = 8, hash_lowpass: int = 2):
        import ctypes as C

        from . import _capi
        from .engine import DeviceBuffer
        self._C, self._capi = C, _capi
        self._lib = _capi.load()
        self.device = device
        self.n_pixels = int(n_pixels)
        self._n = int(sums.shape[0])
        self._sums = DeviceBuffer(max(1, sums.nbytes), device)
        self._sums.upload(sums.view(np.uint8).reshape(-1))
        self._hist = None
        if yhist is not None:
            self._hist = DeviceBuffer(max(1, yhist.nbytes), device)
            self._hist.upload(np.ascontiguousarray(yhist).view(np.uint8).reshape(-1))
        self._hashes = None
        self.hash_size = int(hash_size)
        if hashes is not None:
            self._hashes = DeviceBuffer(max(1, hashes.nbytes), device)
            self._hashes.upload(np.ascontiguousarray(hashes).view(np.uint8).reshape(-1))
        self._DeviceBuffer = DeviceBuffer

    @property
    def frame_count(self) -> int:
        return self._n

    # the part of the `Engine` interface `device_cuts.DeviceCuts` needs: the gathered arrays live in HBM
    compute_stream = 0  # scans and automata run on the default stream, the downloads below are stream-ordered

    def device_results(self):
        return self._sums.ptr, (self._hist.ptr if self._hist is not None else None)

    def device_hash(self):
        return self._hashes.ptr if self._hashes is not None else None

    def device_edge_sads(self):
        return None  # the gathered sums' own sad_edges

    def sync(self):
        pass

    def _out(self, count: int):
        return self._DeviceBuffer(max(8, count * 8), self.device)

    def _fetch(self, buf, count: int) -> np.ndarray:
        return buf.download(count * 8).view(np.float64).copy()

    def scan_content(self, weights, first: int = 0, n: int | None = None):
        n = self._n - first if n is None else n
        w = (self._C.c_double * 4)(*[float(x) for x in weights])
        wsum = float(sum(abs(x) for x in weights))
        val, comps = self._out(n), self._out(4 * n)
        self._capi.check(self._lib.psd_scan_content(self._sums.ptr + first * 64, n, self.n_pixels, w, wsum,
                                                    comps.ptr, val.ptr, None), "psd_scan_content")
        return self._fetch(val, n), self._fetch(comps, 4 * n).reshape(n, 4)

    def scan_adaptive(self, scores: np.ndarray, window_width: int, min_content_val: float) -> np.ndarray:
        s = np.ascontiguousarray(scores, dtype=np.float64)
        n = s.shape[0]
        inp, out = self._out(n), self._out(n)
        inp.upload(s.view(np.uint8))
        self._capi.check(self._lib.psd_scan_adaptive(inp.ptr, n, int(window_width), float(min_content_val),
                                                     out.ptr, None), "psd_scan_adaptive")
        return self._fetch(out, n)

    def scan_average(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self._n - first if n is None else n
        out = self._out(n)
        self._capi.check(self._lib.psd_scan_average(self._sums.ptr + first * 64, n, self.n_pixels * 3,
                                                    out.ptr, None), "psd_scan_average")
        return self._fetch(out, n)

    def scan_hash_dist(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self._n - first if n is None else n
        out = self._out(n)
        row = 8 * hash_words(self.hash_size)   # bytes per frame: the PSD_HASH_WORDS_FOR(size) stride
        prev = self._hashes.ptr + (first - 1) * row if first > 0 else None
        self._capi.check(self._lib.psd_scan_hash_dist(self._hashes.ptr + first * row, n, self.hash_size,
                                                      prev, out.ptr, None), "psd_scan_hash_dist")
        return self._fetch(out, n)

    def scan_hist_correl(self, bins: int, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self._n - first if n is None else n
        out = self._out(n)
        prev = self._hist.ptr + (first - 1) * 1024 if first > 0 else None
        self._capi.check(self._lib.psd_scan_hist_correl(self._hist.ptr + first * 1024, n, int(bins), prev,
                                                        out.ptr, None), "psd_scan_hist_correl")
        return self._fetch(out, n)


def detect_sharded(frames_local: np.ndarray, first_index: int, total_frames: int, detector, fps,
                   comm, engine_factory=None, results_factory=None, batch_size: int = 64,
                   n_local: int | None = None, pinned: bool = False, device: int = 0,
                   timings: dict | None = None):
    """Run `detector` over a sequence that is split across ranks by contiguous time range.

    frames_local: this rank's frames (n_local,H,W,3) = global frames [first_index, first_index+n_local).
    If `n_local` is larger than the array, the array is cycled (a page-locked ring of distinct
    frames, as bench.py's end-to-end leg uses); `pinned=True` DMAs straight from it.
    Returns (cut_frame_numbers, gathered_sums) on rank 0 and (None, None) elsewhere.
    `engine_factory` / `results_factory` exist so the CPU tests can substitute oracle-backed
    scorers; the defaults are the CUDA engine and the C-ABI device scans.

    On rank 0 the cut list comes from the device automata (`device_cuts.DeviceCuts`: psd_scan_* +
    psd_cuts_* over the gathered arrays, only the cut frame numbers travel back) unless the detector
    carries a StatsManager - then the per-frame Python state machines run so that every metric row
    is recorded.  `timings`, if given, receives the wall seconds of the phases (halo, score incl. H2D,
    gather, cuts).
    """
    import time

    from .compat import FrameTimecode
    from .detectors._base import pixel_group_of
    t_start = time.perf_counter()
    if engine_factory is None:
        from .engine import Engine as engine_factory  # noqa: N813
    if results_factory is None:
        results_factory = GatheredResults
    ring, h, w = frames_local.shape[0], frames_local.shape[1], frames_local.shape[2]
    n_local = ring if n_local is None else int(n_local)
    group = pixel_group_of(detector)
    features = group.features
    eng = engine_factory(w, h, features, device=device, max_batch=batch_size,
                         edge_kernel_size=group.edge_kernel_size, **dict(group.engine_kwargs))
    halo = comm.exchange_halo(frames_local[(n_local - 1) % ring] if n_local else None, (h, w, 3))
    if halo is not None:
        if isinstance(halo, np.ndarray):
            eng.set_halo(halo)
        else:
            eng.set_halo_device(halo.data_ptr())
    t_halo = time.perf_counter()
    i = 0
    while i < n_local:
        j = i % ring
        k = min(batch_size, n_local - i, ring - j)
        eng.submit(frames_local[j:j + k], pinned=pinned)
        i += k
    sums = eng.read_sums()
    yh = eng.read_yhist() if features & F_YHIST else None
    hs = eng.read_hash() if features & F_HASH else None
    t_score = time.perf_counter()
    counts = [b - a for a, b in zip(shard_bounds(total_frames, comm.world)[:-1],
                                    shard_bounds(total_frames, comm.world)[1:])]
    assert counts[comm.rank] == n_local and shard_bounds(total_frames, comm.world)[comm.rank] == first_index
    all_sums = comm.gather_rows(sums, counts)
    all_hist = comm.gather_rows(yh, counts) if yh is not None else None
    all_hash = comm.gather_rows(hs, counts) if hs is not None else None
    eng.close()
    t_gather = time.perf_counter()

    def note(t_end):
        if timings is not None:
            timings.update(halo_s=t_halo - t_start, score_s=t_score - t_halo, gather_s=t_gather - t_score,
                           cuts_s=t_end - t_gather)
    if comm.rank != 0:
        note(t_gather)
        return None, None
    assert all_sums.dtype == SUMS_DTYPE and all_sums.shape[0] == total_frames
    res = (results_factory(all_sums, all_hist, w * h, device, hashes=all_hash, **detector.engine_kwargs())
           if all_hash is not None else results_factory(all_sums, all_hist, w * h, device))
    detector.attach_engine(res)
    detector._base_index = 0
    if detector.stats_manager is None and hasattr(res, "device_results"):
        from .device_cuts import DeviceCuts, cuts_for_detector
        cut_frames = sorted(set(cuts_for_detector(DeviceCuts(res), detector, fps)))
        note(time.perf_counter())
        return cut_frames, all_sums
    tcs =[FrameTimecode(i, fps) for i in range(total_frames)]
    cuts = []
    for i in range(0, total_frames, 4096):
        cuts += detector.consume_results(tcs[i:i + 4096], i)
    cuts += detector.post_process(tcs[-1])
    note(time.perf_counter())
    return sorted({c.frame_num for c in cuts}), all_sums
