// Many clips scored back to back into one engine (clips.py).  The fused pass scores a frame from that frame and
// its predecessor only, so the integer results of the concatenated stream are each clip's own except at the clip
// edges, where a frame was diffed against the previous clip's last frame.  Two kernels finish the job:
//   psd_clip_fill    after a psd_scan_* over the whole pass, sets the metric entries at every clip's head and tail
//                    to what a one-clip engine's scan writes there, bit for bit (0.0 for content_val, the scan's
//                    NaN for an incomplete adaptive window or a frame without a predecessor)
//   psd_clip_cuts    one thread per (cell, clip) runs the cell's automaton (cut_automata.cuh) over the clip's slice
//                    of the metric arrays, with the clip's first frame number and min_frames: a counting pass, an
//                    exclusive scan of the counts, then a writing pass into one compact cut array
// Either is one launch (three for psd_clip_cuts) per pass whatever the number of clips.
#include <math_constants.h>

#include "cut_automata.cuh"

namespace psd {

__global__ void __launch_bounds__(256) psd_clip_fill_kernel(double* __restrict__ values, int64_t n,
                                                            const int64_t* __restrict__ offsets, int32_t n_clips,
                                                            int32_t head, int32_t tail, int fill_nan, double fill) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t per = (int64_t)head + tail;
    if (t >= (int64_t)n_clips * per) return;
    const int64_t j = t / per, k = t % per;
    // clamped to [0, n): a malformed table writes nothing outside the array
    const int64_t b = min(max(offsets[j], (int64_t)0), n), e = min(max(offsets[j + 1], b), n);
    const int64_t i = k < head ? b + k : e - tail + (k - head);
    if (i < b || i >= e) return;
    values[i] = fill_nan ? CUDART_NAN : fill;  // psd_scan_adaptive's and psd_scan_hist_correl's NaN (sign bit set)
}

// Counting pass (WRITE = false): cut_offsets[t] = how many cuts (cell, clip) t emits.  Writing pass: the cuts of t
// at cuts[cut_offsets[t] ..], after psd_clip_scan_kernel turned the counts into offsets; nothing when the total
// exceeds cap.  t = cell * n_clips + clip, so one cell's clips are adjacent threads.
template <bool WRITE>
__global__ void __launch_bounds__(128) psd_clip_cuts_kernel(const psd_sweep_cell* __restrict__ cells, int32_t n_cells,
                                                            const int64_t* __restrict__ offsets,
                                                            const int64_t* __restrict__ first_frame, int32_t n_clips,
                                                            const int64_t* __restrict__ min_frames,
                                                            int64_t* __restrict__ cuts, int64_t cap,
                                                            int64_t* __restrict__ cut_offsets) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t m = (int64_t)n_cells * n_clips;
    if (t >= m) return;
    const int64_t k = t / n_clips, j = t % n_clips;
    const int64_t b = max(offsets[j], (int64_t)0), e = max(offsets[j + 1], b);
    CutSink out{nullptr, 0, 0};  // cap 0: counts only
    if (WRITE) {
        if (cut_offsets[m] > cap) return;
        const int64_t o = cut_offsets[t];
        out.cuts = cuts + o;
        out.cap = (int32_t)(cut_offsets[t + 1] - o);
    }
    run_cell(cells[k], b, e - b, first_frame[j], min_frames[t], out);
    if (!WRITE) cut_offsets[t] = out.n;
}

// In place: v[0, m) counts -> exclusive offsets, v[m] = their sum.  One block walks the array 1024 entries at a
// time (m is cells x clips, a few thousand to a few hundred thousand).
__global__ void __launch_bounds__(1024) psd_clip_scan_kernel(int64_t* __restrict__ v, int64_t m) {
    __shared__ int64_t warp_sums[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t carry = 0;
    for (int64_t base = 0; base < m; base += 1024) {
        const int64_t i = base + threadIdx.x;
        const int64_t x = i < m ? v[i] : 0;
        int64_t s = x;  // inclusive scan within the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xFFFFFFFFu, s, o);
            if (lane >= o) s += y;
        }
        if (lane == 31) warp_sums[w] = s;
        __syncthreads();
        if (w == 0) {
            int64_t ws = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int64_t y = __shfl_up_sync(0xFFFFFFFFu, ws, o);
                if (lane >= o) ws += y;
            }
            warp_sums[lane] = ws;
        }
        __syncthreads();
        if (i < m) v[i] = carry + (w ? warp_sums[w - 1] : 0) + s - x;
        carry += warp_sums[31];
        __syncthreads();  // warp_sums is rewritten by the next chunk
    }
    if (threadIdx.x == 0) v[m] = carry;
}

}  // namespace psd

using namespace psd;

extern "C" int psd_clip_fill(double* values, int64_t n, const int64_t* clip_offsets, int32_t n_clips, int32_t head,
                             int32_t tail, int32_t fill_nan, double fill, void* stream) {
    PSD_REQUIRE(clip_offsets, "psd_clip_fill: no clip table");
    PSD_REQUIRE(n >= 0 && n_clips >= 0 && head >= 0 && tail >= 0 && (fill_nan == 0 || fill_nan == 1),
                "psd_clip_fill: bad args");
    const int64_t threads = (int64_t)n_clips * ((int64_t)head + tail);
    if (n == 0 || threads == 0) return PSD_OK;
    PSD_REQUIRE(values, "psd_clip_fill: no metric array");
    psd_clip_fill_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        values, n, clip_offsets, n_clips, head, tail, fill_nan, fill);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_clip_cuts(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                             const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                             int64_t cuts_cap, int64_t* cut_offsets, void* stream) {
    PSD_REQUIRE(clip_offsets, "psd_clip_cuts: no clip table");
    PSD_REQUIRE(n_cells >= 0 && n_clips >= 0 && cuts_cap >= 0, "psd_clip_cuts: bad args");
    PSD_REQUIRE(cut_offsets, "psd_clip_cuts: no cut_offsets array");
    const int rc = validate_sweep_cells(cells, n_cells, "psd_clip_cuts");
    if (rc != PSD_OK) return rc;
    const int64_t m = (int64_t)n_cells * n_clips;
    cudaStream_t s = (cudaStream_t)stream;
    if (m == 0) {
        PSD_CUDA(cudaMemsetAsync(cut_offsets, 0, sizeof(int64_t), s));
        return PSD_OK;
    }
    PSD_REQUIRE(clip_first_frame && min_frames, "psd_clip_cuts: no clip first frames / min_frames");
    PSD_REQUIRE(cuts || cuts_cap == 0, "psd_clip_cuts: no cut array");
    psd_sweep_cell* d_cells = nullptr;
    const size_t bytes = sizeof(psd_sweep_cell) * (size_t)n_cells;
    PSD_CUDA(cudaMallocAsync((void**)&d_cells, bytes, s));
    PSD_CUDA(cudaMemcpyAsync(d_cells, cells, bytes, cudaMemcpyHostToDevice, s));  // pageable: staged before return
    const unsigned blocks = (unsigned)((m + 127) / 128);
    psd_clip_cuts_kernel<false><<<blocks, 128, 0, s>>>(d_cells, n_cells, clip_offsets, clip_first_frame, n_clips,
                                                       min_frames, cuts, cuts_cap, cut_offsets);
    PSD_CHECK_LAUNCH();
    psd_clip_scan_kernel<<<1, 1024, 0, s>>>(cut_offsets, m);
    PSD_CHECK_LAUNCH();
    psd_clip_cuts_kernel<true><<<blocks, 128, 0, s>>>(d_cells, n_cells, clip_offsets, clip_first_frame, n_clips,
                                                      min_frames, cuts, cuts_cap, cut_offsets);
    PSD_CHECK_LAUNCH();
    count_launch(3);
    PSD_CUDA(cudaFreeAsync(d_cells, s));
    return PSD_OK;
}
