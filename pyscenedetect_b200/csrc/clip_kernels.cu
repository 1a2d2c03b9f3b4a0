// Many clips scored back to back into one engine (clips.py).  The fused pass scores a frame from that frame and
// its predecessor only, so the integer results of the concatenated stream are each clip's own except at the clip
// edges, where a frame was diffed against the previous clip's last frame.  Two kernels finish the job:
//   psd_clip_fill    after a psd_scan_* over the whole pass, sets the metric entries at every clip's head and tail
//                    to what a one-clip engine's scan writes there, bit for bit (0.0 for content_val, the scan's
//                    NaN for an incomplete adaptive window or a frame without a predecessor)
//   psd_clip_cuts    one thread per (cell, clip) runs the cell's automaton (cut_automata.cuh) over the clip's slice
//                    of the metric arrays, with the clip's first frame number and min_frames: a counting pass, an
//                    exclusive scan of the counts, then a writing pass into one compact cut array
//   psd_clip_eval    the counterpart of psd_sweep_eval for psd_clip_cuts' compact output: every (cell, clip) list
//                    turned in place into its predicted list, every (cell, clip, tolerance) scored against clip j's
//                    ground truth with score_predictions (sweep_eval.cuh), and the counts summed over the clips
// Each is one launch (three for psd_clip_cuts and psd_clip_eval) per pass whatever the number of cells and clips.
#include <math_constants.h>

#include "cut_automata.cuh"
#include "sweep_eval.cuh"

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

// [lo, hi) of segment i of a CSR array of `total` entries, clamped: a malformed table reads and writes nothing outside
// the arrays and the workspace
__device__ __forceinline__ void segment(const int64_t* __restrict__ offsets, int64_t i, int64_t total, int64_t& lo,
                                        int64_t& hi) {
    lo = min(max(offsets[i], (int64_t)0), total);
    hi = min(max(offsets[i + 1], lo), total);
}

// One thread per (cell, clip) t: its cut list -> the predicted list of sweep.py:169 in place, as
// psd_sweep_pred_kernel does; n_pred[t] = its length with the end frame, which is not stored.  A list longer than
// max_cuts is not scored (n_pred -1) and the lowest such t goes to *over.
__global__ void __launch_bounds__(128) clip_pred_kernel(int64_t* __restrict__ cuts,
                                                        const int64_t* __restrict__ cut_offsets, int64_t m,
                                                        int64_t cuts_total, int64_t max_cuts,
                                                        int32_t* __restrict__ n_pred,
                                                        unsigned long long* __restrict__ over) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    int64_t b, e;
    segment(cut_offsets, t, cuts_total, b, e);
    if (e - b > max_cuts) {
        n_pred[t] = -1;
        atomicMin(over, (unsigned long long)t);
        return;
    }
    const int32_t u = sort_unique(cuts + b, (int32_t)(e - b));
    n_pred[t] = u ? u + 1 : 0;
}

// One thread per (cell k, clip j, tolerance q), tid = (k * n_clips + j) * n_tol + q.  The matching bitmaps are laid
// out so that their offsets follow from the CSR offsets alone: list t's bits start at word t + floor(o_t / 32) of
// tolerance q's block of words_p, clip j's ground-truth bits at word j + floor(gb_j / 32) of the (k, q) block of
// words_g (likewise the fades).  Segment t needs floor(c_t / 32) + 1 words, and t + 1 starts at least that far on.
__global__ void __launch_bounds__(128) clip_eval_kernel(
    const int64_t* __restrict__ cuts, const int64_t* __restrict__ cut_offsets, const int32_t* __restrict__ n_pred,
    int32_t n_cells, int32_t n_clips, int64_t cuts_total, const int64_t* __restrict__ end_frame,
    const int64_t* __restrict__ gt_offsets, const int64_t* __restrict__ gt, int32_t n_gt,
    const int64_t* __restrict__ fade_offsets, const int64_t* __restrict__ fades, int32_t n_fades, Tolerances tols,
    int32_t n_tol, uint32_t* __restrict__ workspace, int64_t words_p, int64_t words_g, int64_t words_f,
    int64_t* __restrict__ out_hard, int64_t* __restrict__ out_fades) {
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t m = (int64_t)n_cells * n_clips;
    if (tid >= m * n_tol) return;
    const int64_t t = tid / n_tol, k = t / n_clips, j = t % n_clips;
    const int32_t q = (int32_t)(tid % n_tol);
    int64_t* hard = out_hard + tid * 5;
    int64_t* fade_counts = q == 0 ? out_fades + t * 3 : nullptr;
    const int32_t np = n_pred[t];
    if (np < 0) {
        for (int r = 0; r < 5; ++r) hard[r] = 0;
        if (fade_counts)
            for (int r = 0; r < 3; ++r) fade_counts[r] = 0;
        return;
    }
    int64_t b, e, gb, ge, fb, fe;
    segment(cut_offsets, t, cuts_total, b, e);
    segment(gt_offsets, j, n_gt, gb, ge);
    segment(fade_offsets, j, n_fades, fb, fe);
    const int64_t kq = k * n_tol + q;
    uint32_t* used_p = workspace + q * words_p + t + b / 32;
    uint32_t* used_g = workspace + n_tol * words_p + kq * words_g + j + gb / 32;
    uint32_t* used_f = workspace + n_tol * words_p + (int64_t)n_cells * n_tol * words_g + kq * words_f + j + fb / 32;
    for (int64_t w = 0; w < words_for(np); ++w) used_p[w] = 0u;
    for (int64_t w = 0; w < words_for(ge - gb); ++w) used_g[w] = 0u;
    for (int64_t w = 0; w < words_for(fe - fb); ++w) used_f[w] = 0u;
    score_predictions(cuts + b, np, end_frame[j], gt + gb, (int32_t)(ge - gb), fades + 2 * fb, (int32_t)(fe - fb),
                      tolerance_at(tols, q), used_p, used_g, used_f, hard, fade_counts);
}

// One thread per (cell, count): the count summed over the clips, totals_hard[k][q][5] then totals_fades[k][3].
// Integer sums: the same in any order.
__global__ void __launch_bounds__(256) clip_totals_kernel(const int64_t* __restrict__ hard,
                                                          const int64_t* __restrict__ fades, int32_t n_cells,
                                                          int32_t n_clips, int32_t n_tol,
                                                          int64_t* __restrict__ totals_hard,
                                                          int64_t* __restrict__ totals_fades) {
    const int64_t per = (int64_t)n_tol * 5 + 3;
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (tid >= n_cells * per) return;
    const int64_t k = tid / per, r = tid % per;
    int64_t s = 0;
    if (r < (int64_t)n_tol * 5) {
        const int64_t row = (int64_t)n_tol * 5;
        for (int32_t j = 0; j < n_clips; ++j) s += hard[(k * n_clips + j) * row + r];
        totals_hard[k * row + r] = s;
    } else {
        for (int32_t j = 0; j < n_clips; ++j) s += fades[(k * n_clips + j) * 3 + (r - (int64_t)n_tol * 5)];
        totals_fades[k * 3 + (r - (int64_t)n_tol * 5)] = s;
    }
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

extern "C" int psd_clip_eval(int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips,
                             int64_t cuts_total, int64_t max_cuts, const int64_t* clip_end_frame,
                             const int64_t* gt_offsets, const int64_t* gt_cuts, int32_t n_gt,
                             const int64_t* fade_offsets, const int64_t* fades, int32_t n_fades,
                             const int32_t* tolerances, int32_t n_tol, void* workspace, size_t workspace_bytes,
                             int32_t* out_n_pred, int64_t* out_hard, int64_t* out_fades, int64_t* out_totals_hard,
                             int64_t* out_totals_fades, int64_t* out_over, void* stream) {
    PSD_REQUIRE(n_cells >= 0 && n_clips >= 0 && cuts_total >= 0 && n_gt >= 0 && n_fades >= 0,
                "psd_clip_eval: bad args");
    PSD_REQUIRE(max_cuts >= 0 && max_cuts <= INT32_MAX, "psd_clip_eval: max_cuts must be 0 to %d", INT32_MAX);
    PSD_REQUIRE(tolerances && n_tol >= 1 && n_tol <= PSD_SWEEP_MAX_TOLERANCES, "psd_clip_eval: 1 to %d tolerances",
                PSD_SWEEP_MAX_TOLERANCES);
    Tolerances tols{};
    for (int32_t q = 0; q < n_tol; ++q) {
        PSD_REQUIRE(tolerances[q] >= 0, "psd_clip_eval: tolerance %d is negative", tolerances[q]);
        tols.t[q] = tolerances[q];
    }
    PSD_REQUIRE(out_over, "psd_clip_eval: no out_over");
    const int64_t m = (int64_t)n_cells * n_clips;
    PSD_REQUIRE(n_cells == 0 || (out_totals_hard && out_totals_fades), "psd_clip_eval: no totals arrays");
    if (m > 0) {
        PSD_REQUIRE(cut_offsets && clip_end_frame && gt_offsets && fade_offsets, "psd_clip_eval: no clip tables");
        PSD_REQUIRE(cuts || cuts_total == 0, "psd_clip_eval: cuts is NULL");
        PSD_REQUIRE(n_gt == 0 || gt_cuts, "psd_clip_eval: gt_cuts is NULL");
        PSD_REQUIRE(n_fades == 0 || fades, "psd_clip_eval: fades is NULL");
        PSD_REQUIRE(out_n_pred && out_hard && out_fades, "psd_clip_eval: no output arrays");
    }
    const int64_t wp = m + words_for(cuts_total), wg = n_clips + words_for(n_gt), wf = n_clips + words_for(n_fades);
    const size_t need = 4u * ((size_t)n_tol * (size_t)wp + (size_t)n_cells * (size_t)n_tol * (size_t)(wg + wf));
    PSD_REQUIRE(m == 0 || (workspace && workspace_bytes >= need), "psd_clip_eval: workspace needs %zu bytes", need);
    cudaStream_t s = (cudaStream_t)stream;
    PSD_CUDA(cudaMemsetAsync(out_over, 0xFF, sizeof(int64_t), s));  // -1: no list longer than max_cuts
    if (m == 0) {  // no clip: every total is 0
        if (n_cells > 0) {
            PSD_CUDA(cudaMemsetAsync(out_totals_hard, 0, sizeof(int64_t) * 5 * (size_t)n_cells * n_tol, s));
            PSD_CUDA(cudaMemsetAsync(out_totals_fades, 0, sizeof(int64_t) * 3 * (size_t)n_cells, s));
        }
        return PSD_OK;
    }
    clip_pred_kernel<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(cuts, cut_offsets, m, cuts_total, max_cuts,
                                                                  out_n_pred, (unsigned long long*)out_over);
    PSD_CHECK_LAUNCH();
    const int64_t threads = m * n_tol;
    clip_eval_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
        cuts, cut_offsets, out_n_pred, n_cells, n_clips, cuts_total, clip_end_frame, gt_offsets, gt_cuts, n_gt,
        fade_offsets, fades, n_fades, tols, n_tol, (uint32_t*)workspace, wp, wg, wf, out_hard, out_fades);
    PSD_CHECK_LAUNCH();
    const int64_t sums = (int64_t)n_cells * ((int64_t)n_tol * 5 + 3);
    clip_totals_kernel<<<(unsigned)((sums + 255) / 256), 256, 0, s>>>(out_hard, out_fades, n_cells, n_clips, n_tol,
                                                                     out_totals_hard, out_totals_fades);
    PSD_CHECK_LAUNCH();
    count_launch(3);
    return PSD_OK;
}
