// Parameter sweep on the device: every cell of a detector-parameter grid over one scored video.
//   psd_sweep_cuts   benchmark/sweep.py:142-187 (one SceneManager + detector per cell): one thread per
//                    cell runs the cell's automaton (cut_automata.cuh) over the metric arrays the existing
//                    psd_scan_* produced.  The host sorts cells by metric array, so a warp's 32 cells load
//                    each frame's value together (one broadcast load per warp) and take the same branch
//                    most of the time: they only diverge on the frames where some of them cut.
//   psd_sweep_eval   benchmark/evaluator.py:227-331 (score_video) per (cell, tolerance): first the
//                    predicted list of sweep.py:169, then fade matching, then greedy hard-cut matching.
// The automata are sequential walks, so the sweep is bounded by one thread's latency per frame (a load, a
// compare, a few integer ops): G cells cost about as much as one cell until the cells fill the GPU.
#include "cut_automata.cuh"

namespace psd {

__global__ void __launch_bounds__(128) psd_sweep_cuts_kernel(const psd_sweep_cell* __restrict__ cells,
                                                             int32_t n_cells, int64_t n, int64_t first_frame,
                                                             int64_t* __restrict__ cuts,
                                                             int32_t* __restrict__ count, int32_t cap) {
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_cells) return;
    const psd_sweep_cell c = cells[k];
    CutSink out{cuts + (int64_t)k * cap, cap, 0};
    switch (c.kind) {
        case PSD_SWEEP_CONTENT: {
            // content_detector.py:210 inside the automaton: no per-cell flag array
            const double* __restrict__ val = c.metric;
            const double thr = c.threshold;
            flash_filter_cuts([&](int64_t i) { return val[i] >= thr; }, n, first_frame, c.min_frames, c.mode, out);
            break;
        }
        case PSD_SWEEP_ADAPTIVE:
            adaptive_cuts(c.metric, c.metric2, n, first_frame, c.window, c.threshold, c.min_content_val,
                          c.min_frames, out);
            break;
        case PSD_SWEEP_THRESHOLD:
            threshold_cuts(c.metric, n, first_frame, c.threshold, c.mode, c.fade_bias, c.min_frames,
                           c.add_final_scene, out);
            break;
        case PSD_SWEEP_HISTOGRAM:
            histogram_cuts(c.metric, n, first_frame, c.threshold, c.min_frames, out);
            break;
        default:  // PSD_SWEEP_HASH (the host rejects any other kind)
            hash_cuts(c.metric, n, first_frame, c.threshold, c.min_frames, out);
            break;
    }
    count[k] = out.n;
}

// Cell k's cut slice -> the predicted list of sweep.py:169, in place: sorted(set(cuts)), then end_frame
// when there is a cut.  The end is not stored (the slice may be full): entry n_pred - 1 is end_frame.
// Insertion sort is linear on the strictly increasing lists every automaton but a |fade_bias| > 1
// ThresholdDetector emits (cut_automata.cuh).
__global__ void __launch_bounds__(128) psd_sweep_pred_kernel(int64_t* __restrict__ cuts,
                                                             const int32_t* __restrict__ count, int32_t n_cells,
                                                             int32_t cap, int32_t* __restrict__ n_pred) {
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_cells) return;
    const int32_t c = count[k];
    if (c > cap) {  // overflowed: not scored, the host raises
        n_pred[k] = -1;
        return;
    }
    int64_t* p = cuts + (int64_t)k * cap;
    for (int32_t i = 1; i < c; ++i) {
        const int64_t v = p[i];
        int32_t j = i - 1;
        if (p[j] <= v) continue;
        while (j >= 0 && p[j] > v) {
            p[j + 1] = p[j];
            --j;
        }
        p[j + 1] = v;
    }
    int32_t u = 0;
    for (int32_t i = 0; i < c; ++i)
        if (u == 0 || p[i] != p[u - 1]) p[u++] = p[i];
    n_pred[k] = u ? u + 1 : 0;
}

struct Tolerances {
    int32_t t[PSD_SWEEP_MAX_TOLERANCES];
};

__device__ __forceinline__ bool bit_test_set(uint32_t* bits, int32_t i) {
    const uint32_t m = 1u << (i & 31);
    const bool was = (bits[i >> 5] & m) != 0;
    bits[i >> 5] |= m;
    return was;
}

__device__ __forceinline__ int32_t find_frame(const int64_t* __restrict__ gt, int32_t n_gt, int64_t g) {
    int32_t lo = 0, hi = n_gt;  // first index with gt[index] >= g
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (gt[mid] < g) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n_gt && gt[lo] == g) ? lo : -1;
}

// One thread per (cell, tolerance).  Hard-cut matching (evaluator.py:227-266) claims (d, i, j) pairs in
// sorted order.  With strictly increasing ground truth a prediction p_i has at most two partners at
// distance d, g = p_i - d before g = p_i + d in j order, so the sorted walk is: for d = 0..tol, for i in
// order, claim (i, p_i - d) else (i, p_i + d) if both sides are unused.  No candidate list is built.
__global__ void __launch_bounds__(128) psd_sweep_eval_kernel(
    const int64_t* __restrict__ cuts, const int32_t* __restrict__ n_pred, int32_t n_cells, int32_t cap,
    int64_t end_frame, const int64_t* __restrict__ gt, int32_t n_gt, const int64_t* __restrict__ fades,
    int32_t n_fades, Tolerances tols, int32_t n_tol, uint32_t* __restrict__ workspace, int32_t words_p,
    int32_t words_g, int32_t words_f, int64_t* __restrict__ out_hard, int64_t* __restrict__ out_fades) {
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (tid >= (int64_t)n_cells * n_tol) return;
    const int32_t k = (int32_t)(tid / n_tol), q = (int32_t)(tid % n_tol);
    int64_t* hard = out_hard + tid * 5;
    const int32_t np = n_pred[k];
    if (np < 0) {
        for (int r = 0; r < 5; ++r) hard[r] = 0;
        if (q == 0)
            for (int r = 0; r < 3; ++r) out_fades[(int64_t)k * 3 + r] = 0;
        return;
    }
    const int64_t* p = cuts + (int64_t)k * cap;
    auto pred = [&](int32_t i) { return i < np - 1 ? p[i] : end_frame; };
    uint32_t* used_p = workspace + tid * (int64_t)(words_p + words_g + words_f);
    uint32_t* used_g = used_p + words_p;
    uint32_t* used_f = used_g + words_g;
    for (int32_t w = 0; w < words_p + words_g + words_f; ++w) used_p[w] = 0u;

    // fades (evaluator.py:269-304): first interval containing the prediction consumes it
    int64_t fm = 0, ffp = 0, remaining = np;
    for (int32_t i = 0; i < np; ++i) {
        const int64_t v = pred(i);
        for (int32_t f = 0; f < n_fades; ++f) {
            if (fades[2 * f] <= v && v <= fades[2 * f + 1]) {
                bit_test_set(used_p, i);
                --remaining;
                if (bit_test_set(used_f, f)) ++ffp;
                else ++fm;
                break;
            }
        }
    }
    // hard cuts on the predictions no fade consumed
    int32_t tol = 0;  // a select, not tols.t[q]: a dynamic index would copy the array to local memory
#pragma unroll
    for (int r = 0; r < PSD_SWEEP_MAX_TOLERANCES; ++r)
        if (r == q) tol = tols.t[r];
    int64_t matched = 0, offset_sum = 0;
    for (int32_t d = 0; d <= tol; ++d) {
        for (int32_t i = 0; i < np; ++i) {
            if (used_p[i >> 5] & (1u << (i & 31))) continue;
            const int64_t v = pred(i);
            int32_t j = find_frame(gt, n_gt, v - d);
            if (j < 0 || (used_g[j >> 5] & (1u << (j & 31)))) {
                j = d ? find_frame(gt, n_gt, v + d) : -1;
                if (j < 0 || (used_g[j >> 5] & (1u << (j & 31)))) continue;
            }
            bit_test_set(used_g, j);
            bit_test_set(used_p, i);
            ++matched;
            offset_sum += d;
        }
    }
    hard[0] = matched;
    hard[1] = remaining - matched;
    hard[2] = n_gt - matched;
    hard[3] = offset_sum;
    hard[4] = matched;
    if (q == 0) {
        out_fades[(int64_t)k * 3 + 0] = fm;
        out_fades[(int64_t)k * 3 + 1] = ffp;
        out_fades[(int64_t)k * 3 + 2] = n_fades - fm;
    }
}

static inline int32_t words_for(int64_t bits) { return (int32_t)((bits + 31) / 32); }

}  // namespace psd

using namespace psd;

extern "C" int psd_sweep_cuts(const psd_sweep_cell* cells, int32_t n_cells, int64_t n, int64_t first_frame,
                              int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    PSD_REQUIRE(n_cells >= 0 && n >= 0 && cap >= 0, "psd_sweep_cuts: bad args");
    if (n_cells == 0) return PSD_OK;
    PSD_REQUIRE(cells && cuts && count, "psd_sweep_cuts: bad args");
    for (int32_t k = 0; k < n_cells; ++k) {
        const psd_sweep_cell& c = cells[k];
        PSD_REQUIRE(c.kind >= PSD_SWEEP_CONTENT && c.kind <= PSD_SWEEP_HASH, "psd_sweep_cuts: cell %d: unknown kind %d",
                    k, c.kind);
        PSD_REQUIRE(c.metric, "psd_sweep_cuts: cell %d: no metric array", k);
        PSD_REQUIRE(c.mode == 0 || ((c.kind == PSD_SWEEP_CONTENT || c.kind == PSD_SWEEP_THRESHOLD) && c.mode == 1),
                    "psd_sweep_cuts: cell %d: bad mode %d", k, c.mode);
        PSD_REQUIRE(c.kind != PSD_SWEEP_ADAPTIVE || (c.metric2 && c.window >= 1),
                    "psd_sweep_cuts: cell %d: adaptive cells need metric2 and window >= 1", k);
        PSD_REQUIRE(c.add_final_scene == 0 || (c.kind == PSD_SWEEP_THRESHOLD && c.add_final_scene == 1),
                    "psd_sweep_cuts: cell %d: bad add_final_scene", k);
    }
    cudaStream_t s = (cudaStream_t)stream;
    psd_sweep_cell* d_cells = nullptr;
    const size_t bytes = sizeof(psd_sweep_cell) * (size_t)n_cells;
    PSD_CUDA(cudaMallocAsync((void**)&d_cells, bytes, s));
    PSD_CUDA(cudaMemcpyAsync(d_cells, cells, bytes, cudaMemcpyHostToDevice, s));  // pageable: staged before return
    psd_sweep_cuts_kernel<<<(n_cells + 127) / 128, 128, 0, s>>>(d_cells, n_cells, n, first_frame, cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    PSD_CUDA(cudaFreeAsync(d_cells, s));
    return PSD_OK;
}

extern "C" int psd_sweep_eval(int64_t* cuts, const int32_t* count, int32_t n_cells, int32_t cap, int64_t end_frame,
                              const int64_t* gt_cuts, int32_t n_gt, const int64_t* fades, int32_t n_fades,
                              const int32_t* tolerances, int32_t n_tol, void* workspace, size_t workspace_bytes,
                              int32_t* out_n_pred, int64_t* out_hard, int64_t* out_fades, void* stream) {
    PSD_REQUIRE(n_cells >= 0 && cap >= 0 && n_gt >= 0 && n_fades >= 0, "psd_sweep_eval: bad args");
    PSD_REQUIRE(tolerances && n_tol >= 1 && n_tol <= PSD_SWEEP_MAX_TOLERANCES,
                "psd_sweep_eval: 1 to %d tolerances", PSD_SWEEP_MAX_TOLERANCES);
    Tolerances tols{};
    for (int32_t q = 0; q < n_tol; ++q) {
        PSD_REQUIRE(tolerances[q] >= 0, "psd_sweep_eval: tolerance %d is negative", tolerances[q]);
        tols.t[q] = tolerances[q];
    }
    if (n_cells == 0) return PSD_OK;
    PSD_REQUIRE(cuts && count && out_n_pred && out_hard && out_fades, "psd_sweep_eval: bad args");
    PSD_REQUIRE(n_gt == 0 || gt_cuts, "psd_sweep_eval: gt_cuts is NULL");
    PSD_REQUIRE(n_fades == 0 || fades, "psd_sweep_eval: fades is NULL");
    const int32_t wp = words_for((int64_t)cap + 1), wg = words_for(n_gt), wf = words_for(n_fades);
    const int64_t threads = (int64_t)n_cells * n_tol;
    const size_t need = (size_t)threads * 4u * (size_t)(wp + wg + wf);
    PSD_REQUIRE(workspace && workspace_bytes >= need, "psd_sweep_eval: workspace needs %zu bytes", need);
    cudaStream_t s = (cudaStream_t)stream;
    psd_sweep_pred_kernel<<<(n_cells + 127) / 128, 128, 0, s>>>(cuts, count, n_cells, cap, out_n_pred);
    PSD_CHECK_LAUNCH();
    psd_sweep_eval_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
        cuts, out_n_pred, n_cells, cap, end_frame, gt_cuts, n_gt, fades, n_fades, tols, n_tol,
        (uint32_t*)workspace, wp, wg, wf, out_hard, out_fades);
    PSD_CHECK_LAUNCH();
    count_launch(2);
    return PSD_OK;
}
