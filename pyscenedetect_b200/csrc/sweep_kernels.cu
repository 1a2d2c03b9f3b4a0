// Parameter sweep on the device: every cell of a detector-parameter grid over one scored video.
//   psd_sweep_cuts   benchmark/sweep.py:142-187 (one SceneManager + detector per cell): one thread per
//                    cell runs the cell's automaton (cut_automata.cuh) over the metric arrays the existing
//                    psd_scan_* produced.  The host sorts cells by metric array, so a warp's 32 cells load
//                    each frame's value together (one broadcast load per warp) and take the same branch
//                    most of the time: they only diverge on the frames where some of them cut.
//   psd_sweep_eval   benchmark/evaluator.py:227-331 (score_video) per (cell, tolerance): first the
//                    predicted list of sweep.py:169, then fade matching, then greedy hard-cut matching
//                    (sweep_eval.cuh, shared with psd_clip_eval).
// The automata are sequential walks, so the sweep is bounded by one thread's latency per frame (a load, a
// compare, a few integer ops): G cells cost about as much as one cell until the cells fill the GPU.
#include "cut_automata.cuh"
#include "sweep_eval.cuh"

namespace psd {

__global__ void __launch_bounds__(128) psd_sweep_cuts_kernel(const psd_sweep_cell* __restrict__ cells,
                                                             int32_t n_cells, int64_t n, int64_t first_frame,
                                                             int64_t* __restrict__ cuts,
                                                             int32_t* __restrict__ count, int32_t cap) {
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_cells) return;
    const psd_sweep_cell c = cells[k];
    CutSink out{cuts + (int64_t)k * cap, cap, 0};
    run_cell(c, 0, n, first_frame, 1, first_frame + n - 1, c.min_frames, out);
    count[k] = out.n;
}

// Cell k's cut slice -> the predicted list of sweep.py:169, in place: sorted(set(cuts)), then end_frame
// when there is a cut.  The end is not stored (the slice may be full): entry n_pred - 1 is end_frame.
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
    const int32_t u = sort_unique(cuts + (int64_t)k * cap, c);
    n_pred[k] = u ? u + 1 : 0;
}

// One thread per (cell, tolerance): score_predictions (sweep_eval.cuh) on the cell's predicted list.
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
    uint32_t* used_p = workspace + tid * (int64_t)(words_p + words_g + words_f);
    for (int32_t w = 0; w < words_p + words_g + words_f; ++w) used_p[w] = 0u;
    score_predictions(cuts + (int64_t)k * cap, np, end_frame, gt, n_gt, fades, n_fades, tolerance_at(tols, q), used_p,
                      used_p + words_p, used_p + words_p + words_g, hard,
                      q == 0 ? out_fades + (int64_t)k * 3 : nullptr);
}

int validate_sweep_cells(const psd_sweep_cell* cells, int32_t n_cells, const char* who) {
    PSD_REQUIRE(n_cells == 0 || cells, "%s: no cells", who);
    for (int32_t k = 0; k < n_cells; ++k) {
        const psd_sweep_cell& c = cells[k];
        PSD_REQUIRE(c.kind >= PSD_SWEEP_CONTENT && c.kind <= PSD_SWEEP_HASH, "%s: cell %d: unknown kind %d", who, k,
                    c.kind);
        PSD_REQUIRE(c.metric, "%s: cell %d: no metric array", who, k);
        PSD_REQUIRE(c.mode == 0 || ((c.kind == PSD_SWEEP_CONTENT || c.kind == PSD_SWEEP_THRESHOLD) && c.mode == 1),
                    "%s: cell %d: bad mode %d", who, k, c.mode);
        PSD_REQUIRE(c.kind != PSD_SWEEP_ADAPTIVE || (c.metric2 && c.window >= 1),
                    "%s: cell %d: adaptive cells need metric2 and window >= 1", who, k);
        PSD_REQUIRE(c.add_final_scene == 0 || (c.kind == PSD_SWEEP_THRESHOLD && c.add_final_scene == 1),
                    "%s: cell %d: bad add_final_scene", who, k);
    }
    return PSD_OK;
}

}  // namespace psd

using namespace psd;

extern "C" int psd_sweep_cuts(const psd_sweep_cell* cells, int32_t n_cells, int64_t n, int64_t first_frame,
                              int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    PSD_REQUIRE(n_cells >= 0 && n >= 0 && cap >= 0, "psd_sweep_cuts: bad args");
    if (n_cells == 0) return PSD_OK;
    PSD_REQUIRE(cells && cuts && count, "psd_sweep_cuts: bad args");
    const int rc = validate_sweep_cells(cells, n_cells, "psd_sweep_cuts");
    if (rc != PSD_OK) return rc;
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
    const int32_t wp = (int32_t)words_for((int64_t)cap + 1), wg = (int32_t)words_for(n_gt);
    const int32_t wf = (int32_t)words_for(n_fades);
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
