// Many clips scored back to back into one engine (clips.py).  The fused pass scores a frame from that frame and
// its predecessor only, so the integer results of the concatenated stream are each clip's own except at the clip
// edges, where a frame was diffed against the previous clip's last frame.  Two kernels finish the job:
//   psd_clip_fill    after a psd_scan_* over the whole pass, sets the metric entries at every clip's head and tail
//                    to what a one-clip engine's scan writes there, bit for bit (0.0 for content_val, the scan's
//                    NaN for an incomplete adaptive window or a frame without a predecessor)
//   psd_clip_cuts    one thread per (cell, clip) runs the cell's automaton (cut_automata.cuh) over the clip's slice
//                    of the metric arrays, with the clip's first frame number and min_frames: a counting pass, an
//                    exclusive scan of the counts, then a writing pass into one compact cut array.
//                    psd_clip_cuts_step runs the same kernels on clips read with a frame skip: slice element i is
//                    frame first + i * step, and post_process sees each clip's end position; psd_clip_cuts_steps
//                    gives each clip its own step (clips read with different frame skips); psd_clip_cuts_tables
//                    gives each cell its own clip table (one per setting of a sweep over settings), and the other
//                    three are its one-table calls; psd_clip_cuts_tables_steps gives each (table, clip) its own step
//   psd_clip_eval    the counterpart of psd_sweep_eval for psd_clip_cuts' compact output: every (cell, clip) list
//                    turned in place into its predicted list, every (cell, clip, tolerance) scored against clip j's
//                    ground truth with score_predictions (sweep_eval.cuh), and the counts summed over the clips;
//                    psd_clip_eval_tables ends each cell's lists at the end frames of the cell's clip table
//   psd_clip_union   the cut list of a cell that is a set of detectors (SceneManager.get_cut_list over several
//                    detectors): one thread per (list, clip) sorts psd_clip_cuts' list in place, one thread per
//                    (cell, clip) counts the merged unique length of its member lists, an exclusive scan, then a
//                    writing pass emits the strictly increasing union into one compact array
//   psd_clip_stats_csv  every clip's StatsManager CSV rows (stats_csv.cuh formats them): one thread per frame counts
//                    its row's bytes, an exclusive scan gives the row offsets, and the writing pass prints each row in
//                    place, so one download carries every clip's text
// Each is one launch (three for psd_clip_cuts, psd_clip_eval and psd_clip_stats_csv, three and one for the counting and
// the writing call of psd_clip_union) per pass whatever the number of cells and clips.
#include <math_constants.h>

#include <cstddef>

#include "cut_automata.cuh"
#include "stats_csv.cuh"
#include "sweep_eval.cuh"

namespace psd {

// A psd_clip_table as the kernels read it, under a name of this namespace: every symbol that starts psd_clip_ is then
// a clip_kernels.cu kernel or entry, never a parameter type.
// The last field is a psd_clip_table's frame_step, or a psd_clip_steps_table's per-clip steps: every table of a call is
// one kind or the other.
struct ClipTable {
    const int64_t* offsets;
    const int64_t* first_frame;
    const int64_t* end_frame;
    union {
        int64_t frame_step;
        const int64_t* frame_steps;
    };
};
static_assert(sizeof(ClipTable) == sizeof(psd_clip_table) && offsetof(ClipTable, end_frame) ==
                  offsetof(psd_clip_table, end_frame) && offsetof(ClipTable, frame_step) ==
                  offsetof(psd_clip_table, frame_step), "ClipTable must be laid out as psd_clip_table");
static_assert(sizeof(ClipTable) == sizeof(psd_clip_steps_table) && offsetof(ClipTable, end_frame) ==
                  offsetof(psd_clip_steps_table, end_frame) && offsetof(ClipTable, frame_steps) ==
                  offsetof(psd_clip_steps_table, frame_step), "ClipTable must be laid out as psd_clip_steps_table");

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
// exceeds cap.  t = cell * n_clips + clip, so one cell's clips are adjacent threads.  Cell k reads clip table
// tables[cell_table[k]] (tables[0] when cell_table is NULL): element i of clip j is frame first_frame[j] + i * step,
// step being the table's frame_steps[j] when clip_steps is set, else its frame_step; post_process's position is
// end_frame[j] - 1, or the last element's frame when end_frame is NULL.
template <bool WRITE>
__global__ void __launch_bounds__(128) psd_clip_cuts_kernel(const psd_sweep_cell* __restrict__ cells, int32_t n_cells,
                                                            const ClipTable* __restrict__ tables,
                                                            const int32_t* __restrict__ cell_table,
                                                            int clip_steps, int32_t n_clips,
                                                            const int64_t* __restrict__ min_frames,
                                                            int64_t* __restrict__ cuts, int64_t cap,
                                                            int64_t* __restrict__ cut_offsets) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t m = (int64_t)n_cells * n_clips;
    if (t >= m) return;
    const int64_t k = t / n_clips, j = t % n_clips;
    const ClipTable tb = tables[cell_table ? cell_table[k] : 0];
    const int64_t b = max(tb.offsets[j], (int64_t)0), e = max(tb.offsets[j + 1], b);
    CutSink out{nullptr, 0, 0};  // cap 0: counts only
    if (WRITE) {
        if (cut_offsets[m] > cap) return;
        const int64_t o = cut_offsets[t];
        out.cuts = cuts + o;
        out.cap = (int32_t)(cut_offsets[t + 1] - o);
    }
    const int64_t first = tb.first_frame[j], step = clip_steps ? tb.frame_steps[j] : tb.frame_step;
    const int64_t last = tb.end_frame ? tb.end_frame[j] - 1 : first + (e - b - 1) * step;
    run_cell(cells[k], b, e - b, first, step, last, min_frames[t], out);
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

// One thread per (cell k, clip j, tolerance q), tid = (k * n_clips + j) * n_tol + q; clip j ends at end_frame[j] of
// cell k's clip table (as in psd_clip_cuts_kernel).  The matching bitmaps are laid
// out so that their offsets follow from the CSR offsets alone: list t's bits start at word t + floor(o_t / 32) of
// tolerance q's block of words_p, clip j's ground-truth bits at word j + floor(gb_j / 32) of the (k, q) block of
// words_g (likewise the fades).  Segment t needs floor(c_t / 32) + 1 words, and t + 1 starts at least that far on.
__global__ void __launch_bounds__(128) clip_eval_kernel(
    const int64_t* __restrict__ cuts, const int64_t* __restrict__ cut_offsets, const int32_t* __restrict__ n_pred,
    int32_t n_cells, int32_t n_clips, int64_t cuts_total, const ClipTable* __restrict__ tables,
    const int32_t* __restrict__ cell_table, const int64_t* __restrict__ gt_offsets, const int64_t* __restrict__ gt,
    int32_t n_gt,
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
    const int64_t end_frame = tables[cell_table ? cell_table[k] : 0].end_frame[j];
    score_predictions(cuts + b, np, end_frame, gt + gb, (int32_t)(ge - gb), fades + 2 * fb, (int32_t)(fe - fb),
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

// One thread per (list, clip) t of psd_clip_cuts' output: the list sorted and de-duplicated in place (linear on the
// strictly increasing lists of every automaton but a |fade_bias| > 1 ThresholdDetector), unique[t] its new length.
// Many cells share one list, so this is the only writer of the lists.  A list longer than max_cuts is left as it is,
// counts as empty, and the lowest such t goes to *over.
__global__ void __launch_bounds__(128) clip_union_sort_kernel(int64_t* __restrict__ cuts,
                                                              const int64_t* __restrict__ cut_offsets, int64_t m,
                                                              int64_t cuts_total, int64_t max_cuts,
                                                              int32_t* __restrict__ unique,
                                                              unsigned long long* __restrict__ over) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    int64_t b, e;
    segment(cut_offsets, t, cuts_total, b, e);
    if (e - b > max_cuts) {
        unique[t] = 0;
        atomicMin(over, (unsigned long long)t);
        return;
    }
    unique[t] = sort_unique(cuts + b, (int32_t)(e - b));
}

// The first entry greater than v of the strictly increasing p[0, n), or INT64_MAX when there is none.
__device__ __forceinline__ int64_t first_above(const int64_t* __restrict__ p, int32_t n, int64_t v) {
    int32_t lo = 0, hi = n;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (p[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo < n ? p[lo] : INT64_MAX;
}

// One thread per (cell k, clip j), t = k * n_clips + j: the union of the lists cell_lists[cell_offsets[k] ..
// cell_offsets[k + 1]) on clip j, walked in increasing order with no cursor array: each next value is the least
// first_above(previous) over the member lists (a binary search in each).  Counting pass (WRITE = false):
// out_offsets[t] = the union's length.  Writing pass: the union at out_cuts[out_offsets[t] ..], after
// psd_clip_scan_kernel turned the lengths into offsets; nothing when the total exceeds out_cap.
template <bool WRITE>
__global__ void __launch_bounds__(128) clip_union_kernel(const int64_t* __restrict__ cuts,
                                                         const int64_t* __restrict__ cut_offsets, int64_t cuts_total,
                                                         const int32_t* __restrict__ unique, int32_t n_clips,
                                                         const int32_t* __restrict__ cell_offsets,
                                                         const int32_t* __restrict__ cell_lists, int32_t n_cells,
                                                         int64_t* __restrict__ out_cuts, int64_t out_cap,
                                                         int64_t* __restrict__ out_offsets) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t m = (int64_t)n_cells * n_clips;
    if (t >= m) return;
    if (WRITE && out_offsets[m] > out_cap) return;
    const int64_t k = t / n_clips, j = t % n_clips;
    const int32_t lb = cell_offsets[k], le = cell_offsets[k + 1];
    int64_t* out = WRITE ? out_cuts + out_offsets[t] : nullptr;
    int64_t n = 0, v = INT64_MIN;
    for (;;) {
        int64_t next = INT64_MAX;
        for (int32_t i = lb; i < le; ++i) {
            const int64_t l = (int64_t)cell_lists[i] * n_clips + j;
            const int64_t b = min(max(cut_offsets[l], (int64_t)0), cuts_total);
            next = min(next, first_above(cuts + b, unique[l], v));
        }
        if (next == INT64_MAX) break;
        if (WRITE) out[n] = next;
        ++n;
        v = next;
    }
    if (!WRITE) out_offsets[t] = n;
}

// The clip that pass frame i belongs to: the last j with offsets[j] <= i (empty clips share their offset with the next
// clip, so this is the clip that holds i).
__device__ __forceinline__ int32_t clip_of(const int64_t* __restrict__ offsets, int32_t n_clips, int64_t i) {
    int32_t lo = 0, hi = n_clips - 1;
    while (lo < hi) {
        const int32_t mid = (lo + hi + 1) >> 1;
        if (offsets[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// A row's cells.  Counting pass (WRITE = false): row_offsets[i] = the bytes of frame i's row (0: no row).  Writing
// pass: the row at out + row_offsets[i], after psd_clip_scan_kernel made them offsets; nothing when the total exceeds
// cap.  The writing pass's threads n .. n + n_clips write the clip byte offsets.
template <bool WRITE>
__global__ void __launch_bounds__(128) stats_rows_kernel(const psd_stats_column* __restrict__ cols, int32_t n_cols,
                                                         const int64_t* __restrict__ offsets,
                                                         const int64_t* __restrict__ first_frame,
                                                         const double* __restrict__ rate, int32_t n_clips, int64_t n,
                                                         int64_t* __restrict__ row_offsets, char* __restrict__ out,
                                                         int64_t cap, int64_t* __restrict__ clip_bytes) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (WRITE && i >= n) {
        if (i <= n + n_clips) clip_bytes[i - n] = row_offsets[min(max(offsets[i - n], (int64_t)0), n)];
        return;
    }
    if (i >= n) return;
    const int32_t j = clip_of(offsets, n_clips, i);
    const int64_t b = offsets[j], local = i - b, len = offsets[j + 1] - b;
    bool row = false;
    for (int32_t c = 0; c < n_cols; ++c) row |= local >= cols[c].head && local < len - cols[c].tail;
    if (WRITE && (!row || row_offsets[n] > cap)) return;
    if (!row) {
        row_offsets[i] = 0;
        return;
    }
    const int64_t frame = first_frame[j] + local;
    const Timecode tc = timecode_of(frame, rate[j]);
    char* p = WRITE ? out + row_offsets[i] : nullptr;
    int64_t bytes = uint_len((uint64_t)frame + 1) + 1 + timecode_len(tc);
    if (WRITE) {
        p = uint_write((uint64_t)frame + 1, p);
        *p++ = ',';
        p = timecode_write(tc, p);
    }
    for (int32_t c = 0; c < n_cols; ++c) {
        const psd_stats_column col = cols[c];
        const bool has = local >= col.head && local < len - col.tail;
        if (has) {
            const Decimal d = f64_decimal(col.values[i * col.stride]);
            bytes += 1 + f64_len(d);
            if (WRITE) {
                *p++ = ',';
                p = f64_write(d, p);
            }
        } else {
            bytes += 5;
            if (WRITE) {
                *p++ = ',';
                put3(p, 'N', 'o', 'n');
                p[3] = 'e';
                p += 4;
            }
        }
    }
    if (WRITE) *p = '\n';
    else row_offsets[i] = bytes + 1;
}

__global__ void __launch_bounds__(128) format_f64_kernel(const double* __restrict__ v, int64_t n, char* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    char* p = out + i * 32;
    const Decimal d = f64_decimal(v[i]);
    const int len = f64_len(d);
    f64_write(d, p);
    for (int k = len; k < 32; ++k) p[k] = 0;
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

// The cells, the clip tables, the clips' steps and the cells' table indices, copied in one device allocation on `s`
// (pageable: staged before return); *d_cells NULL when the copy failed.  clip_step, a HOST int64[n_clips] for one
// table, is copied too, and the copied table steps each clip by it.
static int copy_tables(const psd_sweep_cell* cells, int32_t n_cells, const ClipTable* tables, int32_t n_tables,
                       const int64_t* clip_step, int32_t n_clips, const int32_t* cell_table, cudaStream_t s,
                       psd_sweep_cell** d_cells, ClipTable** d_tables, int32_t** d_cell_table) {
    const size_t cb = sizeof(psd_sweep_cell) * (size_t)(cells ? n_cells : 0);
    const size_t tb = sizeof(ClipTable) * (size_t)n_tables;
    const size_t sb = clip_step ? sizeof(int64_t) * (size_t)n_clips : 0;
    const size_t ib = cell_table ? sizeof(int32_t) * (size_t)n_cells : 0;
    char* d = nullptr;
    *d_cells = nullptr;
    PSD_CUDA(cudaMallocAsync((void**)&d, cb + tb + sb + ib, s));
    if (cb) PSD_CUDA(cudaMemcpyAsync(d, cells, cb, cudaMemcpyHostToDevice, s));
    if (clip_step) {
        ClipTable t = tables[0];
        t.frame_steps = (const int64_t*)(d + cb + tb);
        PSD_CUDA(cudaMemcpyAsync(d + cb, &t, sizeof(t), cudaMemcpyHostToDevice, s));
        if (sb) PSD_CUDA(cudaMemcpyAsync(d + cb + tb, clip_step, sb, cudaMemcpyHostToDevice, s));
    } else {
        PSD_CUDA(cudaMemcpyAsync(d + cb, tables, tb, cudaMemcpyHostToDevice, s));
    }
    if (ib) PSD_CUDA(cudaMemcpyAsync(d + cb + tb + sb, cell_table, ib, cudaMemcpyHostToDevice, s));
    *d_cells = (psd_sweep_cell*)d;
    *d_tables = (ClipTable*)(d + cb);
    *d_cell_table = ib ? (int32_t*)(d + cb + tb + sb) : nullptr;
    return PSD_OK;
}

// Every cell's table index in [0, n_tables).
static int check_tables(const char* name, int32_t n_tables, const int32_t* cell_table, int32_t n_cells) {
    if (cell_table)
        for (int32_t k = 0; k < n_cells; ++k)
            PSD_REQUIRE(cell_table[k] >= 0 && cell_table[k] < n_tables, "%s: cell %d names table %d of %d", name, k,
                        cell_table[k], n_tables);
    return PSD_OK;
}

// Each clip steps by its table's frame_step (clip_step NULL, table_steps false), by a HOST int64[n_clips] clip_step
// (one table), or by its table's DEVICE frame_steps (table_steps true: psd_clip_steps_table).
static int clip_cuts(const char* name, const psd_sweep_cell* cells, int32_t n_cells, const ClipTable* tables,
                     int32_t n_tables, const int32_t* cell_table, const int64_t* clip_step, bool table_steps,
                     int32_t n_clips, const int64_t* min_frames, int64_t* cuts, int64_t cuts_cap,
                     int64_t* cut_offsets, void* stream) {
    PSD_REQUIRE(tables && n_tables >= 1, "%s: no clip table", name);
    for (int32_t i = 0; i < n_tables; ++i) PSD_REQUIRE(tables[i].offsets, "%s: no clip table", name);
    PSD_REQUIRE(n_cells >= 0 && n_clips >= 0 && cuts_cap >= 0, "%s: bad args", name);
    for (int32_t i = 0; i < n_tables; ++i) {
        if (table_steps)
            PSD_REQUIRE(tables[i].frame_steps || n_clips == 0, "%s: table %d has no frame_step array", name, i);
        else
            PSD_REQUIRE(tables[i].frame_step >= 1, "%s: frame_step must be >= 1", name);
    }
    if (clip_step)
        for (int32_t j = 0; j < n_clips; ++j)
            PSD_REQUIRE(clip_step[j] >= 1, "%s: frame_step[%d] is %lld, must be >= 1", name, j,
                        (long long)clip_step[j]);
    PSD_REQUIRE(cut_offsets, "%s: no cut_offsets array", name);
    int rc = check_tables(name, n_tables, cell_table, n_cells);
    if (rc != PSD_OK) return rc;
    rc = validate_sweep_cells(cells, n_cells, name);
    if (rc != PSD_OK) return rc;
    const int64_t m = (int64_t)n_cells * n_clips;
    cudaStream_t s = (cudaStream_t)stream;
    if (m == 0) {
        PSD_CUDA(cudaMemsetAsync(cut_offsets, 0, sizeof(int64_t), s));
        return PSD_OK;
    }
    for (int32_t i = 0; i < n_tables; ++i)
        PSD_REQUIRE(tables[i].first_frame && min_frames, "%s: no clip first frames / min_frames", name);
    PSD_REQUIRE(cuts || cuts_cap == 0, "%s: no cut array", name);
    psd_sweep_cell* d_cells;
    ClipTable* d_tables;
    int32_t* d_cell_table;
    rc = copy_tables(cells, n_cells, tables, n_tables, clip_step, n_clips, cell_table, s, &d_cells, &d_tables,
                     &d_cell_table);
    if (rc != PSD_OK) return rc;
    const int steps = clip_step || table_steps;
    const unsigned blocks = (unsigned)((m + 127) / 128);
    psd_clip_cuts_kernel<false><<<blocks, 128, 0, s>>>(d_cells, n_cells, d_tables, d_cell_table, steps, n_clips,
                                                       min_frames, cuts, cuts_cap, cut_offsets);
    PSD_CHECK_LAUNCH();
    psd_clip_scan_kernel<<<1, 1024, 0, s>>>(cut_offsets, m);
    PSD_CHECK_LAUNCH();
    psd_clip_cuts_kernel<true><<<blocks, 128, 0, s>>>(d_cells, n_cells, d_tables, d_cell_table, steps, n_clips,
                                                      min_frames, cuts, cuts_cap, cut_offsets);
    PSD_CHECK_LAUNCH();
    count_launch(3);
    PSD_CUDA(cudaFreeAsync(d_cells, s));
    return PSD_OK;
}

// A psd_clip_table or psd_clip_steps_table as the kernels read it (the layouts are asserted above).
static const ClipTable* clip_tables(const psd_clip_table* t) { return reinterpret_cast<const ClipTable*>(t); }
static const ClipTable* clip_tables(const psd_clip_steps_table* t) { return reinterpret_cast<const ClipTable*>(t); }

extern "C" int psd_clip_cuts(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                             const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                             int64_t cuts_cap, int64_t* cut_offsets, void* stream) {
    const psd_clip_table table{clip_offsets, clip_first_frame, nullptr, 1};
    return clip_cuts("psd_clip_cuts", cells, n_cells, clip_tables(&table), 1, nullptr, nullptr, false, n_clips,
                     min_frames, cuts, cuts_cap, cut_offsets, stream);
}

extern "C" int psd_clip_cuts_step(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                                  const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames,
                                  int64_t* cuts, int64_t cuts_cap, int64_t* cut_offsets, int64_t frame_step,
                                  const int64_t* clip_end_frame, void* stream) {
    const psd_clip_table table{clip_offsets, clip_first_frame, clip_end_frame, frame_step};
    return clip_cuts("psd_clip_cuts_step", cells, n_cells, clip_tables(&table), 1, nullptr, nullptr, false, n_clips,
                     min_frames, cuts, cuts_cap, cut_offsets, stream);
}

extern "C" int psd_clip_cuts_steps(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                                   const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames,
                                   int64_t* cuts, int64_t cuts_cap, int64_t* cut_offsets, const int64_t* frame_step,
                                   const int64_t* clip_end_frame, void* stream) {
    PSD_REQUIRE(frame_step || n_clips <= 0, "psd_clip_cuts_steps: no frame_step array");
    const psd_clip_table table{clip_offsets, clip_first_frame, clip_end_frame, 1};
    return clip_cuts("psd_clip_cuts_steps", cells, n_cells, clip_tables(&table), 1, nullptr, frame_step, false,
                     n_clips, min_frames, cuts, cuts_cap, cut_offsets, stream);
}

extern "C" int psd_clip_cuts_tables(const psd_sweep_cell* cells, int32_t n_cells, const psd_clip_table* tables,
                                    int32_t n_tables, const int32_t* cell_table, int32_t n_clips,
                                    const int64_t* min_frames, int64_t* cuts, int64_t cuts_cap, int64_t* cut_offsets,
                                    void* stream) {
    return clip_cuts("psd_clip_cuts_tables", cells, n_cells, clip_tables(tables), n_tables, cell_table, nullptr, false,
                     n_clips, min_frames, cuts, cuts_cap, cut_offsets, stream);
}

extern "C" int psd_clip_cuts_tables_steps(const psd_sweep_cell* cells, int32_t n_cells,
                                          const psd_clip_steps_table* tables, int32_t n_tables,
                                          const int32_t* cell_table, int32_t n_clips, const int64_t* min_frames,
                                          int64_t* cuts, int64_t cuts_cap, int64_t* cut_offsets, void* stream) {
    return clip_cuts("psd_clip_cuts_tables_steps", cells, n_cells, clip_tables(tables), n_tables, cell_table, nullptr,
                     true, n_clips, min_frames, cuts, cuts_cap, cut_offsets, stream);
}

static int clip_eval(const char* name, int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips,
                     int64_t cuts_total, int64_t max_cuts, const psd_clip_table* tables, int32_t n_tables,
                     const int32_t* cell_table, const int64_t* gt_offsets, const int64_t* gt_cuts, int32_t n_gt,
                     const int64_t* fade_offsets, const int64_t* fades, int32_t n_fades, const int32_t* tolerances,
                     int32_t n_tol, void* workspace, size_t workspace_bytes, int32_t* out_n_pred, int64_t* out_hard,
                     int64_t* out_fades, int64_t* out_totals_hard, int64_t* out_totals_fades, int64_t* out_over,
                     void* stream) {
    PSD_REQUIRE(n_cells >= 0 && n_clips >= 0 && cuts_total >= 0 && n_gt >= 0 && n_fades >= 0, "%s: bad args", name);
    PSD_REQUIRE(max_cuts >= 0 && max_cuts <= INT32_MAX, "%s: max_cuts must be 0 to %d", name, INT32_MAX);
    PSD_REQUIRE(tolerances && n_tol >= 1 && n_tol <= PSD_SWEEP_MAX_TOLERANCES, "%s: 1 to %d tolerances", name,
                PSD_SWEEP_MAX_TOLERANCES);
    Tolerances tols{};
    for (int32_t q = 0; q < n_tol; ++q) {
        PSD_REQUIRE(tolerances[q] >= 0, "%s: tolerance %d is negative", name, tolerances[q]);
        tols.t[q] = tolerances[q];
    }
    PSD_REQUIRE(out_over, "%s: no out_over", name);
    const int64_t m = (int64_t)n_cells * n_clips;
    PSD_REQUIRE(n_cells == 0 || (out_totals_hard && out_totals_fades), "%s: no totals arrays", name);
    if (m > 0) {
        bool ends = tables && n_tables >= 1;
        for (int32_t i = 0; ends && i < n_tables; ++i) ends = tables[i].end_frame != nullptr;
        PSD_REQUIRE(cut_offsets && ends && gt_offsets && fade_offsets, "%s: no clip tables", name);
        PSD_REQUIRE(cuts || cuts_total == 0, "%s: cuts is NULL", name);
        PSD_REQUIRE(n_gt == 0 || gt_cuts, "%s: gt_cuts is NULL", name);
        PSD_REQUIRE(n_fades == 0 || fades, "%s: fades is NULL", name);
        PSD_REQUIRE(out_n_pred && out_hard && out_fades, "%s: no output arrays", name);
        const int rc = check_tables(name, n_tables, cell_table, n_cells);
        if (rc != PSD_OK) return rc;
    }
    const int64_t wp = m + words_for(cuts_total), wg = n_clips + words_for(n_gt), wf = n_clips + words_for(n_fades);
    const size_t need = 4u * ((size_t)n_tol * (size_t)wp + (size_t)n_cells * (size_t)n_tol * (size_t)(wg + wf));
    PSD_REQUIRE(m == 0 || (workspace && workspace_bytes >= need), "%s: workspace needs %zu bytes", name, need);
    cudaStream_t s = (cudaStream_t)stream;
    PSD_CUDA(cudaMemsetAsync(out_over, 0xFF, sizeof(int64_t), s));  // -1: no list longer than max_cuts
    if (m == 0) {  // no clip: every total is 0
        if (n_cells > 0) {
            PSD_CUDA(cudaMemsetAsync(out_totals_hard, 0, sizeof(int64_t) * 5 * (size_t)n_cells * n_tol, s));
            PSD_CUDA(cudaMemsetAsync(out_totals_fades, 0, sizeof(int64_t) * 3 * (size_t)n_cells, s));
        }
        return PSD_OK;
    }
    psd_sweep_cell* d_alloc;
    ClipTable* d_tables;
    int32_t* d_cell_table;
    int rc = copy_tables(nullptr, n_cells, clip_tables(tables), n_tables, nullptr, n_clips, cell_table, s, &d_alloc,
                         &d_tables, &d_cell_table);
    if (rc != PSD_OK) return rc;
    clip_pred_kernel<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(cuts, cut_offsets, m, cuts_total, max_cuts,
                                                                  out_n_pred, (unsigned long long*)out_over);
    PSD_CHECK_LAUNCH();
    const int64_t threads = m * n_tol;
    clip_eval_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
        cuts, cut_offsets, out_n_pred, n_cells, n_clips, cuts_total, d_tables, d_cell_table, gt_offsets, gt_cuts, n_gt,
        fade_offsets, fades, n_fades, tols, n_tol, (uint32_t*)workspace, wp, wg, wf, out_hard, out_fades);
    PSD_CHECK_LAUNCH();
    const int64_t sums = (int64_t)n_cells * ((int64_t)n_tol * 5 + 3);
    clip_totals_kernel<<<(unsigned)((sums + 255) / 256), 256, 0, s>>>(out_hard, out_fades, n_cells, n_clips, n_tol,
                                                                     out_totals_hard, out_totals_fades);
    PSD_CHECK_LAUNCH();
    count_launch(3);
    PSD_CUDA(cudaFreeAsync(d_alloc, s));
    return PSD_OK;
}

extern "C" int psd_clip_eval(int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips,
                             int64_t cuts_total, int64_t max_cuts, const int64_t* clip_end_frame,
                             const int64_t* gt_offsets, const int64_t* gt_cuts, int32_t n_gt,
                             const int64_t* fade_offsets, const int64_t* fades, int32_t n_fades,
                             const int32_t* tolerances, int32_t n_tol, void* workspace, size_t workspace_bytes,
                             int32_t* out_n_pred, int64_t* out_hard, int64_t* out_fades, int64_t* out_totals_hard,
                             int64_t* out_totals_fades, int64_t* out_over, void* stream) {
    const psd_clip_table table{nullptr, nullptr, clip_end_frame, 1};
    return clip_eval("psd_clip_eval", cuts, cut_offsets, n_cells, n_clips, cuts_total, max_cuts, &table, 1, nullptr,
                     gt_offsets, gt_cuts, n_gt, fade_offsets, fades, n_fades, tolerances, n_tol, workspace,
                     workspace_bytes, out_n_pred, out_hard, out_fades, out_totals_hard, out_totals_fades, out_over,
                     stream);
}

extern "C" int psd_clip_eval_tables(int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips,
                                    int64_t cuts_total, int64_t max_cuts, const psd_clip_table* tables,
                                    int32_t n_tables, const int32_t* cell_table, const int64_t* gt_offsets,
                                    const int64_t* gt_cuts, int32_t n_gt, const int64_t* fade_offsets,
                                    const int64_t* fades, int32_t n_fades, const int32_t* tolerances, int32_t n_tol,
                                    void* workspace, size_t workspace_bytes, int32_t* out_n_pred, int64_t* out_hard,
                                    int64_t* out_fades, int64_t* out_totals_hard, int64_t* out_totals_fades,
                                    int64_t* out_over, void* stream) {
    return clip_eval("psd_clip_eval_tables", cuts, cut_offsets, n_cells, n_clips, cuts_total, max_cuts, tables,
                     n_tables, cell_table, gt_offsets, gt_cuts, n_gt, fade_offsets, fades, n_fades, tolerances, n_tol,
                     workspace, workspace_bytes, out_n_pred, out_hard, out_fades, out_totals_hard, out_totals_fades,
                     out_over, stream);
}

extern "C" int psd_clip_union(int64_t* cuts, const int64_t* cut_offsets, int32_t n_lists, int32_t n_clips,
                              int64_t cuts_total, int64_t max_cuts, const int32_t* cell_offsets,
                              const int32_t* cell_lists, int32_t n_cells, int32_t* unique, int64_t* out_cuts,
                              int64_t out_cap, int64_t* out_offsets, int64_t* out_over, void* stream) {
    PSD_REQUIRE(n_lists >= 0 && n_clips >= 0 && n_cells >= 0 && cuts_total >= 0 && out_cap >= 0,
                "psd_clip_union: bad args");
    PSD_REQUIRE(max_cuts >= 0 && max_cuts <= INT32_MAX, "psd_clip_union: max_cuts must be 0 to %d", INT32_MAX);
    PSD_REQUIRE(cell_offsets && out_offsets && out_over, "psd_clip_union: no cell table / out_offsets / out_over");
    PSD_REQUIRE(cell_offsets[0] == 0, "psd_clip_union: cell_offsets[0] is %d, not 0", cell_offsets[0]);
    for (int32_t k = 0; k < n_cells; ++k) {
        const int64_t n = (int64_t)cell_offsets[k + 1] - cell_offsets[k];
        PSD_REQUIRE(n >= 1 && n <= PSD_SWEEP_MAX_MEMBERS, "psd_clip_union: cell %d has %lld lists, not 1 to %d", k,
                    (long long)n, PSD_SWEEP_MAX_MEMBERS);
        PSD_REQUIRE(cell_lists, "psd_clip_union: no cell_lists");
        for (int32_t i = cell_offsets[k]; i < cell_offsets[k + 1]; ++i)
            PSD_REQUIRE(cell_lists[i] >= 0 && cell_lists[i] < n_lists, "psd_clip_union: cell %d names list %d of %d",
                        k, cell_lists[i], n_lists);
    }
    PSD_REQUIRE(out_cuts || out_cap == 0, "psd_clip_union: no out_cuts array");
    const int64_t m = (int64_t)n_cells * n_clips, lists = (int64_t)n_lists * n_clips;
    PSD_REQUIRE(m == 0 || (cut_offsets && (cuts || cuts_total == 0)), "psd_clip_union: no cuts / cut_offsets");
    PSD_REQUIRE(m == 0 || unique, "psd_clip_union: no unique workspace");
    const bool write = out_cuts != nullptr;
    cudaStream_t s = (cudaStream_t)stream;
    if (!write) PSD_CUDA(cudaMemsetAsync(out_over, 0xFF, sizeof(int64_t), s));  // -1: no list longer than max_cuts
    if (m == 0) {
        if (!write) PSD_CUDA(cudaMemsetAsync(out_offsets, 0, sizeof(int64_t), s));
        return PSD_OK;
    }
    // the cell table in one allocation (pageable: staged before return)
    const size_t tb = sizeof(int32_t) * ((size_t)n_cells + 1 + (size_t)cell_offsets[n_cells]);
    int32_t* d = nullptr;
    PSD_CUDA(cudaMallocAsync((void**)&d, tb, s));
    PSD_CUDA(cudaMemcpyAsync(d, cell_offsets, sizeof(int32_t) * ((size_t)n_cells + 1), cudaMemcpyHostToDevice, s));
    PSD_CUDA(cudaMemcpyAsync(d + n_cells + 1, cell_lists, sizeof(int32_t) * (size_t)cell_offsets[n_cells],
                             cudaMemcpyHostToDevice, s));
    const int32_t* d_lists = d + n_cells + 1;
    const unsigned blocks = (unsigned)((m + 127) / 128);
    if (!write) {  // sort every list in place, count every union, scan the counts
        clip_union_sort_kernel<<<(unsigned)((lists + 127) / 128), 128, 0, s>>>(cuts, cut_offsets, lists, cuts_total,
                                                                              max_cuts, unique,
                                                                              (unsigned long long*)out_over);
        PSD_CHECK_LAUNCH();
        clip_union_kernel<false><<<blocks, 128, 0, s>>>(cuts, cut_offsets, cuts_total, unique, n_clips, d, d_lists,
                                                        n_cells, nullptr, 0, out_offsets);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(out_offsets, m);
        PSD_CHECK_LAUNCH();
        count_launch(3);
    } else {  // the unions, from what the counting call left in the lists, `unique` and out_offsets
        clip_union_kernel<true><<<blocks, 128, 0, s>>>(cuts, cut_offsets, cuts_total, unique, n_clips, d, d_lists,
                                                       n_cells, out_cuts, out_cap, out_offsets);
        PSD_CHECK_LAUNCH();
        count_launch();
    }
    PSD_CUDA(cudaFreeAsync(d, s));
    return PSD_OK;
}

extern "C" int psd_clip_stats_csv(const psd_stats_column* columns, int32_t n_columns, const int64_t* clip_offsets,
                                  const int64_t* clip_first_frame, const double* clip_rate, int32_t n_clips, int64_t n,
                                  int64_t* row_offsets, char* out, int64_t out_cap, int64_t* clip_bytes,
                                  void* stream) {
    PSD_REQUIRE(clip_offsets && clip_bytes, "psd_clip_stats_csv: no clip table / clip_bytes");
    PSD_REQUIRE(n >= 0 && n_clips >= 0 && out_cap >= 0, "psd_clip_stats_csv: bad args");
    PSD_REQUIRE(columns && n_columns >= 1 && n_columns <= PSD_STATS_MAX_COLUMNS,
                "psd_clip_stats_csv: 1 to %d columns", PSD_STATS_MAX_COLUMNS);
    for (int32_t c = 0; c < n_columns; ++c)
        PSD_REQUIRE(columns[c].values && columns[c].stride >= 1 && columns[c].head >= 0 && columns[c].tail >= 0,
                    "psd_clip_stats_csv: column %d: no values, or a stride < 1, or a negative head / tail", c);
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0 || n_clips == 0) {
        PSD_CUDA(cudaMemsetAsync(clip_bytes, 0, sizeof(int64_t) * ((size_t)n_clips + 1), s));
        return PSD_OK;
    }
    PSD_REQUIRE(clip_first_frame && clip_rate && row_offsets, "psd_clip_stats_csv: no first frames / rates / row_offsets");
    PSD_REQUIRE(out || out_cap == 0, "psd_clip_stats_csv: no output buffer");
    psd_stats_column* d_cols = nullptr;
    const size_t bytes = sizeof(psd_stats_column) * (size_t)n_columns;
    PSD_CUDA(cudaMallocAsync((void**)&d_cols, bytes, s));
    PSD_CUDA(cudaMemcpyAsync(d_cols, columns, bytes, cudaMemcpyHostToDevice, s));  // pageable: staged before return
    stats_rows_kernel<false><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(
        d_cols, n_columns, clip_offsets, clip_first_frame, clip_rate, n_clips, n, row_offsets, out, out_cap, clip_bytes);
    PSD_CHECK_LAUNCH();
    psd_clip_scan_kernel<<<1, 1024, 0, s>>>(row_offsets, n);
    PSD_CHECK_LAUNCH();
    const int64_t threads = n + n_clips + 1;
    stats_rows_kernel<true><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
        d_cols, n_columns, clip_offsets, clip_first_frame, clip_rate, n_clips, n, row_offsets, out, out_cap, clip_bytes);
    PSD_CHECK_LAUNCH();
    count_launch(3);
    PSD_CUDA(cudaFreeAsync(d_cols, s));
    return PSD_OK;
}

extern "C" int psd_test_format_f64(int device, const double* values_host, int64_t n, char* text_out) {
    PSD_REQUIRE(n >= 0 && (n == 0 || (values_host && text_out)), "psd_test_format_f64: bad args");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(device));
    double* d_v = nullptr;
    char* d_text = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_v, sizeof(double) * (size_t)n);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_text, 32 * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_v, values_host, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        format_f64_kernel<<<(unsigned)((n + 127) / 128), 128>>>(d_v, n, d_text);
        e = cudaGetLastError();
        count_launch();
    }
    if (e == cudaSuccess) e = cudaMemcpy(text_out, d_text, 32 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaFree(d_v);
    cudaFree(d_text);
    PSD_CUDA(e);
    return PSD_OK;
}
