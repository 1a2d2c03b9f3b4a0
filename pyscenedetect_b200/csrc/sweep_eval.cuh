// Scoring of predicted lists against a video's ground truth as device functions: one thread turns one cut list into
// the predicted list of benchmark/sweep.py:169, and one thread scores one (list, tolerance) as
// benchmark/evaluator.py:227-331 (score_video) does.  psd_sweep_eval (sweep_kernels.cu, one list per grid cell) and
// psd_clip_eval (clip_kernels.cu, one list per (cell, clip)) both call these, so the matcher exists once.
#pragma once

#include "psd_common.cuh"

namespace psd {

struct Tolerances {
    int32_t t[PSD_SWEEP_MAX_TOLERANCES];
};

// tols.t[q] as a select: a dynamic index would copy the array to local memory
__device__ __forceinline__ int32_t tolerance_at(const Tolerances& tols, int32_t q) {
    int32_t tol = 0;
#pragma unroll
    for (int r = 0; r < PSD_SWEEP_MAX_TOLERANCES; ++r)
        if (r == q) tol = tols.t[r];
    return tol;
}

__host__ __device__ __forceinline__ int64_t words_for(int64_t bits) { return (bits + 31) / 32; }

// p[0, c) -> sorted(set(p)) in place; returns how many remain.  Insertion sort is linear on the strictly increasing
// lists every automaton but a |fade_bias| > 1 ThresholdDetector emits (cut_automata.cuh).
__device__ __forceinline__ int32_t sort_unique(int64_t* __restrict__ p, int32_t c) {
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
    return u;
}

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

// One predicted list of np entries (p[0, np - 1) then end_frame) scored at tolerance `tol` against strictly
// increasing hard cuts gt[n_gt] and inclusive fade intervals fades[n_fades][2].  used_p / used_g / used_f are this
// thread's matching bitmaps of np / n_gt / n_fades bits, cleared by the caller (psd_sweep_eval_kernel clears its
// three adjacent bitmaps in one loop, which keeps it free of spills).  hard[5] = matched, false_positives, missed,
// offset_sum, offset_count; fade_counts[3] = matched, false_positives, missed, written when not NULL.
// Hard-cut matching (evaluator.py:227-266) claims (d, i, j) pairs in sorted order.  With strictly increasing ground
// truth a prediction p_i has at most two partners at distance d, g = p_i - d before g = p_i + d in j order, so the
// sorted walk is: for d = 0..tol, for i in order, claim (i, p_i - d) else (i, p_i + d) if both sides are unused.  No
// candidate list is built.
__device__ __forceinline__ void score_predictions(const int64_t* __restrict__ p, int32_t np, int64_t end_frame,
                                                  const int64_t* __restrict__ gt, int32_t n_gt,
                                                  const int64_t* __restrict__ fades, int32_t n_fades, int32_t tol,
                                                  uint32_t* used_p, uint32_t* used_g, uint32_t* used_f,
                                                  int64_t* __restrict__ hard, int64_t* __restrict__ fade_counts) {
    auto pred = [&](int32_t i) { return i < np - 1 ? p[i] : end_frame; };

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
    if (fade_counts) {
        fade_counts[0] = fm;
        fade_counts[1] = ffp;
        fade_counts[2] = n_fades - fm;
    }
}

}  // namespace psd
