// The five cut state machines as device functions: one thread walks one cell's frame sequence.  The
// single-cell kernels of cut_kernels.cu (psd_cuts_*) and the batched kernel of sweep_kernels.cu
// (psd_sweep_cuts, one thread per grid cell) both call these, so each automaton exists once.
//   flash_filter_cuts   detector.py:160-224   (FlashFilter MERGE / SUPPRESS over `above(i)`)
//   adaptive_cuts       adaptive_detector.py:134-143
//   histogram_cuts      histogram_detector.py:87-112
//   hash_cuts           hash_detector.py:79-109
//   threshold_cuts      threshold_detector.py:113-168, 170-191
// Every automaton emits strictly increasing frames except threshold_cuts with |fade_bias| > 1 (its cut
// is fade_frame + round((t - fade_frame) * (1 + bias) / 2), which then leaves [fade_frame, t]);
// psd_sweep_eval therefore sorts and de-duplicates each cell's list itself.
#pragma once

#include "psd_common.cuh"

namespace psd {

// A cell's cut list: the count lives in a register and is stored once at the end.
struct CutSink {
    int64_t* cuts;
    int32_t cap;
    int32_t n;
    __device__ __forceinline__ void push(int64_t frame) {
        if (n < cap) cuts[n] = frame;
        ++n;
    }
};

template <class Above>
__device__ __forceinline__ void flash_filter_cuts(Above above, int64_t n, int64_t first_frame, int64_t min_frames,
                                                  int mode, CutSink& out) {
    if (min_frames <= 0) {  // filter disabled: every above-threshold frame is a cut (detector.py:161-162)
        for (int64_t i = 0; i < n; ++i)
            if (above(i)) out.push(first_frame + i);
        return;
    }
    int64_t last_above = first_frame;  // initialised to the first frame seen (detector.py:163-164)
    bool merge_enabled = false, merge_triggered = false;
    int64_t merge_start = 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t t = first_frame + i;
        const bool a = above(i);
        const bool met = (t - last_above) >= min_frames;
        if (mode == 1) {  // SUPPRESS (detector.py:171-187)
            if (a && met) {
                last_above = t;
                out.push(t);
            }
            continue;
        }
        if (a) last_above = t;  // MERGE (detector.py:189-224)
        if (merge_triggered) {
            if (met && !a && (last_above - merge_start) >= min_frames) {
                merge_triggered = false;
                out.push(last_above);
            }
            continue;
        }
        if (!a) continue;
        if (met) {
            merge_enabled = true;
            out.push(t);
        } else if (merge_enabled) {
            merge_triggered = true;
            merge_start = t;
        }
    }
}

__device__ __forceinline__ void adaptive_cuts(const double* __restrict__ ratio, const double* __restrict__ score,
                                              int64_t n, int64_t first_frame, int window, double adaptive_threshold,
                                              double min_content_val, int64_t min_frames, CutSink& out) {
    int64_t last_cut = first_frame;  // adaptive_detector.py:108-109
    for (int64_t i = window; i + window < n; ++i) {  // target i is decided when frame i+w arrives
        const bool met = ratio[i] >= adaptive_threshold && score[i] >= min_content_val;
        const int64_t current = first_frame + i + window;
        if (met && (current - last_cut) >= min_frames) {
            last_cut = first_frame + i;
            out.push(first_frame + i);
        }
    }
}

__device__ __forceinline__ void histogram_cuts(const double* __restrict__ correl, int64_t n, int64_t first_frame,
                                               double threshold, int64_t min_frames, CutSink& out) {
    int64_t last_cut = first_frame;  // histogram_detector.py:87-88 (a FrameTimecode is always truthy)
    for (int64_t i = 1; i < n; ++i) {    // frame 0 has nothing to compare with
        const int64_t t = first_frame + i;
        if (correl[i] <= threshold && (t - last_cut) >= min_frames) {
            out.push(t);
            last_cut = t;
        }
    }
}

__device__ __forceinline__ void hash_cuts(const double* __restrict__ dist, int64_t n, int64_t first_frame,
                                          double threshold, int64_t min_frames, CutSink& out) {
    int64_t last_cut = first_frame;  // hash_detector.py:79-80
    for (int64_t i = 0; i < n; ++i) {
        const double d = dist[i];
        if (d != d) continue;         // NaN: no predecessor frame (hash_detector.py:83)
        const int64_t t = first_frame + i;
        if (d >= threshold && (t - last_cut) >= min_frames) {
            out.push(t);
            last_cut = t;
        }
    }
}

__device__ __forceinline__ void threshold_cuts(const double* __restrict__ avg, int64_t n, int64_t first_frame,
                                               double threshold, int method_ceiling, double fade_bias,
                                               int64_t min_frames, int add_final_scene, CutSink& out) {
    if (n <= 0) return;
    int64_t last_scene_cut = first_frame, fade_frame = first_frame;
    bool fade_in = !(avg[0] < threshold);  // first frame: 'out' iff avg < threshold (any method)
    for (int64_t i = 1; i < n; ++i) {
        const int64_t t = first_frame + i;
        const double v = avg[i];
        const bool below = method_ceiling ? (v >= threshold) : (v < threshold);  // "faded out" condition
        if (fade_in && below) {
            fade_in = false;
            fade_frame = t;
        } else if (!fade_in && !below) {
            if ((t - last_scene_cut) >= min_frames) {
                const double half = __dmul_rn((double)(t - fade_frame), __dadd_rn(1.0, fade_bias)) / 2.0;
                out.push(fade_frame + (int64_t)rint(half));  // Python round(): half to even
                last_scene_cut = t;
            }
            fade_in = true;
            fade_frame = t;
        }
    }
    // post_process (threshold_detector.py:170-191) with timecode = last frame
    const int64_t last = first_frame + n - 1;
    if (!fade_in && add_final_scene && (last - last_scene_cut) >= min_frames) out.push(fade_frame);
}

}  // namespace psd
