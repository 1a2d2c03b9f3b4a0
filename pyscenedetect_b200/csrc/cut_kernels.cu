// Cut state machines as trailing device scans (SURVEY.md §8(f) N2): the O(N) per-frame logic the
// detectors run in Python, restated on frame NUMBERS for constant-frame-rate input (the host turns
// every `min_scene_len` form into a frame count with FrameTimecode's own rounding rule,
// common.py:480-486,627-638).  One thread walks the sequence: these are strictly sequential
// automata over a few bytes per frame; at 100k frames they take ~1 ms and keep the cut list on the
// device next to the scores.  The automata themselves are the device functions of cut_automata.cuh,
// which psd_sweep_cuts (sweep_kernels.cu) runs once per grid cell.
//   psd_cuts_flash_filter   detector.py:160-224   (FlashFilter MERGE / SUPPRESS over score >= threshold)
//   psd_cuts_adaptive       adaptive_detector.py:134-143
//   psd_cuts_histogram      histogram_detector.py:87-112
//   psd_cuts_hash           hash_detector.py:79-109
//   psd_cuts_threshold      threshold_detector.py:113-168, 170-191
#include "cut_automata.cuh"

namespace psd {

__global__ void psd_cuts_flash_filter_kernel(const uint8_t* __restrict__ above, int64_t n, int64_t first_frame,
                                             int64_t min_frames, int mode, int64_t* cuts, int32_t* count,
                                             int32_t cap) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    CutSink out{cuts, cap, 0};
    flash_filter_cuts([&](int64_t i) { return above[i] != 0; }, n, first_frame, 1, min_frames, mode, out);
    *count = out.n;
}

__global__ void psd_cuts_adaptive_kernel(const double* __restrict__ ratio, const double* __restrict__ score,
                                         int64_t n, int64_t first_frame, int window, double adaptive_threshold,
                                         double min_content_val, int64_t min_frames, int64_t* cuts,
                                         int32_t* count, int32_t cap) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    CutSink out{cuts, cap, 0};
    adaptive_cuts(ratio, score, n, first_frame, 1, window, adaptive_threshold, min_content_val, min_frames, out);
    *count = out.n;
}

__global__ void psd_cuts_histogram_kernel(const double* __restrict__ correl, int64_t n, int64_t first_frame,
                                          double threshold, int64_t min_frames, int64_t* cuts, int32_t* count,
                                          int32_t cap) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    CutSink out{cuts, cap, 0};
    histogram_cuts(correl, n, first_frame, 1, threshold, min_frames, out);
    *count = out.n;
}

__global__ void psd_cuts_hash_kernel(const double* __restrict__ dist, int64_t n, int64_t first_frame,
                                     double threshold, int64_t min_frames, int64_t* cuts, int32_t* count,
                                     int32_t cap) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    CutSink out{cuts, cap, 0};
    hash_cuts(dist, n, first_frame, 1, threshold, min_frames, out);
    *count = out.n;
}

__global__ void psd_cuts_threshold_kernel(const double* __restrict__ avg, int64_t n, int64_t first_frame,
                                          double threshold, int method_ceiling, double fade_bias,
                                          int64_t min_frames, int add_final_scene, int64_t* cuts,
                                          int32_t* count, int32_t cap) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    CutSink out{cuts, cap, 0};
    threshold_cuts(avg, n, first_frame, 1, first_frame + n - 1, threshold, method_ceiling, fade_bias, min_frames,
                   add_final_scene, out);
    *count = out.n;
}

}  // namespace psd

using namespace psd;

#define CUT_ARGS_OK(p) PSD_REQUIRE((p) && cuts && count && cap >= 0 && n >= 0, "psd_cuts_*: bad args")

extern "C" int psd_cuts_flash_filter(const uint8_t* above, int64_t n, int64_t first_frame, int64_t min_frames,
                                     int32_t mode, int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    CUT_ARGS_OK(above);
    PSD_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (MERGE) or 1 (SUPPRESS)");
    psd_cuts_flash_filter_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(above, n, first_frame, min_frames, mode, cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_cuts_adaptive(const double* ratio, const double* score, int64_t n, int64_t first_frame,
                                 int32_t window_width, double adaptive_threshold, double min_content_val,
                                 int64_t min_frames, int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    CUT_ARGS_OK(ratio);
    PSD_REQUIRE(score && window_width >= 1, "psd_cuts_adaptive: bad args");
    psd_cuts_adaptive_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(ratio, score, n, first_frame, window_width,
                                                                 adaptive_threshold, min_content_val, min_frames,
                                                                 cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_cuts_hash(const double* dist, int64_t n, int64_t first_frame, double threshold,
                             int64_t min_frames, int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    CUT_ARGS_OK(dist);
    psd_cuts_hash_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(dist, n, first_frame, threshold, min_frames, cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_cuts_histogram(const double* correl, int64_t n, int64_t first_frame, double threshold,
                                  int64_t min_frames, int64_t* cuts, int32_t* count, int32_t cap, void* stream) {
    CUT_ARGS_OK(correl);
    psd_cuts_histogram_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(correl, n, first_frame, threshold, min_frames,
                                                                  cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_cuts_threshold(const double* average, int64_t n, int64_t first_frame, double threshold,
                                  int32_t method_ceiling, double fade_bias, int64_t min_frames,
                                  int32_t add_final_scene, int64_t* cuts, int32_t* count, int32_t cap,
                                  void* stream) {
    CUT_ARGS_OK(average);
    psd_cuts_threshold_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(average, n, first_frame, threshold,
                                                                  method_ceiling, fade_bias, min_frames,
                                                                  add_final_scene, cuts, count, cap);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}
