// Trailing device scans: integer per-frame sums -> the detectors' float64 metrics.
// Every fp64 operation is an explicit IEEE round-to-nearest op in the reference's operation
// order (no FMA contraction), so the metrics are bit-identical to numpy/CPython:
//   components / content_val    content_detector.py:29-36,166-180
//   adaptive_ratio              adaptive_detector.py:116-128
//   average_rgb                 threshold_detector.py:127
//   hist_diff                   histogram_detector.py:98,159-163 (cv2.normalize + HISTCMP_CORREL)
#include <math_constants.h>

#include "psd_common.cuh"

namespace psd {

// sad_edges: the edge SAD of another dilation kernel size (an engine's edge slot), read in place of
// sums[i].sad_edges; nullptr = the sums' own
__global__ void psd_scan_content_kernel(const psd_frame_sums* __restrict__ sums,
                                        const uint64_t* __restrict__ sad_edges, int64_t n,
                                        double n_pixels, double w0, double w1, double w2, double w3,
                                        double wsum, double* __restrict__ comps,
                                        double* __restrict__ score) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const psd_frame_sums s = sums[i];
    double c[4] = {0.0, 0.0, 0.0, 0.0};
    double val = 0.0;
    if (s.has_prev) {
        // numpy.sum(int) / float(num_pixels): exact integer -> one fp64 divide
        c[0] = __ddiv_rn(__ull2double_rn(s.sad_hue), n_pixels);
        c[1] = __ddiv_rn(__ull2double_rn(s.sad_sat), n_pixels);
        c[2] = __ddiv_rn(__ull2double_rn(s.sad_lum), n_pixels);
        c[3] = __ddiv_rn(__ull2double_rn(sad_edges ? sad_edges[i] : s.sad_edges), n_pixels);
        // sum(component * weight ...) : 0 + p0, + p1, + p2, + p3 (plain sequential fp64 adds)
        double acc = __dadd_rn(0.0, __dmul_rn(c[0], w0));
        acc = __dadd_rn(acc, __dmul_rn(c[1], w1));
        acc = __dadd_rn(acc, __dmul_rn(c[2], w2));
        acc = __dadd_rn(acc, __dmul_rn(c[3], w3));
        val = __ddiv_rn(acc, wsum);
    }
    if (comps) {
        comps[4 * i + 0] = c[0];
        comps[4 * i + 1] = c[1];
        comps[4 * i + 2] = c[2];
        comps[4 * i + 3] = c[3];
    }
    score[i] = val;
}

__global__ void psd_scan_adaptive_kernel(const double* __restrict__ scores, int64_t n, int w,
                                         double min_content_val, double* __restrict__ ratio) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i < w || i + w >= n) {
        ratio[i] = CUDART_NAN;  // window incomplete: the reference emits no ratio for this frame
        return;
    }
    // sum(score for j != centre) in buffer order, sequential adds (a prefix sum would round
    // differently), then / (2.0 * window_width)
    double acc = 0.0;
    bool first = true;
    for (int64_t j = i - w; j <= i + w; ++j) {
        if (j == i) continue;
        acc = first ? scores[j] : __dadd_rn(acc, scores[j]);
        first = false;
    }
    const double avg = __ddiv_rn(acc, __dmul_rn(2.0, (double)w));
    const double target = scores[i];
    double r = 0.0;
    if (!(fabs(avg) < 0.00001)) {
        const double q = __ddiv_rn(target, avg);
        r = (255.0 < q) ? 255.0 : q;  // min(q, 255.0)
    } else if (target >= min_content_val) {
        r = 255.0;
    }
    ratio[i] = r;
}

__global__ void psd_scan_average_kernel(const psd_frame_sums* __restrict__ sums, int64_t n,
                                        double n_values, double* __restrict__ avg) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    avg[i] = __ddiv_rn(__ull2double_rn(sums[i].bgr_sum), n_values);
}

// One warp per frame.  hist[] are raw 256-bin counts; bins <= 256 rebinning is
// floor(v * bins / 256) as cv2.calcHist does for uniform ranges.
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}

__device__ __forceinline__ void load_normalised(const uint32_t* __restrict__ h256, int bins, int lane,
                                                float (&out)[8]) {
    // lane owns bins lane, lane+32, ...
    double sq = 0.0;
    float cnt[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int b = lane + 32 * k;
        uint32_t c = 0;
        if (b < bins) {
            // values v with floor(v*bins/256) == b  <=>  v in [ceil(256 b / bins), ceil(256 (b+1) / bins))
            const int v0 = (256 * b + bins - 1) / bins, v1 = (256 * (b + 1) + bins - 1) / bins;
            for (int v = v0; v < v1; ++v) c += h256[v];
        }
        cnt[k] = (float)c;  // calcHist output is float32 (exact below 2^24 counts per bin)
        sq = __dadd_rn(sq, __dmul_rn((double)cnt[k], (double)cnt[k]));
    }
    const double norm = sqrt(warp_sum(sq));  // cv2.norm(NORM_L2) in fp64 (integer-exact sum)
    const float scale = (norm > 2.220446049250313e-16) ? (float)__ddiv_rn(1.0, norm) : 0.0f;
#pragma unroll
    for (int k = 0; k < 8; ++k) out[k] = __fmul_rn(cnt[k], scale);
}

__global__ void psd_scan_hist_correl_kernel(const uint32_t* __restrict__ yhist, int64_t n, int bins,
                                            const uint32_t* __restrict__ prev_hist,
                                            double* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    const uint32_t* hp = (i == 0) ? prev_hist : yhist + (i - 1) * 256;
    if (hp == nullptr) {
        if (lane == 0) out[i] = CUDART_NAN;
        return;
    }
    float a[8], b[8];
    load_normalised(hp, bins, lane, a);
    load_normalised(yhist + i * 256, bins, lane, b);
    double s1 = 0, s2 = 0, s11 = 0, s22 = 0, s12 = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const double x = (double)a[k], y = (double)b[k];
        s1 = __dadd_rn(s1, x);
        s2 = __dadd_rn(s2, y);
        s11 = __dadd_rn(s11, __dmul_rn(x, x));
        s22 = __dadd_rn(s22, __dmul_rn(y, y));
        s12 = __dadd_rn(s12, __dmul_rn(x, y));
    }
    s1 = warp_sum(s1); s2 = warp_sum(s2); s11 = warp_sum(s11); s22 = warp_sum(s22); s12 = warp_sum(s12);
    if (lane == 0) {
        const double scale = __ddiv_rn(1.0, (double)bins);
        const double num = __dsub_rn(s12, __dmul_rn(__dmul_rn(s1, s2), scale));
        const double d1 = __dsub_rn(s11, __dmul_rn(__dmul_rn(s1, s1), scale));
        const double d2 = __dsub_rn(s22, __dmul_rn(__dmul_rn(s2, s2), scale));
        const double den2 = __dmul_rn(d1, d2);
        out[i] = (fabs(den2) > 2.220446049250313e-16) ? __ddiv_rn(num, sqrt(den2)) : 1.0;
    }
}

__global__ void psd_scan_compare_kernel(const double* __restrict__ v, int64_t n, double thr, int op,
                                        uint8_t* __restrict__ flags) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = v[i];
    flags[i] = (op == 0) ? (x >= thr) : (op == 1) ? (x <= thr) : (x < thr);
}

}  // namespace psd

using namespace psd;

extern "C" int psd_scan_content_edges(const psd_frame_sums* sums, const uint64_t* sad_edges, int64_t n,
                                      int64_t n_pixels, const double weights[4], double weight_abs_sum,
                                      double* out_components, double* out_content_val, void* stream) {
    PSD_REQUIRE(sums && out_content_val && weights && n >= 0 && n_pixels > 0, "psd_scan_content: bad args");
    if (n == 0) return PSD_OK;
    psd_scan_content_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        sums, sad_edges, n, (double)n_pixels, weights[0], weights[1], weights[2], weights[3], weight_abs_sum,
        out_components, out_content_val);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_scan_content(const psd_frame_sums* sums, int64_t n, int64_t n_pixels,
                                const double weights[4], double weight_abs_sum, double* out_components,
                                double* out_content_val, void* stream) {
    return psd_scan_content_edges(sums, nullptr, n, n_pixels, weights, weight_abs_sum, out_components,
                                  out_content_val, stream);
}

extern "C" int psd_scan_adaptive(const double* scores, int64_t n, int32_t window_width,
                                 double min_content_val, double* out_ratio, void* stream) {
    PSD_REQUIRE(scores && out_ratio && n >= 0 && window_width >= 1, "psd_scan_adaptive: bad args");
    if (n == 0) return PSD_OK;
    psd_scan_adaptive_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        scores, n, window_width, min_content_val, out_ratio);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_scan_average(const psd_frame_sums* sums, int64_t n, int64_t n_values, double* out_avg,
                                void* stream) {
    PSD_REQUIRE(sums && out_avg && n >= 0 && n_values > 0, "psd_scan_average: bad args");
    if (n == 0) return PSD_OK;
    psd_scan_average_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        sums, n, (double)n_values, out_avg);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_scan_hist_correl(const uint32_t* yhist, int64_t n, int32_t bins,
                                    const uint32_t* prev_hist, double* out_correl, void* stream) {
    PSD_REQUIRE(yhist && out_correl && n >= 0 && bins >= 1 && bins <= 256,
                "psd_scan_hist_correl: bins must be in [1,256]");
    if (n == 0) return PSD_OK;
    psd_scan_hist_correl_kernel<<<(unsigned)((n * 32 + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        yhist, n, bins, prev_hist, out_correl);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

extern "C" int psd_scan_compare(const double* values, int64_t n, double threshold, int32_t op,
                                uint8_t* out_flags, void* stream) {
    PSD_REQUIRE(values && out_flags && n >= 0 && op >= 0 && op <= 2, "psd_scan_compare: bad args");
    if (n == 0) return PSD_OK;
    psd_scan_compare_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        values, n, threshold, op, out_flags);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}
