// Exact cv2.resize(..., INTER_LINEAR) for 8UC3 (scene_manager.py:670-678), the downscale
// SceneManager applies before handing a frame to the detectors.  Restates OpenCV's fixed-point
// bilinear (resize.cpp: INTER_RESIZE_COEF_BITS = 11; tap tables built on the host with float32
// coefficient generation, see engine.cu build_taps(); oracle/intmath.py:resize_linear is the
// pinned CPU twin).  Only the 2x2 source taps of each output pixel are read, through a psd_frame_layout, so a
// crop, a planar (NCHW) frame or RGB channel order is resized from where it lies, with no copy before.
#include <algorithm>

#include "psd_common.cuh"

namespace psd {

__global__ void __launch_bounds__(256) psd_resize_kernel(const uint8_t* __restrict__ src, psd_frame_layout l,
                                                         int sw, int sh, uint8_t* __restrict__ dst,
                                                         int64_t dst_frame_stride, int dw, int dh, ResizeTaps taps) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t f = blockIdx.z;
    if (x >= dw) return;
    const int sx0 = taps.xofs[x];
    const int sx1 = min(sx0 + 1, sw - 1);
    const int a0 = taps.xa[2 * x], a1 = taps.xa[2 * x + 1];
    const int64_t p0 = (int64_t)sx0 * l.pixel_stride, p1 = (int64_t)sx1 * l.pixel_stride;
    // grid.y is capped at 65 535 (launch_resize), so taller outputs take several rows per block
    for (int y = blockIdx.y; y < dh; y += gridDim.y) {
        const int sy0 = taps.yofs[y];
        const int sy1 = min(sy0 + 1, sh - 1);
        const int b0 = taps.ya[2 * y], b1 = taps.ya[2 * y + 1];
        const uint8_t* r0 = src + f * l.frame_stride + (int64_t)sy0 * l.row_stride;
        const uint8_t* r1 = src + f * l.frame_stride + (int64_t)sy1 * l.row_stride;
        uint8_t* o = dst + f * dst_frame_stride + ((int64_t)y * dw + x) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int64_t cs = c * l.channel_stride;
            const int h0 = r0[p0 + cs] * a0 + r0[p1 + cs] * a1;  // x2048
            const int h1 = r1[p0 + cs] * a0 + r1[p1 + cs] * a1;
            const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            o[c] = (uint8_t)min(max(v, 0), 255);
        }
    }
}

int launch_resize(const uint8_t* src, const psd_frame_layout& layout, int sw, int sh, uint8_t* dst,
                  int64_t dst_frame_stride, int dw, int dh, int64_t n, const ResizeTaps& taps, cudaStream_t stream) {
    PSD_REQUIRE(n > 0 && n <= 65535, "resize batch out of range");
    dim3 grid((dw + 255) / 256, (unsigned)std::min(dh, 65535), (unsigned)n);
    psd_resize_kernel<<<grid, 256, 0, stream>>>(src, layout, sw, sh, dst, dst_frame_stride, dw, dh, taps);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

}  // namespace psd
