// Frames in any psd_frame_layout -> packed BGR24, the form the fused pass reads (engine.cu run_batch) and the one
// SceneManager callbacks receive.  GPU decoders hand out two layouts, and each has a path that moves whole 32-bit
// words: planar rows (NCHW), where one load per plane gives 4 pixels and three __byte_perm-built stores write their
// 12 bytes, and packed RGB24 rows, where 4 pixels are 3 words in and 3 words out with the bytes swapped.  A packed
// BGR24 frame that is one contiguous span is a 2D copy on the copy engine.  Everything else (odd crop offsets, zero
// strides, a row pitch that is not a multiple of 4) takes the per-pixel path.  The kernel moves 6 bytes per pixel.
#include <algorithm>

#include "psd_common.cuh"

namespace psd {

enum GatherMode { kPixels = 0, kPlanar = 1, kPackedBgr = 2, kPackedRgb = 3 };

template <int kMode>
__global__ void __launch_bounds__(128) psd_gather_bgr_kernel(const uint8_t* __restrict__ src, psd_frame_layout l,
                                                             int w, int h, uint8_t* __restrict__ dst,
                                                             int64_t dst_frame_stride) {
    const int64_t f = blockIdx.z;
    const int u = blockIdx.x * blockDim.x + threadIdx.x;  // a pixel (kPixels) or a group of 4 pixels
    if (u >= (kMode == kPixels ? w : w / 4)) return;
    for (int y = blockIdx.y; y < h; y += gridDim.y) {
        const uint8_t* row = src + f * l.frame_stride + (int64_t)y * l.row_stride;
        uint8_t* out = dst + f * dst_frame_stride + (int64_t)y * w * 3;
        if constexpr (kMode == kPixels) {
            const uint8_t* p = row + (int64_t)u * l.pixel_stride;
            out[3 * u] = p[0];
            out[3 * u + 1] = p[l.channel_stride];
            out[3 * u + 2] = p[2 * l.channel_stride];
        } else {
            uint32_t o0, o1, o2;
            if constexpr (kMode == kPlanar) {
                const uint32_t b = *reinterpret_cast<const uint32_t*>(row + 4 * u);
                const uint32_t g = *reinterpret_cast<const uint32_t*>(row + l.channel_stride + 4 * u);
                const uint32_t r = *reinterpret_cast<const uint32_t*>(row + 2 * l.channel_stride + 4 * u);
                // out bytes: b0 g0 r0 b1 | g1 r1 b2 g2 | r2 b3 g3 r3
                o0 = __byte_perm(__byte_perm(b, g, 0x0140), r, 0x2410);  // (b0 g0 b1 .) + r0
                o1 = __byte_perm(__byte_perm(g, r, 0x0251), b, 0x2610);  // (g1 r1 g2 .) + b2
                o2 = __byte_perm(__byte_perm(b, g, 0x0073), r, 0x7106);  // (b3 g3 . .) + r2, r3
            } else {
                // the lowest byte of pixel 0 is B for BGR, R (2 below the base) for RGB
                const uint32_t* in = reinterpret_cast<const uint32_t*>(row - (kMode == kPackedRgb ? 2 : 0) + 12 * u);
                const uint32_t i0 = in[0], i1 = in[1], i2 = in[2];
                if constexpr (kMode == kPackedRgb) {
                    // in bytes: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
                    o0 = __byte_perm(i0, i1, 0x5012);
                    o1 = __byte_perm(__byte_perm(i1, i0, 0x3070), i2, 0x3410);
                    o2 = __byte_perm(i1, i2, 0x5672);
                } else {
                    o0 = i0, o1 = i1, o2 = i2;
                }
            }
            uint32_t* o = reinterpret_cast<uint32_t*>(out + 12 * u);
            o[0] = o0;
            o[1] = o1;
            o[2] = o2;
        }
    }
}

static int gather_mode(const uint8_t* src, const psd_frame_layout& l, int w, const uint8_t* dst, int64_t dfs) {
    const uint64_t common = (uint64_t)l.frame_stride | (uint64_t)l.row_stride | (uint64_t)(uintptr_t)dst |
                            (uint64_t)dfs;
    if (w % 4 != 0 || (common & 3)) return kPixels;
    if (l.pixel_stride == 1 && (((uintptr_t)src | (uint64_t)l.channel_stride) & 3) == 0) return kPlanar;
    if (l.pixel_stride == 3 && l.channel_stride == 1 && ((uintptr_t)src & 3) == 0) return kPackedBgr;
    if (l.pixel_stride == 3 && l.channel_stride == -1 && (((uintptr_t)src - 2) & 3) == 0) return kPackedRgb;
    return kPixels;
}

int launch_gather(const uint8_t* src, const psd_frame_layout& l, int64_t n, int w, int h, uint8_t* dst,
                  int64_t dst_frame_stride, cudaStream_t stream) {
    const int64_t frame_bytes = (int64_t)w * h * 3;
    const int64_t sfs = n == 1 ? frame_bytes : l.frame_stride, dfs = n == 1 ? frame_bytes : dst_frame_stride;
    if (layout_packed_bgr(l, w) && sfs >= frame_bytes && dfs >= frame_bytes) {
        PSD_CUDA(cudaMemcpy2DAsync(dst, (size_t)dfs, src, (size_t)sfs, (size_t)frame_bytes, (size_t)n,
                                   cudaMemcpyDeviceToDevice, stream));
        return PSD_OK;
    }
    const int mode = gather_mode(src, l, w, dst, dst_frame_stride);
    const int units = mode == kPixels ? w : w / 4;
    for (int64_t done = 0; done < n; done += 65535) {
        const int64_t b = std::min<int64_t>(n - done, 65535);
        const dim3 grid((unsigned)((units + 127) / 128), (unsigned)std::min(h, 65535), (unsigned)b);
        const uint8_t* s = src + done * l.frame_stride;
        uint8_t* d = dst + done * dst_frame_stride;
        switch (mode) {
            case kPlanar: psd_gather_bgr_kernel<kPlanar><<<grid, 128, 0, stream>>>(s, l, w, h, d, dst_frame_stride); break;
            case kPackedBgr: psd_gather_bgr_kernel<kPackedBgr><<<grid, 128, 0, stream>>>(s, l, w, h, d, dst_frame_stride); break;
            case kPackedRgb: psd_gather_bgr_kernel<kPackedRgb><<<grid, 128, 0, stream>>>(s, l, w, h, d, dst_frame_stride); break;
            default: psd_gather_bgr_kernel<kPixels><<<grid, 128, 0, stream>>>(s, l, w, h, d, dst_frame_stride); break;
        }
        PSD_CHECK_LAUNCH();
        count_launch();
    }
    return PSD_OK;
}

}  // namespace psd
