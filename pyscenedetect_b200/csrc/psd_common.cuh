// Shared helpers for the psd_b200 CUDA translation units (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "../../include/psd_b200.h"

namespace psd {

// ---- error plumbing (thread-local message, no exceptions across the ABI) ----
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define PSD_CUDA(expr)                                                                           \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            psd::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,     \
                           __LINE__);                                                            \
            return (_e == cudaErrorMemoryAllocation) ? PSD_ERR_OOM : PSD_ERR_CUDA;               \
        }                                                                                        \
    } while (0)

#define PSD_CHECK_LAUNCH()                                                                       \
    do {                                                                                         \
        cudaError_t _e = cudaGetLastError();                                                     \
        if (_e != cudaSuccess) {                                                                 \
            psd::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                            \
            return PSD_ERR_CUDA;                                                                 \
        }                                                                                        \
    } while (0)

#define PSD_REQUIRE(cond, ...)                                                                   \
    do {                                                                                         \
        if (!(cond)) {                                                                           \
            psd::set_error(__VA_ARGS__);                                                         \
            return PSD_ERR_INVALID;                                                              \
        }                                                                                        \
    } while (0)

// PSD_OK if p is device or managed memory of `device`, else PSD_ERR_INVALID with a message prefixed by `what`
int require_device_memory(const void* p, int device, const char* what);

// ---- fused score pass (score_kernel.cu) ----
struct ScoreArgs {
    const uint8_t* frames;   // n frames, frame_stride apart, tightly packed rows (3*W bytes); 16-byte aligned
    const uint8_t* prev;     // predecessor of frames[0] or nullptr; 16-byte aligned
    int64_t frame_stride;    // a multiple of 16
    int32_t n_frames;
    int32_t n_pixels;        // W*H
    int32_t n_chunks;        // time chunks (the persistent kernel splits the frames into n_chunks near-equal runs)
    uint32_t features;       // PSD_F_* mask of the launch (for the persistent kernel: a copy of the template argument)
    int32_t n_strips;
    psd_frame_sums* sums;    // [n] (pre-zeroed)
    uint32_t* yhist;         // [n][256] (pre-zeroed) or nullptr
    uint32_t* vhist;         // [n][256] (pre-zeroed) or nullptr
    uint8_t* vplane;         // [n][n_pixels] or nullptr
    uint32_t shift24;        // 0x01000000, passed at run time: the kernel derives a zero the compiler cannot fold from it
};
int launch_score(const ScoreArgs& a, uint32_t features, cudaStream_t stream);

// ---- resize (resize_kernel.cu) ----
struct ResizeTaps {  // device arrays built on the host exactly as OpenCV builds them
    const int32_t* xofs;  // [dw] source column of tap 0
    const int16_t* xa;    // [dw][2] 11-bit coefficients
    const int32_t* yofs;  // [dh]
    const int16_t* ya;    // [dh][2]
};
int launch_resize(const uint8_t* src, const psd_frame_layout& layout, int sw, int sh, uint8_t* dst,
                  int64_t dst_frame_stride, int dw, int dh, int64_t n, const ResizeTaps& taps, cudaStream_t stream);

// ---- layout gather (gather_kernel.cu) ----
// n frames of w x h in `layout` -> packed BGR24, dst_frame_stride apart (no argument checks: callers validate)
int launch_gather(const uint8_t* src, const psd_frame_layout& layout, int64_t n, int w, int h, uint8_t* dst,
                  int64_t dst_frame_stride, cudaStream_t stream);
// the layout is packed BGR24 rows (3 bytes per pixel, B first, rows 3*w bytes apart)
inline bool layout_packed_bgr(const psd_frame_layout& l, int w) {
    return l.pixel_stride == 3 && l.channel_stride == 1 && l.row_stride == 3 * (int64_t)w;
}

// ---- per-frame result arrays of an engine (engine.cu) ----
// Row 0 belongs to the halo frame, stream frame i sits at row i + 1: at() is the one place that mapping is made.
struct FrameRows {
    uint8_t* d = nullptr;
    int64_t row_bytes = 0;
    template <class T> T* at(int64_t frame) const { return reinterpret_cast<T*>(d + (frame + 1) * row_bytes); }
    // cap zeroed rows holding the first `keep` rows of the current array, if there is one
    int grow(int64_t cap, int64_t keep, cudaStream_t stream);
    int zero(int64_t first, int64_t n, cudaStream_t stream) const;  // the rows of stream frames [first, first + n)
    void release() { cudaFree(d); d = nullptr; }
};

// ---- edge path (edge_kernels.cu) ----
struct EdgeBuffers {
    uint8_t* vplane;    // [n][P] V of HSV (written by the score pass)
    uint32_t* vhist;    // [n][256]
    int32_t* thresholds;// [n][2] low, high
    uint32_t* cand;     // [n][edge_tile_words] Canny candidates (weak or strong pixels), 32 per word, TILE-MAJOR:
                        // tile (ty, tx) = 32 rows x 64 columns = 64 consecutive words, row r at words 2r, 2r+1
    uint32_t* bits_in;  // same layout: strong pixels after classify, the Canny map after hysteresis
    uint32_t* bits_dil; // [n][H][Wq] dilated edges, row-major (of each edge slot in turn)
    uint32_t* bits_hdil;// [n][H][Wq] horizontal pass of the separable dilation (if a kernel size >= 19 is in use, else null)
    uint8_t* tmp;       // [P] scratch for debug taps
    uint8_t* dirty;     // [2][n][tiles] hysteresis: tiles to revisit (double-buffered by round parity)
    int32_t* hyst_flags;// [3] hysteresis: "some tile changed" per round (rotating)
};
// the Canny scratch of batches of up to max_batch frames, and what the dilation of kernel size ksize needs
int edge_buffers_create(EdgeBuffers* b, int W, int H, int max_batch, int ksize);
int edge_buffers_add_ksize(EdgeBuffers* b, int W, int H, int max_batch, int ksize);  // another kernel size's needs
void edge_buffers_destroy(EdgeBuffers* b);
struct EdgeSlot {          // one dilation kernel size of an engine
    int ksize;
    uint32_t* carry_bits;  // [H][Wq] this size's dilated edges of the predecessor frame
    FrameRows sads;        // a frame's SAD accumulates into the first uint64 of its row (pre-zeroed): slot 0's rows are
                           // the sums' (psd_frame_sums::sad_edges, 8 words apart), every other slot owns one word a row
};
// Canny (thresholds, classify, hysteresis) once, then a dilation and a SAD per slot; the batch's frame 0 is stream
// frame `first` of the slots' SAD rows
int launch_edges(const EdgeBuffers& b, int n, int width, int height, const EdgeSlot* slots, int n_slots, int64_t first,
                 bool have_prev, cudaStream_t stream);
// frame `index` of the last batch's Canny map (canny_map) or dilated map -> 0/255 bytes in b.tmp
int edge_unpack(const EdgeBuffers& b, int64_t index, bool canny_map, int W, int H, cudaStream_t stream);
int edge_dilate_check(int W, int ksize); // PSD_OK, or PSD_ERR_INVALID if a row of the separable pass is too wide

// ---- perceptual hash (hash_kernels.cu) ----
struct HashPlan {        // per-engine tables for one (frame size, hash size, lowpass)
    int n = 0, size = 0; // hash image edge (size * lowpass), low band edge
    int fast = 0;        // both area scale factors are integers
    int area_w = 0, area_h = 0;
    int32_t *xstart = nullptr, *xsi = nullptr, *ystart = nullptr, *ysi = nullptr;
    int32_t *xmid = nullptr;  // [n][2]: table index of the first whole-pixel tap of a destination column, their count
    float *xalpha = nullptr, *ybeta = nullptr;
    double* cosn = nullptr;   // [4n] cos(pi k / 2n)
    int levels = 1, len[8] = {0}, off[8] = {0};  // folded levels of a length-n vector (hash_kernels.cu:FoldPlan)
    int words = PSD_HASH_WORDS;  // per-frame stride of the hash arrays: PSD_HASH_WORDS_FOR(size)
    int batch = 0;               // frames per sub-batch of the hash pass
    bool global_ws = false;      // the finish kernel's working set lives in `ws`, not in shared memory
    int64_t ws_doubles = 0;      // finish working set per frame (doubles)
    float* rowbuf = nullptr;  // [batch][H][n] horizontal pass
    double* ws = nullptr;     // [batch][ws_doubles] finish workspace (global_ws only)
};
// force_global_ws: the finish kernel's working set in `ws` even where it fits shared memory (psd_test_hash_stages
// reads the normalised image and the low band from there)
int hash_plan_create(HashPlan* p, int W, int H, int size, int lowpass, int max_batch, bool force_global_ws = false);
void hash_plan_destroy(HashPlan* p);
// every plan's hashes of n_frames frames: hashes[g] receives plan g's ([n_frames][plans[g].words]); one gray
// pass and one rows launch per sub-batch feed all the plans
int launch_hash(const HashPlan* plans, int n_plans, const uint8_t* frames, int64_t frame_stride, int n_frames, int W,
                int H, uint64_t* const* hashes, cudaStream_t stream);
int launch_hash_dist(const uint64_t* hashes, int64_t n, int size, const uint64_t* prev_hash, double* out,
                     cudaStream_t stream);

// ---- cut automata over grid cells (sweep_kernels.cu) ----
// the host-side checks of psd_sweep_cuts on an array of cells; `who` prefixes the error message
int validate_sweep_cells(const psd_sweep_cell* cells, int32_t n_cells, const char* who);

// ---- clip tables (clip_kernels.cu) ----
// In place: v[0, m) counts -> exclusive offsets, v[m] = their sum (one block of 1024 threads)
__global__ void __launch_bounds__(1024) psd_clip_scan_kernel(int64_t* __restrict__ v, int64_t m);

// ---- synthetic generator (synth_kernel.cu) ----
int launch_synth(uint8_t* out, const int32_t* d_params, int64_t n, int width, int height,
                 int64_t frame_stride, cudaStream_t stream);

}  // namespace psd
