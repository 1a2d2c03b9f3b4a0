// psd_engine: the stateful C-ABI object behind the detectors' process_frame().
// Owns page-locked staging, device staging, the carried previous frame (the one-frame halo),
// per-frame result arrays in HBM, two streams (copy / compute) and the event plumbing that
// overlaps the H2D of batch k+1 with the kernels of batch k.
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <stddef.h>

#include <memory>
#include <vector>

#include "psd_common.cuh"

namespace psd {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// OpenCV resize.cpp tap generation for INTER_LINEAR (float32 coefficient math, 11-bit fixed point).
// The scale is 1 / (dst / src), as cv::resize derives it from inv_scale_x: it can differ from src / dst in the last
// bit, and at sides above 10 240 pixels that bit can survive the float cast and move a coefficient by one.
static void build_taps(int src, int dst, std::vector<int32_t>& ofs, std::vector<int16_t>& coef) {
    ofs.resize(dst);
    coef.resize(2 * (size_t)dst);
    const double scale = 1.0 / ((double)dst / (double)src);
    for (int d = 0; d < dst; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        f -= (float)s;
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= src - 1) { s = src - 1; f = 0.f; }
        ofs[d] = s;
        const float c0 = (1.f - f) * 2048.f, c1 = f * 2048.f;
        coef[2 * d] = (int16_t)lrintf(c0);  // cvRound: round half to even (default FE_TONEAREST)
        coef[2 * d + 1] = (int16_t)lrintf(c1);
    }
}

// PSD_OK if p is device or managed memory of `device`
int require_device_memory(const void* p, int device, const char* what) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        set_error("%s: %p is not CUDA memory", what, p);
        return PSD_ERR_INVALID;
    }
    PSD_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
                "%s: %p is not device or managed memory", what, p);
    PSD_REQUIRE(at.device == device, "%s: %p is memory of device %d, not of device %d", what, p, at.device, device);
    return PSD_OK;
}

}  // namespace psd

using namespace psd;

struct psd_engine {
    psd_config cfg{};
    int device = 0;
    int sw = 0, sh = 0, W = 0, H = 0;
    int64_t src_frame_bytes = 0, frame_bytes = 0, P = 0;
    bool resize = false;
    uint32_t features = 0;
    int max_batch = 0;
    cudaStream_t copy_stream = nullptr, compute_stream = nullptr;
    // staging (double buffered)
    uint8_t* pinned[2] = {nullptr, nullptr};
    uint8_t* dev_stage[2] = {nullptr, nullptr};
    cudaEvent_t slot_free[2] = {nullptr, nullptr};
    cudaEvent_t h2d_done[2] = {nullptr, nullptr};
    int next_slot = 0;
    // scored-size frames, small_stride apart (a multiple of 16 bytes, as the score pass needs): the resize
    // output, or an aligned copy of a batch whose pointer or frame stride is not a multiple of 16
    uint8_t* small = nullptr;
    int64_t small_stride = 0;
    int32_t* d_xofs = nullptr; int16_t* d_xa = nullptr; int32_t* d_yofs = nullptr; int16_t* d_ya = nullptr;
    // carry (predecessor of the next frame, scored size)
    uint8_t* carry = nullptr;
    bool have_carry = false;
    // per-frame results, `capacity` rows each (FrameRows: row 0 is the halo frame's)
    FrameRows sums{nullptr, sizeof(psd_frame_sums)};
    FrameRows yhist{nullptr, 256 * sizeof(uint32_t)};
    // hash slots: slot 0 is the configured geometry, psd_engine_add_hash_geometry appends
    struct HashSlot { HashPlan plan; FrameRows rows; };   // rows of plan.words uint64
    std::vector<HashSlot> hash;
    int64_t capacity = 0;
    int64_t n_frames = 0;
    bool halo_scored = false;
    // edge path: Canny scratch shared by every edge slot; slot 0 is the configured kernel size,
    // psd_engine_add_edge_kernel_size appends
    EdgeBuffers eb{};
    std::vector<EdgeSlot> edge;
    // last batch bookkeeping for debug taps
    const uint8_t* last_scored = nullptr;
    int64_t last_scored_stride = 0;
    int64_t last_n = 0;
    // timing
    std::vector<cudaEvent_t> ev_pool;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_score, ev_total;
    size_t ev_next = 0;
};

int FrameRows::grow(int64_t cap, int64_t keep, cudaStream_t stream) {
    uint8_t* p = nullptr;
    PSD_CUDA(cudaMalloc(&p, (size_t)cap * row_bytes));
    PSD_CUDA(cudaMemsetAsync(p, 0, (size_t)cap * row_bytes, stream));
    if (d) {
        PSD_CUDA(cudaMemcpyAsync(p, d, (size_t)keep * row_bytes, cudaMemcpyDeviceToDevice, stream));
        PSD_CUDA(cudaStreamSynchronize(stream));
        cudaFree(d);
    }
    d = p;
    return PSD_OK;
}

int FrameRows::zero(int64_t first, int64_t n, cudaStream_t stream) const {
    PSD_CUDA(cudaMemsetAsync(at<uint8_t>(first), 0, (size_t)n * row_bytes, stream));
    return PSD_OK;
}

// The result arrays the score and edge passes accumulate into (zeroed before each batch), then, with `all`, the hash
// slots' (whose pass writes whole rows).  Edge slot 0's SAD rows are part of the sums.
static std::vector<FrameRows*> result_arrays(psd_engine* e, bool all) {
    std::vector<FrameRows*> v{&e->sums};
    if (e->features & PSD_F_YHIST) v.push_back(&e->yhist);
    for (size_t s = 1; s < e->edge.size(); ++s) v.push_back(&e->edge[s].sads);
    if (all)
        for (auto& h : e->hash) v.push_back(&h.rows);
    return v;
}

// the row before stream frame `first`'s (frame first - 1, or the halo frame), nullptr if that frame was not scored
template <class T>
static const T* previous_row(const psd_engine* e, const FrameRows& r, int64_t first) {
    return (first > 0 || e->halo_scored) ? r.at<T>(first - 1) : nullptr;
}

// edge slot 0's SAD rows: psd_frame_sums::sad_edges of the sums, 8 words apart
static FrameRows sums_sad_rows(const psd_engine* e) {
    return FrameRows{e->sums.d + offsetof(psd_frame_sums, sad_edges), e->sums.row_bytes};
}

static int ensure_capacity(psd_engine* e, int64_t need_rows) {
    if (need_rows <= e->capacity) return PSD_OK;
    int64_t cap = e->capacity ? e->capacity : 4096;
    while (cap < need_rows) cap *= 2;
    int rc = PSD_OK;
    for (FrameRows* r : result_arrays(e, true))
        if ((rc = r->grow(cap, e->n_frames + 1, e->compute_stream))) break;
    if (!e->edge.empty())   // slot 0's SADs move with the sums
        e->edge[0].sads = sums_sad_rows(e);
    if (rc) return rc;
    e->capacity = cap;
    return PSD_OK;
}

static cudaEvent_t next_event(psd_engine* e) {
    if (e->ev_next == e->ev_pool.size()) {
        cudaEvent_t ev = nullptr;
        if (cudaEventCreate(&ev) != cudaSuccess) return nullptr;
        e->ev_pool.push_back(ev);
    }
    return e->ev_pool[e->ev_next++];
}

static psd_frame_layout packed_layout(const psd_engine* e, int64_t frame_stride) {
    return psd_frame_layout{frame_stride, (int64_t)e->sw * 3, 3, 1};
}

// the fused pass reads the frames where they are: packed BGR, a frame apart or more, 16-byte aligned
static bool reads_in_place(const psd_engine* e, const uint8_t* src, const psd_frame_layout& l) {
    return !e->resize && layout_packed_bgr(l, e->sw) && l.frame_stride >= e->src_frame_bytes &&
           (((uintptr_t)src | (uintptr_t)l.frame_stride) & 15) == 0;
}

// Score `n` frames at `src` (source size, in layout `l`) that are visible to compute_stream: resized from the
// layout, read in place, or gathered to packed BGR in `small` first (n <= max_batch unless read in place).
// first: stream frame of the first frame (-1 = the halo frame).
static int run_batch(psd_engine* e, const uint8_t* src, const psd_frame_layout& l, int64_t n, int64_t first) {
    cudaStream_t st = e->compute_stream;
    cudaEvent_t t0 = next_event(e), t1 = next_event(e), k0 = next_event(e), k1 = next_event(e);
    if (!t0 || !t1 || !k0 || !k1) { set_error("cudaEventCreate failed"); return PSD_ERR_CUDA; }
    PSD_CUDA(cudaEventRecord(t0, st));
    const uint8_t* scored = src;
    int64_t scored_stride = l.frame_stride;
    if (e->resize) {
        ResizeTaps taps{e->d_xofs, e->d_xa, e->d_yofs, e->d_ya};
        int rc = launch_resize(src, l, e->sw, e->sh, e->small, e->small_stride, e->W, e->H, n, taps, st);
        if (rc) return rc;
        scored = e->small;
        scored_stride = e->small_stride;
    } else if (!reads_in_place(e, src, l)) {
        if (!e->small) PSD_CUDA(cudaMalloc(&e->small, (size_t)e->small_stride * e->max_batch));
        int rc = launch_gather(src, l, n, e->sw, e->sh, e->small, e->small_stride, st);
        if (rc) return rc;
        scored = e->small;
        scored_stride = e->small_stride;
    }
    for (FrameRows* r : result_arrays(e, false)) {
        int rc = r->zero(first, n, st);
        if (rc) return rc;
    }
    if (e->features & PSD_F_EDGES) PSD_CUDA(cudaMemsetAsync(e->eb.vhist, 0, (size_t)n * 256 * sizeof(uint32_t), st));
    ScoreArgs a{};
    a.frames = scored;
    a.prev = (e->have_carry && first >= 0) ? e->carry : nullptr;
    a.frame_stride = scored_stride;
    a.n_frames = (int32_t)n;
    a.n_pixels = (int32_t)e->P;
    a.sums = e->sums.at<psd_frame_sums>(first);
    a.yhist = (e->features & PSD_F_YHIST) ? e->yhist.at<uint32_t>(first) : nullptr;
    a.vhist = (e->features & PSD_F_EDGES) ? e->eb.vhist : nullptr;
    a.vplane = (e->features & PSD_F_EDGES) ? e->eb.vplane : nullptr;
    PSD_CUDA(cudaEventRecord(k0, st));
    int rc = PSD_OK;
    if (e->features & 15u) {  // the fused pass (HSV / byte sum / Y histogram / edges)
        rc = launch_score(a, e->features & 15u, st);
        if (rc) return rc;
    }
    if (e->features & PSD_F_HASH) {
        std::vector<HashPlan> plans; std::vector<uint64_t*> outs;
        for (const auto& h : e->hash) { plans.push_back(h.plan); outs.push_back(h.rows.at<uint64_t>(first)); }
        rc = launch_hash(plans.data(), (int)plans.size(), scored, scored_stride, (int)n, e->W, e->H, outs.data(), st);
        if (rc) return rc;
    }
    PSD_CUDA(cudaEventRecord(k1, st));
    e->ev_score.push_back({k0, k1});
    if (e->features & PSD_F_EDGES) {
        rc = launch_edges(e->eb, (int)n, e->W, e->H, e->edge.data(), (int)e->edge.size(), first, a.prev != nullptr, st);
        if (rc) return rc;
    }
    // carry the last frame (scored size) for the next batch
    PSD_CUDA(cudaMemcpyAsync(e->carry, scored + (n - 1) * scored_stride, (size_t)e->frame_bytes,
                             cudaMemcpyDeviceToDevice, st));
    e->have_carry = true;
    e->last_scored = scored;
    e->last_scored_stride = scored_stride;
    e->last_n = n;
    PSD_CUDA(cudaEventRecord(t1, st));
    e->ev_total.push_back({t0, t1});
    return PSD_OK;
}

extern "C" {

int psd_abi_version(void) { return PSD_ABI_VERSION; }
const char* psd_version(void) { return "psd_b200 0.1.0 (sm_90a)"; }
const char* psd_last_error(void) { return g_err; }
uint64_t psd_launch_count(void) { return g_launches.load(); }

int psd_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int psd_device_info(int device, char* name_out, size_t name_cap, int* cc_major, int* cc_minor,
                    int* sm_count, uint64_t* total_mem) {
    cudaDeviceProp p{};
    PSD_CUDA(cudaGetDeviceProperties(&p, device));
    if (name_out && name_cap) { strncpy(name_out, p.name, name_cap - 1); name_out[name_cap - 1] = 0; }
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (total_mem) *total_mem = (uint64_t)p.totalGlobalMem;
    return PSD_OK;
}

int psd_device_pci_bus_id(int device, char* out, size_t cap) {
    PSD_REQUIRE(out && cap >= 16, "psd_device_pci_bus_id: buffer too small");
    PSD_CUDA(cudaDeviceGetPCIBusId(out, (int)cap, device));
    return PSD_OK;
}

int psd_host_alloc(size_t bytes, void** out) {
    PSD_REQUIRE(out && bytes > 0, "psd_host_alloc: bad args");
    PSD_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    return PSD_OK;
}
int psd_host_free(void* p) {
    if (p) PSD_CUDA(cudaFreeHost(p));
    return PSD_OK;
}
int psd_device_alloc(int device, size_t bytes, void** out) {
    PSD_REQUIRE(out && bytes > 0, "psd_device_alloc: bad args");
    PSD_CUDA(cudaSetDevice(device));
    PSD_CUDA(cudaMalloc(out, bytes));
    return PSD_OK;
}
int psd_device_free(int device, void* p) {
    PSD_CUDA(cudaSetDevice(device));
    if (p) PSD_CUDA(cudaFree(p));
    return PSD_OK;
}
int psd_memcpy_h2d(int device, void* dst, const void* src, size_t bytes) {
    PSD_CUDA(cudaSetDevice(device));
    PSD_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    return PSD_OK;
}
int psd_memcpy_d2h(int device, void* dst, const void* src, size_t bytes) {
    PSD_CUDA(cudaSetDevice(device));
    PSD_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return PSD_OK;
}

void psd_engine_destroy(psd_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->compute_stream) cudaStreamSynchronize(e->compute_stream);
    if (e->copy_stream) cudaStreamSynchronize(e->copy_stream);
    for (int s = 0; s < 2; ++s) {
        if (e->pinned[s]) cudaFreeHost(e->pinned[s]);
        if (e->dev_stage[s]) cudaFree(e->dev_stage[s]);
        if (e->slot_free[s]) cudaEventDestroy(e->slot_free[s]);
        if (e->h2d_done[s]) cudaEventDestroy(e->h2d_done[s]);
    }
    cudaFree(e->small); cudaFree(e->d_xofs); cudaFree(e->d_xa); cudaFree(e->d_yofs); cudaFree(e->d_ya);
    cudaFree(e->carry);
    for (FrameRows* r : result_arrays(e, true)) r->release();
    for (auto& h : e->hash) hash_plan_destroy(&h.plan);
    for (auto& s : e->edge) cudaFree(s.carry_bits);
    edge_buffers_destroy(&e->eb);
    for (cudaEvent_t ev : e->ev_pool) cudaEventDestroy(ev);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    if (e->compute_stream) cudaStreamDestroy(e->compute_stream);
    delete e;
}

// the dilation kernel size of a ContentDetector(kernel_size=k) at the engine's scored size (k = 0: automatic)
static int effective_ksize(const psd_engine* e, int k) {
    if (k == 0) {  // content_detector.py:39-46; Python round() is half-to-even like nearbyint
        k = 4 + (int)nearbyint(sqrt((double)e->W * (double)e->H) / 192.0);
        if ((k & 1) == 0) k += 1;
    }
    return k;
}

// a new edge slot of kernel size k: its scratch, its carried edges and its SAD rows (slot 0's are the sums')
static int add_edge_slot(psd_engine* e, int k) {
    int rc = edge_dilate_check(e->W, k);
    if (rc) return rc;
    rc = e->edge.empty() ? edge_buffers_create(&e->eb, e->W, e->H, e->max_batch, k)
                         : edge_buffers_add_ksize(&e->eb, e->W, e->H, e->max_batch, k);
    if (rc) return rc;
    EdgeSlot s{k, nullptr, FrameRows{nullptr, sizeof(uint64_t)}};
    PSD_CUDA(cudaMalloc(&s.carry_bits, (size_t)e->H * ((e->W + 31) / 32) * 4));
    if (e->edge.empty())
        s.sads = sums_sad_rows(e);
    else if ((rc = s.sads.grow(e->capacity, 0, e->compute_stream))) {
        cudaFree(s.carry_bits);
        return rc;
    }
    e->edge.push_back(s);
    return PSD_OK;
}

// a new hash slot: its plan and its rows
static int add_hash_slot(psd_engine* e, int size, int lowpass) {
    psd_engine::HashSlot h{};
    int rc = hash_plan_create(&h.plan, e->W, e->H, size, lowpass, e->max_batch);
    h.rows.row_bytes = (int64_t)h.plan.words * sizeof(uint64_t);
    if (!rc) rc = h.rows.grow(e->capacity, 0, e->compute_stream);
    if (rc) {
        hash_plan_destroy(&h.plan);
        h.rows.release();
        return rc;
    }
    e->hash.push_back(h);
    return PSD_OK;
}

int psd_engine_create(const psd_config* cfg, psd_engine** out) {
    PSD_REQUIRE(cfg && out, "psd_engine_create: null argument");
    PSD_REQUIRE(cfg->struct_size == (int32_t)sizeof(psd_config), "psd_config.struct_size mismatch");
    PSD_REQUIRE(cfg->src_width > 0 && cfg->src_height > 0 && cfg->width > 0 && cfg->height > 0,
                "frame sizes must be positive");
    PSD_REQUIRE((int64_t)cfg->src_width * cfg->src_height < (1LL << 30), "frame too large");
    PSD_REQUIRE(cfg->features != 0 && (cfg->features & ~31u) == 0, "bad feature mask 0x%x", cfg->features);
    PSD_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= 4096, "max_batch must be in [1,4096]");
    PSD_REQUIRE(cfg->edge_kernel_size == 0 || (cfg->edge_kernel_size >= 3 && (cfg->edge_kernel_size & 1)),
                "kernel_size must be odd integer >= 3");
    PSD_REQUIRE(cfg->flags == 0, "psd_config.flags must be 0 (no flags are defined), got 0x%x", cfg->flags);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error("no CUDA device visible (this engine has no CPU fallback)");
        return PSD_ERR_NODEVICE;
    }
    PSD_REQUIRE(cfg->device >= 0 && cfg->device < ndev, "device %d out of range (%d visible)", cfg->device, ndev);
    cudaDeviceProp prop{};
    PSD_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
        set_error("device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major,
                  prop.minor);
        return PSD_ERR_NODEVICE;
    }
    PSD_CUDA(cudaSetDevice(cfg->device));
    // the engine is destroyed on every return before it is handed out (psd_engine_destroy takes a partial engine)
    std::unique_ptr<psd_engine, void (*)(psd_engine*)> guard(new (std::nothrow) psd_engine(), psd_engine_destroy);
    psd_engine* e = guard.get();
    if (!e) { set_error("out of host memory"); return PSD_ERR_OOM; }
    e->cfg = *cfg;
    e->device = cfg->device;
    e->sw = cfg->src_width; e->sh = cfg->src_height; e->W = cfg->width; e->H = cfg->height;
    e->resize = (e->sw != e->W) || (e->sh != e->H);
    e->P = (int64_t)e->W * e->H;
    e->frame_bytes = e->P * 3;
    e->small_stride = (e->frame_bytes + 15) & ~(int64_t)15;
    e->src_frame_bytes = (int64_t)e->sw * e->sh * 3;
    e->features = cfg->features | ((cfg->features & PSD_F_EDGES) ? PSD_F_HSV : 0);
    e->max_batch = cfg->max_batch;
    PSD_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    PSD_CUDA(cudaStreamCreateWithFlags(&e->compute_stream, cudaStreamNonBlocking));
    for (int s = 0; s < 2; ++s) {
        PSD_CUDA(cudaEventCreateWithFlags(&e->slot_free[s], cudaEventDisableTiming));
        PSD_CUDA(cudaEventCreateWithFlags(&e->h2d_done[s], cudaEventDisableTiming));
    }
    PSD_CUDA(cudaMalloc(&e->carry, (size_t)e->frame_bytes));
    // without resizing, staged batches of a frame size that is not a multiple of 16 bytes are always copied
    // (user device pointers that are not 16-byte aligned allocate it on first use, in run_batch)
    if (e->resize || e->frame_bytes % 16 != 0)
        PSD_CUDA(cudaMalloc(&e->small, (size_t)e->small_stride * e->max_batch));
    if (e->resize) {
        std::vector<int32_t> xo, yo; std::vector<int16_t> xa, ya;
        build_taps(e->sw, e->W, xo, xa);
        build_taps(e->sh, e->H, yo, ya);
        PSD_CUDA(cudaMalloc(&e->d_xofs, xo.size() * 4)); PSD_CUDA(cudaMalloc(&e->d_xa, xa.size() * 2));
        PSD_CUDA(cudaMalloc(&e->d_yofs, yo.size() * 4)); PSD_CUDA(cudaMalloc(&e->d_ya, ya.size() * 2));
        PSD_CUDA(cudaMemcpy(e->d_xofs, xo.data(), xo.size() * 4, cudaMemcpyHostToDevice));
        PSD_CUDA(cudaMemcpy(e->d_xa, xa.data(), xa.size() * 2, cudaMemcpyHostToDevice));
        PSD_CUDA(cudaMemcpy(e->d_yofs, yo.data(), yo.size() * 4, cudaMemcpyHostToDevice));
        PSD_CUDA(cudaMemcpy(e->d_ya, ya.data(), ya.size() * 2, cudaMemcpyHostToDevice));
    }
    int rc = ensure_capacity(e, 4096);
    if (rc) return rc;
    if (e->features & PSD_F_EDGES) {
        if ((rc = add_edge_slot(e, effective_ksize(e, cfg->edge_kernel_size)))) return rc;
    }
    if (e->features & PSD_F_HASH) {
        rc = add_hash_slot(e, cfg->hash_size ? cfg->hash_size : 8, cfg->hash_lowpass ? cfg->hash_lowpass : 2);
        if (rc) return rc;
    }
    *out = guard.release();
    return PSD_OK;
}

int psd_engine_reset(psd_engine* e) {
    PSD_REQUIRE(e, "null engine");
    PSD_CUDA(cudaSetDevice(e->device));
    PSD_CUDA(cudaStreamSynchronize(e->copy_stream));
    PSD_CUDA(cudaStreamSynchronize(e->compute_stream));
    e->n_frames = 0;
    e->have_carry = false;
    e->halo_scored = false;
    e->last_n = 0;
    e->ev_next = 0; e->ev_score.clear(); e->ev_total.clear();
    return PSD_OK;
}

static int ensure_staging(psd_engine* e) {
    for (int s = 0; s < 2; ++s) {
        if (!e->dev_stage[s]) PSD_CUDA(cudaMalloc(&e->dev_stage[s], (size_t)e->src_frame_bytes * e->max_batch));
    }
    return PSD_OK;
}
static int ensure_pinned(psd_engine* e) {
    for (int s = 0; s < 2; ++s) {
        if (!e->pinned[s])
            PSD_CUDA(cudaHostAlloc((void**)&e->pinned[s], (size_t)e->src_frame_bytes * e->max_batch,
                                   cudaHostAllocDefault));
    }
    return PSD_OK;
}

// copy host frames (arbitrary strides) -> device staging slot, tightly packed
static int stage_host(psd_engine* e, const uint8_t* bgr, int64_t n, int64_t frame_stride,
                      int64_t row_pitch, uint32_t flags, int slot) {
    const int64_t tight_row = (int64_t)e->sw * 3;
    PSD_CUDA(cudaEventSynchronize(e->slot_free[slot]));
    const uint8_t* src = bgr;
    int64_t fs = frame_stride, rp = row_pitch;
    if (!(flags & PSD_SUBMIT_PINNED)) {
        int rc = ensure_pinned(e);
        if (rc) return rc;
        uint8_t* dst = e->pinned[slot];
        if (rp == tight_row && fs == e->src_frame_bytes) {
            memcpy(dst, bgr, (size_t)(n * e->src_frame_bytes));
        } else {
            for (int64_t f = 0; f < n; ++f)
                for (int y = 0; y < e->sh; ++y)
                    memcpy(dst + f * e->src_frame_bytes + (int64_t)y * tight_row,
                           bgr + f * frame_stride + (int64_t)y * row_pitch, (size_t)tight_row);
        }
        src = dst; fs = e->src_frame_bytes; rp = tight_row;
    }
    if (rp == tight_row && fs == e->src_frame_bytes) {
        PSD_CUDA(cudaMemcpyAsync(e->dev_stage[slot], src, (size_t)(n * e->src_frame_bytes),
                                 cudaMemcpyHostToDevice, e->copy_stream));
    } else {
        for (int64_t f = 0; f < n; ++f)
            PSD_CUDA(cudaMemcpy2DAsync(e->dev_stage[slot] + f * e->src_frame_bytes, (size_t)tight_row,
                                       src + f * fs, (size_t)rp, (size_t)tight_row, (size_t)e->sh,
                                       cudaMemcpyHostToDevice, e->copy_stream));
    }
    PSD_CUDA(cudaEventRecord(e->h2d_done[slot], e->copy_stream));
    PSD_CUDA(cudaStreamWaitEvent(e->compute_stream, e->h2d_done[slot], 0));
    return PSD_OK;
}

int psd_engine_set_halo_device(psd_engine* e, const void* dptr) {
    PSD_REQUIRE(e && dptr, "psd_engine_set_halo_device: null argument");
    PSD_REQUIRE(e->n_frames == 0, "halo must be set before the first frame is submitted");
    PSD_CUDA(cudaSetDevice(e->device));
    e->have_carry = false;
    int rc = run_batch(e, (const uint8_t*)dptr, packed_layout(e, e->src_frame_bytes), 1, -1);
    if (rc) return rc;
    e->halo_scored = true;
    return PSD_OK;
}

int psd_engine_set_halo_host(psd_engine* e, const uint8_t* bgr, int64_t row_pitch) {
    PSD_REQUIRE(e && bgr, "psd_engine_set_halo_host: null argument");
    PSD_REQUIRE(e->n_frames == 0, "halo must be set before the first frame is submitted");
    PSD_REQUIRE(row_pitch >= (int64_t)e->sw * 3, "row_pitch smaller than a row");
    PSD_CUDA(cudaSetDevice(e->device));
    int rc = ensure_staging(e);
    if (rc) return rc;
    const int slot = e->next_slot;
    e->next_slot ^= 1;
    rc = stage_host(e, bgr, 1, row_pitch * e->sh, row_pitch, 0, slot);
    if (rc) return rc;
    rc = psd_engine_set_halo_device(e, e->dev_stage[slot]);
    if (rc) return rc;
    PSD_CUDA(cudaEventRecord(e->slot_free[slot], e->compute_stream));
    return PSD_OK;
}

int psd_engine_submit_device(psd_engine* e, const void* dptr, int64_t n, int64_t frame_stride) {
    PSD_REQUIRE(e && dptr, "psd_engine_submit_device: null argument");
    PSD_REQUIRE(frame_stride >= e->src_frame_bytes, "frame_stride smaller than a frame");
    const psd_frame_layout l = packed_layout(e, frame_stride);
    return psd_engine_submit_device_layout(e, dptr, n, &l);
}

int psd_engine_submit_device_layout(psd_engine* e, const void* base, int64_t n, const psd_frame_layout* layout) {
    PSD_REQUIRE(e && layout, "psd_engine_submit_device_layout: null argument");
    PSD_REQUIRE(n >= 0, "negative frame count");
    if (n == 0) return PSD_OK;  // an empty array may have no data pointer at all
    PSD_REQUIRE(base, "psd_engine_submit_device_layout: null frames");
    PSD_CUDA(cudaSetDevice(e->device));
    int rc = require_device_memory(base, e->device, "psd_engine_submit_device_layout");
    if (rc) return rc;
    rc = ensure_capacity(e, e->n_frames + n + 1);
    if (rc) return rc;
    const uint8_t* p = (const uint8_t*)base;
    const psd_frame_layout l = *layout;
    // Frames the fused pass can read where they are (no resize, no edge or hash scratch, packed and 16-byte
    // aligned) are scored in one launch: max_batch only sizes staging and those per-batch buffers, and every launch
    // costs a pipeline fill and drain and a work split whose busiest SM sets the launch's time.  Only the kernels'
    // int32 frame counts limit such a batch (2^30 keeps their grid arithmetic clear of overflow too).  Every other
    // batch is resized or gathered into max_batch frames of scratch.
    const bool in_place = !(e->features & (PSD_F_EDGES | PSD_F_HASH)) && reads_in_place(e, p, l);
    const int64_t batch = in_place ? ((int64_t)1 << 30) : (int64_t)e->max_batch;
    int64_t done = 0;
    while (done < n) {
        const int64_t b = (n - done < batch) ? (n - done) : batch;
        rc = run_batch(e, p + done * l.frame_stride, l, b, e->n_frames);
        if (rc) return rc;
        e->n_frames += b;
        done += b;
    }
    return PSD_OK;
}

int psd_engine_submit_host(psd_engine* e, const uint8_t* bgr, int64_t n, int64_t frame_stride,
                           int64_t row_pitch, uint32_t flags) {
    PSD_REQUIRE(e && bgr, "psd_engine_submit_host: null argument");
    PSD_REQUIRE(n >= 0, "negative frame count");
    PSD_REQUIRE(row_pitch >= (int64_t)e->sw * 3, "row_pitch smaller than a row");
    PSD_REQUIRE(n <= 1 || frame_stride >= (int64_t)e->sw * 3, "bad frame_stride");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    int rc = ensure_staging(e);
    if (rc) return rc;
    rc = ensure_capacity(e, e->n_frames + n + 1);
    if (rc) return rc;
    int64_t done = 0;
    while (done < n) {
        const int64_t b = (n - done < e->max_batch) ? (n - done) : e->max_batch;
        const int slot = e->next_slot;
        e->next_slot ^= 1;
        rc = stage_host(e, bgr + done * frame_stride, b, frame_stride, row_pitch, flags, slot);
        if (rc) return rc;
        rc = run_batch(e, e->dev_stage[slot], packed_layout(e, e->src_frame_bytes), b, e->n_frames);
        if (rc) return rc;
        PSD_CUDA(cudaEventRecord(e->slot_free[slot], e->compute_stream));
        e->n_frames += b;
        done += b;
    }
    return PSD_OK;
}

int psd_engine_sync(psd_engine* e) {
    PSD_REQUIRE(e, "null engine");
    PSD_CUDA(cudaSetDevice(e->device));
    PSD_CUDA(cudaStreamSynchronize(e->copy_stream));
    PSD_CUDA(cudaStreamSynchronize(e->compute_stream));
    return PSD_OK;
}

void* psd_engine_compute_stream(psd_engine* e) { return e ? (void*)e->compute_stream : nullptr; }
int64_t psd_engine_frame_count(const psd_engine* e) { return e ? e->n_frames : -1; }
int psd_engine_edge_kernel_size(const psd_engine* e) { return e ? (e->edge.empty() ? 0 : e->edge[0].ksize) : -1; }

// the rows of stream frames [first, first + n) (first = -1: from the halo frame's) to the host, once the engine is idle
static int read_rows(psd_engine* e, const FrameRows& r, int64_t first, int64_t n, void* out) {
    PSD_REQUIRE(first >= -1 && n >= 0 && first + n <= e->n_frames, "frame range out of bounds");
    int rc = psd_engine_sync(e);
    if (rc) return rc;
    if (n) PSD_CUDA(cudaMemcpy(out, r.at<uint8_t>(first), (size_t)n * r.row_bytes, cudaMemcpyDeviceToHost));
    return PSD_OK;
}

int psd_engine_read_sums(psd_engine* e, int64_t first, int64_t n, psd_frame_sums* out) {
    PSD_REQUIRE(e && out, "psd_engine_read_sums: null argument");
    return read_rows(e, e->sums, first, n, out);
}

int psd_engine_read_yhist(psd_engine* e, int64_t first, int64_t n, uint32_t* out) {
    PSD_REQUIRE(e && out, "psd_engine_read_yhist: null argument");
    PSD_REQUIRE(e->features & PSD_F_YHIST, "engine was created without PSD_F_YHIST");
    return read_rows(e, e->yhist, first, n, out);
}

int psd_engine_read_hash_at(psd_engine* e, int32_t slot, int64_t first, int64_t n, uint64_t* out) {
    PSD_REQUIRE(e && out, "psd_engine_read_hash: null argument");
    PSD_REQUIRE(e->features & PSD_F_HASH, "engine was created without PSD_F_HASH");
    PSD_REQUIRE(slot >= 0 && slot < (int32_t)e->hash.size(), "hash slot %d out of range (%d)", slot, (int)e->hash.size());
    return read_rows(e, e->hash[slot].rows, first, n, out);
}

int psd_engine_read_hash(psd_engine* e, int64_t first, int64_t n, uint64_t* out) {
    return psd_engine_read_hash_at(e, 0, first, n, out);
}

int psd_engine_device_hash_at(psd_engine* e, int32_t slot, const uint64_t** hashes) {
    PSD_REQUIRE(e && hashes, "psd_engine_device_hash: null argument");
    if (e->hash.empty() && slot == 0) { *hashes = nullptr; return PSD_OK; }
    PSD_REQUIRE(slot >= 0 && slot < (int32_t)e->hash.size(), "hash slot %d out of range (%d)", slot, (int)e->hash.size());
    *hashes = e->hash[slot].rows.at<uint64_t>(0);
    return PSD_OK;
}

int psd_engine_device_hash(psd_engine* e, const uint64_t** hashes) { return psd_engine_device_hash_at(e, 0, hashes); }

int psd_engine_device_edge_sads(psd_engine* e, int32_t slot, const uint64_t** sad_edges) {
    PSD_REQUIRE(e && sad_edges, "psd_engine_device_edge_sads: null argument");
    PSD_REQUIRE(slot == 0 || (slot > 0 && slot < (int32_t)e->edge.size()), "edge slot %d out of range (%d)", slot,
                (int)e->edge.size());
    *sad_edges = slot == 0 ? nullptr : e->edge[slot].sads.at<uint64_t>(0);
    return PSD_OK;
}

int psd_engine_edge_kernel_size_at(const psd_engine* e, int32_t slot) {
    if (!e || slot < 0 || slot >= (int32_t)e->edge.size()) return -1;
    return e->edge[slot].ksize;
}

// slots can be added while the engine holds nothing that was scored with fewer slots
static int require_empty(psd_engine* e, const char* what) {
    if (e->n_frames != 0 || e->halo_scored || e->have_carry) {
        set_error("%s: the engine already holds frames (add slots after create or reset, before any submit or halo)",
                  what);
        return PSD_ERR_STATE;
    }
    return PSD_OK;
}

int psd_engine_add_edge_kernel_size(psd_engine* e, int32_t kernel_size, int32_t* slot) {
    PSD_REQUIRE(e && slot, "psd_engine_add_edge_kernel_size: null argument");
    PSD_REQUIRE(e->features & PSD_F_EDGES, "engine was created without PSD_F_EDGES");
    PSD_REQUIRE(kernel_size == 0 || (kernel_size >= 3 && (kernel_size & 1)), "kernel_size must be odd integer >= 3");
    int rc = require_empty(e, "psd_engine_add_edge_kernel_size");
    if (rc) return rc;
    const int k = effective_ksize(e, kernel_size);
    for (size_t s = 0; s < e->edge.size(); ++s)
        if (e->edge[s].ksize == k) { *slot = (int32_t)s; return PSD_OK; }
    PSD_CUDA(cudaSetDevice(e->device));
    rc = add_edge_slot(e, k);
    if (rc) return rc;
    *slot = (int32_t)(e->edge.size() - 1);
    return PSD_OK;
}

int psd_engine_add_hash_geometry(psd_engine* e, int32_t size, int32_t lowpass, int32_t* slot) {
    PSD_REQUIRE(e && slot, "psd_engine_add_hash_geometry: null argument");
    PSD_REQUIRE(e->features & PSD_F_HASH, "engine was created without PSD_F_HASH");
    PSD_REQUIRE(size >= 0 && lowpass >= 0, "HashDetector needs size >= 1 and lowpass >= 1");
    int rc = require_empty(e, "psd_engine_add_hash_geometry");
    if (rc) return rc;
    size = size ? size : 8;
    lowpass = lowpass ? lowpass : 2;
    for (size_t s = 0; s < e->hash.size(); ++s) {
        const HashPlan& p = e->hash[s].plan;
        if (p.size == size && p.n == (int64_t)size * lowpass) { *slot = (int32_t)s; return PSD_OK; }
    }
    PSD_CUDA(cudaSetDevice(e->device));
    rc = add_hash_slot(e, size, lowpass);
    if (rc) return rc;
    *slot = (int32_t)(e->hash.size() - 1);
    return PSD_OK;
}

int psd_engine_device_results(psd_engine* e, const psd_frame_sums** sums, const uint32_t** yhist) {
    PSD_REQUIRE(e, "null engine");
    if (sums) *sums = e->sums.at<psd_frame_sums>(0);
    if (yhist) *yhist = e->yhist.d ? e->yhist.at<uint32_t>(0) : nullptr;
    return PSD_OK;
}

int psd_engine_timing_reset(psd_engine* e) {
    PSD_REQUIRE(e, "null engine");
    int rc = psd_engine_sync(e);
    if (rc) return rc;
    e->ev_next = 0; e->ev_score.clear(); e->ev_total.clear();
    return PSD_OK;
}

int psd_engine_timing_ms(psd_engine* e, float* total_ms, float* score_ms, uint64_t* score_launches) {
    PSD_REQUIRE(e, "null engine");
    int rc = psd_engine_sync(e);
    if (rc) return rc;
    float tot = 0.f, sc = 0.f;
    for (auto& p : e->ev_total) { float ms = 0; PSD_CUDA(cudaEventElapsedTime(&ms, p.first, p.second)); tot += ms; }
    for (auto& p : e->ev_score) { float ms = 0; PSD_CUDA(cudaEventElapsedTime(&ms, p.first, p.second)); sc += ms; }
    if (total_ms) *total_ms = tot;
    if (score_ms) *score_ms = sc;
    if (score_launches) *score_launches = e->ev_score.size();
    return PSD_OK;
}

int psd_engine_debug_plane(psd_engine* e, int which, int64_t index, uint8_t* out, size_t cap) {
    PSD_REQUIRE(e && out, "psd_engine_debug_plane: null argument");
    PSD_REQUIRE(index >= 0 && index < e->last_n, "index outside the last batch");
    int rc = psd_engine_sync(e);
    if (rc) return rc;
    if (which == 0) {
        PSD_REQUIRE(cap >= (size_t)e->frame_bytes, "buffer too small");
        PSD_CUDA(cudaMemcpy(out, e->last_scored + index * e->last_scored_stride, (size_t)e->frame_bytes, cudaMemcpyDeviceToHost));
        return PSD_OK;
    }
    PSD_REQUIRE(e->features & PSD_F_EDGES, "engine was created without PSD_F_EDGES");
    PSD_REQUIRE(cap >= (size_t)e->P, "buffer too small");
    PSD_REQUIRE(which >= 1 && which <= 3, "unknown plane %d", which);
    if (which == 2 || which == 3) {  // bit-packed maps -> 0/255 bytes
        rc = edge_unpack(e->eb, index, which == 2, e->W, e->H, e->compute_stream);
        if (rc) return rc;
        PSD_CUDA(cudaStreamSynchronize(e->compute_stream));
        PSD_CUDA(cudaMemcpy(out, e->eb.tmp, (size_t)e->P, cudaMemcpyDeviceToHost));
        return PSD_OK;
    }
    PSD_CUDA(cudaMemcpy(out, e->eb.vplane + index * e->P, (size_t)e->P, cudaMemcpyDeviceToHost));
    return PSD_OK;
}

// ---- host-convenience scans over the engine-owned arrays ----
static int scan_to_host(psd_engine* e, double* d_tmp, double* out, size_t count) {
    PSD_CUDA(cudaStreamSynchronize(e->compute_stream));
    PSD_CUDA(cudaMemcpy(out, d_tmp, count * sizeof(double), cudaMemcpyDeviceToHost));
    return PSD_OK;
}

// a host scan's device buffer: allocated per call, freed on every return
struct ScanBuffer {
    double* p = nullptr;
    ~ScanBuffer() { cudaFree(p); }
};

int psd_engine_scan_content_host_at(psd_engine* e, int32_t edge_slot, int64_t first, int64_t n,
                                    const double weights[4], double weight_abs_sum, double* out_components,
                                    double* out_content_val) {
    PSD_REQUIRE(e && weights && out_content_val, "psd_engine_scan_content_host: null argument");
    PSD_REQUIRE(first >= 0 && n >= 0 && first + n <= e->n_frames, "frame range out of bounds");
    PSD_REQUIRE(edge_slot == 0 || (edge_slot > 0 && edge_slot < (int32_t)e->edge.size()),
                "edge slot %d out of range (%d)", edge_slot, (int)e->edge.size());
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    ScanBuffer tmp;
    PSD_CUDA(cudaMalloc(&tmp.p, (size_t)n * 5 * sizeof(double)));
    const uint64_t* sad_edges = edge_slot ? e->edge[edge_slot].sads.at<uint64_t>(first) : nullptr;
    int rc = psd_scan_content_edges(e->sums.at<psd_frame_sums>(first), sad_edges, n, e->P, weights, weight_abs_sum,
                                    tmp.p + n, tmp.p, e->compute_stream);
    if (!rc) rc = scan_to_host(e, tmp.p, out_content_val, (size_t)n);
    if (!rc && out_components) rc = scan_to_host(e, tmp.p + n, out_components, (size_t)n * 4);
    return rc;
}

int psd_engine_scan_content_host(psd_engine* e, int64_t first, int64_t n, const double weights[4],
                                 double weight_abs_sum, double* out_components, double* out_content_val) {
    return psd_engine_scan_content_host_at(e, 0, first, n, weights, weight_abs_sum, out_components, out_content_val);
}

int psd_engine_scan_adaptive_host(psd_engine* e, const double* scores_host, int64_t n, int32_t window_width,
                                  double min_content_val, double* out_ratio) {
    PSD_REQUIRE(e && scores_host && out_ratio && n >= 0, "psd_engine_scan_adaptive_host: bad argument");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    ScanBuffer tmp;
    PSD_CUDA(cudaMalloc(&tmp.p, (size_t)n * 2 * sizeof(double)));
    PSD_CUDA(cudaMemcpyAsync(tmp.p, scores_host, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, e->compute_stream));
    int rc = psd_scan_adaptive(tmp.p, n, window_width, min_content_val, tmp.p + n, e->compute_stream);
    return rc ? rc : scan_to_host(e, tmp.p + n, out_ratio, (size_t)n);
}

int psd_engine_scan_average_host(psd_engine* e, int64_t first, int64_t n, double* out_avg) {
    PSD_REQUIRE(e && out_avg, "psd_engine_scan_average_host: null argument");
    PSD_REQUIRE(first >= 0 && n >= 0 && first + n <= e->n_frames, "frame range out of bounds");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    ScanBuffer tmp;
    PSD_CUDA(cudaMalloc(&tmp.p, (size_t)n * sizeof(double)));
    int rc = psd_scan_average(e->sums.at<psd_frame_sums>(first), n, e->P * 3, tmp.p, e->compute_stream);
    return rc ? rc : scan_to_host(e, tmp.p, out_avg, (size_t)n);
}

int psd_engine_scan_hist_correl_host(psd_engine* e, int64_t first, int64_t n, int32_t bins, double* out) {
    PSD_REQUIRE(e && out, "psd_engine_scan_hist_correl_host: null argument");
    PSD_REQUIRE(e->features & PSD_F_YHIST, "engine was created without PSD_F_YHIST");
    PSD_REQUIRE(first >= 0 && n >= 0 && first + n <= e->n_frames, "frame range out of bounds");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    ScanBuffer tmp;
    PSD_CUDA(cudaMalloc(&tmp.p, (size_t)n * sizeof(double)));
    int rc = psd_scan_hist_correl(e->yhist.at<uint32_t>(first), n, bins, previous_row<uint32_t>(e, e->yhist, first),
                                  tmp.p, e->compute_stream);
    return rc ? rc : scan_to_host(e, tmp.p, out, (size_t)n);
}

int psd_scan_hash_dist(const uint64_t* hashes, int64_t n, int32_t hash_size, const uint64_t* prev_hash, double* out,
                       void* stream) {
    PSD_REQUIRE(hashes && out && n >= 0 && hash_size >= 1 && hash_size <= 32768, "psd_scan_hash_dist: bad arguments");
    return launch_hash_dist(hashes, n, hash_size, prev_hash, out, (cudaStream_t)stream);
}

int psd_engine_scan_hash_dist_host_at(psd_engine* e, int32_t hash_slot, int64_t first, int64_t n, double* out) {
    PSD_REQUIRE(e && out, "psd_engine_scan_hash_dist_host: null argument");
    PSD_REQUIRE(e->features & PSD_F_HASH, "engine was created without PSD_F_HASH");
    PSD_REQUIRE(hash_slot >= 0 && hash_slot < (int32_t)e->hash.size(), "hash slot %d out of range (%d)", hash_slot,
                (int)e->hash.size());
    PSD_REQUIRE(first >= 0 && n >= 0 && first + n <= e->n_frames, "frame range out of bounds");
    if (n == 0) return PSD_OK;
    PSD_CUDA(cudaSetDevice(e->device));
    ScanBuffer tmp;
    PSD_CUDA(cudaMalloc(&tmp.p, (size_t)n * sizeof(double)));
    const auto& h = e->hash[hash_slot];
    int rc = psd_scan_hash_dist(h.rows.at<uint64_t>(first), n, h.plan.size, previous_row<uint64_t>(e, h.rows, first),
                                tmp.p, e->compute_stream);
    return rc ? rc : scan_to_host(e, tmp.p, out, (size_t)n);
}

int psd_engine_scan_hash_dist_host(psd_engine* e, int64_t first, int64_t n, double* out) {
    return psd_engine_scan_hash_dist_host_at(e, 0, first, n, out);
}

int psd_synth_frames(int device, void* d_out, const int32_t* params_host, int64_t n, int32_t width,
                     int32_t height, int64_t frame_stride, void* stream) {
    PSD_REQUIRE(d_out && params_host && n > 0 && width > 0 && height > 0, "psd_synth_frames: bad args");
    PSD_REQUIRE(frame_stride >= (int64_t)width * height * 3, "frame_stride smaller than a frame");
    PSD_CUDA(cudaSetDevice(device));
    int32_t* d_params = nullptr;
    PSD_CUDA(cudaMalloc(&d_params, (size_t)n * 24 * 4));
    PSD_CUDA(cudaMemcpy(d_params, params_host, (size_t)n * 24 * 4, cudaMemcpyHostToDevice));
    int rc = PSD_OK;
    int64_t done = 0;
    while (!rc && done < n) {
        const int64_t b = (n - done < 4096) ? (n - done) : 4096;
        rc = launch_synth((uint8_t*)d_out + done * frame_stride, d_params + done * 24, b, width, height,
                          frame_stride, (cudaStream_t)stream);
        done += b;
    }
    if (!rc && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) { set_error("synth sync failed: %s", cudaGetErrorString(cudaGetLastError())); rc = PSD_ERR_CUDA; }
    cudaFree(d_params);
    return rc;
}

int psd_gather_bgr(int device, const void* base, const psd_frame_layout* layout, int64_t n, int32_t width,
                   int32_t height, void* dst, int64_t dst_frame_stride, void* stream) {
    PSD_REQUIRE(layout, "psd_gather_bgr: null layout");
    PSD_REQUIRE(n >= 0 && width > 0 && height > 0, "psd_gather_bgr: bad frame count or size");
    if (n == 0) return PSD_OK;
    PSD_REQUIRE(base && dst, "psd_gather_bgr: null frames");
    PSD_REQUIRE(n <= 1 || dst_frame_stride >= (int64_t)width * height * 3, "dst_frame_stride smaller than a frame");
    PSD_CUDA(cudaSetDevice(device));
    int rc = require_device_memory(base, device, "psd_gather_bgr source");
    if (!rc) rc = require_device_memory(dst, device, "psd_gather_bgr destination");
    if (!rc) rc = launch_gather((const uint8_t*)base, *layout, n, width, height, (uint8_t*)dst, dst_frame_stride,
                                (cudaStream_t)stream);
    return rc;
}

int psd_test_resize_taps(int32_t src, int32_t dst, int32_t* ofs, int16_t* coef) {
    PSD_REQUIRE(src > 0 && dst > 0, "psd_test_resize_taps: sizes must be positive");
    PSD_REQUIRE(ofs && coef, "psd_test_resize_taps: null argument");
    std::vector<int32_t> o;
    std::vector<int16_t> c;
    build_taps(src, dst, o, c);
    memcpy(ofs, o.data(), o.size() * sizeof(int32_t));
    memcpy(coef, c.data(), c.size() * sizeof(int16_t));
    return PSD_OK;
}

}  // extern "C"
