// Fused per-frame score pass: one read of every BGR byte produces
//   * SAD of the H, S, V planes against the previous frame   (content_detector.py:29-36,155,166-175)
//   * the sum of all B,G,R bytes                              (threshold_detector.py:127)
//   * the 256-bin histogram of YUV-Y                          (histogram_detector.py:156-159)
//   * (edge path) the V plane + its 256-bin histogram         (content_detector.py:231,238)
//
// The frames and the predecessor frame must be 16-byte aligned (base pointers and frame stride: the engine
// copies any other input into an aligned buffer first).  The first P16 = P & ~15 pixels of every frame go
// through the persistent warp-specialised kernel psd_score_ws_kernel<F>; the last P - P16 (< 16) pixels, if
// any, through psd_score_tail_kernel with the same HSV device function.  Every partial sum reaches HBM as an
// integer atomic, so the results are order-independent integers and identical for any batching / sharding.
#include "hsv_half2.cuh"
#include "psd_common.cuh"

namespace psd {

constexpr int kPxPerThread = 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes,
                                         unsigned long long* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ---------------------------------------------------------------------------------------------
// Warp-specialised, persistent kernel (the first P16 pixels of every frame).
//
// One CTA per SM for the whole launch: 24 consumer warps + 4 side warps.  The work is cut into items
// (strip of 12288 pixels x chunk of consecutive frames); CTA b walks items b, b + grid, b + 2 grid, ...
// Within an item the previous frame's H,S,V of a thread's 16 pixels stay in registers, so HBM traffic is
// one read of each BGR byte (+1 halo frame per item).
// Frames travel global->shared by 1-D bulk TMA into a 4-stage ring whose stage sequence simply continues
// from one item into the next, so the producer is always kWsStages frames ahead - also across item
// boundaries: there is no pipeline fill / drain per item, the LUT is built once per SM and no SM idles
// between CTAs (the non-persistent form lost ~4 % of the SM time between CTAs and ~5 % of the warp time
// waiting for the first frame of each CTA).
//
// No CTA-wide barrier in the frame loop: consumers wait on the stage's FULL mbarrier (TMA complete_tx),
// pull their 48 bytes, do the arithmetic, add their SADs to the stage's per-lane shared accumulators and
// arrive on the stage's EMPTY mbarrier.  Side warp s (warp 24 + s, so one per SM sub-partition) owns
// stage s: it waits for the 24 arrivals, takes and zeroes the stage's totals and histogram bins, re-arms
// the stage with the frame kWsStages slots ahead (one lane issues the copy) and then flushes what it took
// to HBM with integer atomics.  EMPTY phases complete in slot order, so the copies are still issued in
// slot order.  The stages advance only as fast as their slowest sub-partition, so the per-frame
// bookkeeping is dealt out to all four instead of adding to the issue load of sub-partition 0.
//
// An item whose frame count is not a multiple of the consumer loop's unroll factor is padded with null
// slots (the producer completes the FULL barrier without a copy, the consumers only arrive), so a loop
// body always starts at a stage that is a multiple of the unroll factor and every stage offset inside
// the body is an immediate.
// ---------------------------------------------------------------------------------------------
// 24 consumer warps = 6 per sub-partition (25 was measured 4.5 % slower: 7/6/6/6 is unbalanced).
// The last strip may be partial: it holds the rest of the first P16 pixels, a whole number of 16-pixel
// thread slices (1080p: 168 full strips + one of 9216 px).
constexpr int kWsConsumerWarps = 24;
constexpr int kWsConsumers = kWsConsumerWarps * 32;  // 768
constexpr int kWsStages = 4;
constexpr int kWsSideWarps = kWsStages;              // side warp s retires and re-arms stage s
constexpr int kWsThreads = kWsConsumers + kWsSideWarps * 32;  // 28 warps x 72 registers fit the 64 K register file
static_assert(kWsSideWarps == 4 && kWsConsumerWarps % 4 == 0, "one side warp per SM sub-partition");
constexpr int kWsUnroll = 4;                         // frames per consumer loop body: all stage offsets immediate
constexpr int kWsStripPx = kWsConsumers * kPxPerThread;  // 12288 pixels
constexpr int kWsStripBytes = kWsStripPx * 3;            // 36864 bytes
static_assert(kWsStages % kWsUnroll == 0, "the stage ring must be a whole number of loop bodies");

struct __align__(128) WsSmem {
    uint8_t ring[kWsStages][kWsStripBytes];
    float lut[256 * 64];
    unsigned long long full[kWsStages];
    unsigned long long empty[kWsStages];   // must follow `full` (addressed as full + kWsStages * 8)
    // per-lane totals of sadH, sadS, sadV, bgr: every consumer thread adds its partial to the word of ITS
    // lane (32 distinct banks: one conflict-free red.shared per channel per thread, no warp reduction, no
    // election).  The side warp that retires the stage zeroes them before it hands the stage back.
    uint32_t accl[kWsStages][4][32];
    uint32_t accl_sink[kWsStages][4][32];  // where threads without pixels / without a predecessor frame add
    uint32_t yhist[kWsStages][256];
    uint32_t vhist[kWsStages][256];
};

__device__ __forceinline__ uint32_t sad4_acc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
// try_wait with a long suspend-time hint: the waiting warp sleeps in hardware until the phase
// completes instead of burning issue slots of its sub-partition in a poll loop
template <int OFF>
__device__ __forceinline__ void mbar_wait_hint_off(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0+%3], %1, %2;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar),
        "r"(parity), "r"(20000u), "n"(OFF)
        : "memory");
}
__device__ __forceinline__ void mbar_wait_hint(unsigned long long* bar, uint32_t parity) {
    mbar_wait_hint_off<0>(smem_u32(bar), parity);
}
template <int OFF>
__device__ __forceinline__ void lds128_off(uint32_t addr, uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& w) {
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4+%5];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(addr), "n"(OFF));
}
template <int OFF>
__device__ __forceinline__ void red_shared_add_off(uint32_t addr, uint32_t v) {
    asm volatile("red.shared.add.u32 [%0+%2], %1;" ::"r"(addr), "r"(v), "n"(OFF) : "memory");
}
template <int OFF>
__device__ __forceinline__ void mbar_arrive_off(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0+%1];" ::"r"(bar), "n"(OFF) : "memory");
}

// ---- work decomposition shared by host, producer and consumers ----
// chunk c covers frames [c * N / C, (c + 1) * N / C): sizes differ by at most one frame
__host__ __device__ __forceinline__ int chunk_first(int c, int n_frames, int n_chunks) {
    return (int)(((long long)c * n_frames) / n_chunks);
}
struct WsItem {  // one (strip, chunk) of the launch
    int f0, nf;          // first frame, frames
    int px0, valid_px;   // first pixel, pixels (a multiple of 16)
    int it_begin;        // 0: the walk starts with the predecessor (halo) frame, 1: it has none
    int slots;           // frames walked, padded to a multiple of the unroll factor
    int walked;          // frames walked (halo included)
};
__device__ __forceinline__ WsItem ws_item(const ScoreArgs& a, int item) {
    WsItem w;
    const int chunk = item % a.n_chunks;  // chunk-fastest: CTAs running side by side are on different frames
    const int strip = item / a.n_chunks;
    w.f0 = chunk_first(chunk, a.n_frames, a.n_chunks);
    w.nf = chunk_first(chunk + 1, a.n_frames, a.n_chunks) - w.f0;
    w.px0 = strip * kWsStripPx;
    w.valid_px = min(kWsStripPx, a.n_pixels - w.px0) & ~15;  // the tail kernel takes the last P mod 16 pixels
    const bool have_halo = (a.features & PSD_F_HSV) && (w.f0 > 0 || a.prev != nullptr);
    w.it_begin = have_halo ? 0 : 1;
    w.walked = w.nf + 1 - w.it_begin;
    w.slots = (w.walked + kWsUnroll - 1) / kWsUnroll * kWsUnroll;
    return w;
}

struct WsAddr {  // shared-window addresses of the current loop body's first stage
    uint32_t ring;   // + tid * 48
    uint32_t full;   // FULL mbarrier of the stage; EMPTY mbarriers follow kWsStages * 8 bytes later
    uint32_t acc;    // per-lane accumulators of the stage (this lane's word of channel 0; or the sink's)
};

// One frame of the consumer loop at stage (body base + J).  `sad_acc`: accumulator base the SADs go to (the
// stage's real per-lane words, or the sink); `mine`: the frame is not the halo and the thread owns pixels.
template <uint32_t F, int J>
__device__ __forceinline__ void ws_step(const ScoreArgs& a, WsSmem& sm, const WsAddr& ad, uint32_t parity, int stage0,
                                        uint32_t sad_acc, bool mine, int fi, int my_px, int lane, uint32_t zero,
                                        const LutView7& lut7, const Px16& prev, Px16& cur) {
    constexpr bool kHSV = (F & PSD_F_HSV) != 0;
    constexpr bool kSUM = (F & PSD_F_BGRSUM) != 0;
    constexpr bool kYH = (F & PSD_F_YHIST) != 0;
    constexpr bool kEDGE = (F & PSD_F_EDGES) != 0;
    // HSV pass (issue-bound), even frame of a body: check this frame's and the next frame's barrier back to back,
    // so the latency of the second check hides behind the first; the odd frame then finds its data without asking
    // again.  The byte-sum and histogram passes are bandwidth-bound: waiting for two stages before touching the
    // first would halve their effective ring depth (histogram: 0.85 of the roofline against 0.95), so they wait
    // stage by stage.
    if (kHSV) {
        if ((J & 1) == 0) {
            mbar_wait_hint_off<J * 8>(ad.full, parity);
            mbar_wait_hint_off<J * 8 + 8>(ad.full, parity);
        }
    } else {
        mbar_wait_hint_off<J * 8>(ad.full, parity);
    }
    uint32_t w[12];
    // idle threads of a partial last strip read stale ring bytes; they never contribute (sink / mine)
    lds128_off<J * kWsStripBytes>(ad.ring, w[0], w[1], w[2], w[3]);
    lds128_off<J * kWsStripBytes + 16>(ad.ring, w[4], w[5], w[6], w[7]);
    lds128_off<J * kWsStripBytes + 32>(ad.ring, w[8], w[9], w[10], w[11]);
    if (kHSV) {
        hsv16_v7(w, cur, lut7);
        // one dependent VABSDIFF4.ACC chain per plane (the compiler otherwise splits each into four
        // zero-seeded accumulators plus an IADD3 tree: 12 extra issue slots per frame)
        uint32_t sad_h = sad4_acc(cur.h[0], prev.h[0], zero), sad_s = sad4_acc(cur.s[0], prev.s[0], zero),
                 sad_v = sad4_acc(cur.v[0], prev.v[0], zero);
#pragma unroll
        for (int j = 1; j < 4; ++j) {
            sad_h = sad4_acc(cur.h[j], prev.h[j], sad_h);
            sad_s = sad4_acc(cur.s[j], prev.s[j], sad_s);
            sad_v = sad4_acc(cur.v[j], prev.v[j], sad_v);
        }
        // never predicated: threads whose SADs do not count (no pixels, no predecessor frame) were handed the
        // address of the sink accumulators instead
        red_shared_add_off<J * 512>(sad_acc, sad_h);
        red_shared_add_off<J * 512 + 128>(sad_acc, sad_s);
        red_shared_add_off<J * 512 + 256>(sad_acc, sad_v);
        if (kEDGE && mine) {
            uint8_t* vp = a.vplane + (int64_t)fi * a.n_pixels + my_px;
            if ((a.n_pixels & 15) == 0) {
                *reinterpret_cast<uint4*>(vp) = make_uint4(cur.v[0], cur.v[1], cur.v[2], cur.v[3]);
            } else {
                for (int p = 0; p < kPxPerThread; ++p) vp[p] = (uint8_t)(cur.v[p >> 2] >> ((p & 3) * 8));
            }
            // bin address = histogram base + 4 * byte: one IDP4A with the weight 4 on the pixel's byte
            const uint32_t vh = smem_u32(sm.vhist[stage0 + J]);
#pragma unroll
            for (int p = 0; p < kPxPerThread; ++p)
                red_shared_add_off<0>(__dp4a(cur.v[p >> 2], 4u << ((p & 3) * 8), vh), 1u);
        }
    }
    if (mine) {
        if (kSUM) {
            uint32_t bsum = 0;
#pragma unroll
            for (int j = 0; j < 12; ++j) bsum = __dp4a(w[j], 0x01010101u, bsum);
            red_shared_add_off<J * 512 + 384>(ad.acc, bsum);
        }
        if (kYH) {
            uint32_t* hist = sm.yhist[stage0 + J];
#define PSD_YH(i) atomicAdd(&hist[y_of_pixel<i>(w)], 1u);
            PSD_YH(0) PSD_YH(1) PSD_YH(2) PSD_YH(3) PSD_YH(4) PSD_YH(5) PSD_YH(6) PSD_YH(7)
            PSD_YH(8) PSD_YH(9) PSD_YH(10) PSD_YH(11) PSD_YH(12) PSD_YH(13) PSD_YH(14) PSD_YH(15)
#undef PSD_YH
        }
    }
    // no __syncwarp() in front of lane 0's EMPTY arrival: the warp is converged here (every branch of the step
    // is closed by the compiler's BSSY/BSYNC pair), its lanes' LDS results were consumed by the arithmetic above
    // and its shared REDs entered the same in-order shared-memory pipe before the arrival does
    if (lane == 0) mbar_arrive_off<kWsStages * 8 + J * 8>(ad.full);
}

// A padding slot: nothing was copied, the consumers only hand the stage back.
template <int J>
__device__ __forceinline__ void ws_null_step(const WsAddr& ad, uint32_t parity, int lane) {
    mbar_wait_hint_off<J * 8>(ad.full, parity);
    if (lane == 0) mbar_arrive_off<kWsStages * 8 + J * 8>(ad.full);
}

template <uint32_t F>
__global__ void __launch_bounds__(kWsThreads, 1) psd_score_ws_kernel(const ScoreArgs a) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    WsSmem& sm = *reinterpret_cast<WsSmem*>(smem_raw);
    constexpr bool kHSV = (F & PSD_F_HSV) != 0;
    constexpr bool kSUM = (F & PSD_F_BGRSUM) != 0;
    constexpr bool kYH = (F & PSD_F_YHIST) != 0;
    constexpr bool kEDGE = (F & PSD_F_EDGES) != 0;
    constexpr int U = kWsUnroll;

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int n_items = a.n_chunks * a.n_strips;

    for (int i = tid; i < kWsStages * 256; i += kWsThreads) {
        (&sm.yhist[0][0])[i] = 0;
        (&sm.vhist[0][0])[i] = 0;
    }
    for (int i = tid; i < kWsStages * 4 * 32; i += kWsThreads) {
        (&sm.accl[0][0][0])[i] = 0;
        (&sm.accl_sink[0][0][0])[i] = 0;
    }
    if (kHSV) lut_fill7(sm.lut, tid, kWsThreads);
    if (tid == 0) {
        for (int s = 0; s < kWsStages; ++s) {
            mbar_init(&sm.full[s], 1);
            mbar_init(&sm.empty[s], kWsConsumerWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid >= kWsConsumers) {
        // ===================== side warps =====================
        // Cursors over this CTA's slot sequence (items of this CTA, slots of each item).  Every item has a
        // multiple of kWsStages slots, so slot k of an item always sits in stage k mod kWsStages: side warp
        // `rs` owns slots rs, rs + kWsStages, ... of every item.  It retires them (`ret`) and re-arms its
        // stage with the slot kWsStages further on (`iss`, one lap of the ring ahead of `ret`).
        struct Cursor {
            int item, slot;
            WsItem w;
        };
        const int rs = (tid - kWsConsumers) >> 5;  // the stage this warp owns (= its SM sub-partition)
        auto load = [&](Cursor& c) { if (c.item < n_items) c.w = ws_item(a, c.item); };
        auto advance = [&](Cursor& c) {
            c.slot += kWsStages;
            if (c.slot >= c.w.slots) { c.slot = rs; c.item += gridDim.x; load(c); }
        };
        auto issue = [&](Cursor& c) {
            if (lane == 0) {
                if (c.slot < c.w.walked) {
                    const int fi = c.w.f0 - 1 + c.w.it_begin + c.slot;
                    const uint8_t* src = (fi < 0 ? a.prev : a.frames + (int64_t)fi * a.frame_stride) + (int64_t)c.w.px0 * 3;
                    const uint32_t bytes = (uint32_t)c.w.valid_px * 3u;
                    mbar_expect_tx(&sm.full[rs], bytes);
                    bulk_g2s(sm.ring[rs], src, bytes, &sm.full[rs]);
                } else {
                    mbar_arrive_off<0>(smem_u32(&sm.full[rs]));  // padding slot: complete the phase without a copy
                }
            }
            advance(c);
        };
        Cursor ret{(int)blockIdx.x, rs, {}};
        load(ret);
        Cursor iss = ret;
        issue(iss);
        uint32_t parity = 0;
        while (ret.item < n_items) {
            mbar_wait_hint(&sm.empty[rs], parity);
            const int it = ret.w.it_begin + ret.slot;             // 0 = halo frame
            const bool real = ret.slot < ret.w.walked;
            const bool own = real && it >= 1;                     // this CTA accounts for frame fi
            const int fi = ret.w.f0 - 1 + it;
            // the per-lane totals are taken and zeroed BEFORE the stage is re-armed: no consumer can add the
            // next frame of this stage to them until the copy issued below has landed
            uint32_t tot[4] = {0u, 0u, 0u, 0u};
            if (own && (kHSV || kSUM)) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if ((c < 3 && kHSV) || (c == 3 && kSUM)) {
                        tot[c] = sm.accl[rs][c][lane];
                        sm.accl[rs][c][lane] = 0;
                    }
                }
            }
            if (own) {
                if (kYH) {
#pragma unroll
                    for (int b = lane; b < 256; b += 32) {
                        const uint32_t v = sm.yhist[rs][b];
                        if (v) { sm.yhist[rs][b] = 0; atomicAdd(&a.yhist[(int64_t)fi * 256 + b], v); }
                    }
                }
                if (kEDGE) {
#pragma unroll
                    for (int b = lane; b < 256; b += 32) {
                        const uint32_t v = sm.vhist[rs][b];
                        if (v) { sm.vhist[rs][b] = 0; atomicAdd(&a.vhist[(int64_t)fi * 256 + b], v); }
                    }
                }
                if (ret.item < a.n_chunks && lane == 0)  // an item of strip 0
                    a.sums[fi].has_prev = (fi > 0 || a.prev != nullptr) ? 1ull : 0ull;
            }
            __syncwarp();  // the zeroing above is ordered before lane 0 re-arms the stage
            if (iss.item < n_items) issue(iss);
            if (own && (kHSV || kSUM)) {  // after the re-arm: the copy engine's queue is fed first
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if ((c < 3 && !kHSV) || (c == 3 && !kSUM)) continue;
                    const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, tot[c]);
                    if (lane == 0 && v)
                        atomicAdd(reinterpret_cast<unsigned long long*>(&a.sums[fi]) + (c < 3 ? c : 4),
                                  (unsigned long long)v);
                }
            }
            advance(ret);
            parity ^= 1u;
        }
        return;
    }

    // ===================== consumer warps =====================
    const LutView7 lut7 = make_lut7(smem_u32(sm.lut), lane);
    // a zero the compiler cannot see through: it stays in one register for the whole loop instead of
    // being re-materialised (CS2R) in front of every accumulation chain
    const uint32_t zero = a.shift24 ^ 0x01000000u;
    const uint32_t ring0 = smem_u32(sm.ring[0]) + tid * 48;
    const uint32_t full0 = smem_u32(&sm.full[0]);
    const uint32_t accl0 = smem_u32(&sm.accl[0][0][lane]);
    const uint32_t sink0 = smem_u32(&sm.accl_sink[0][0][lane]);
    int stage0 = 0;        // first stage of the current body
    uint32_t parity = 0;
    WsAddr ad{ring0, full0, 0u};
    auto next_body = [&](uint32_t acc0) {
        stage0 += U;
        if (stage0 == kWsStages) {
            stage0 = 0;
            parity ^= 1u;
            ad.ring = ring0; ad.full = full0; ad.acc = acc0;
        } else {
            ad.ring += U * kWsStripBytes; ad.full += U * 8; ad.acc += U * 512;
        }
    };
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const WsItem wi = ws_item(a, item);
        const int my_px = wi.px0 + tid * kPxPerThread;
        const bool active = tid * kPxPerThread < wi.valid_px;  // only the last strip has idle threads
        // threads without pixels add to the sink for the whole walk; everybody does for the frame without predecessor
        const uint32_t acc0 = active ? accl0 : sink0;
        ad.acc = acc0 + stage0 * 512;
        Px16 P0, P1;
#pragma unroll
        for (int j = 0; j < 4; ++j) P0.h[j] = P0.s[j] = P0.v[j] = P1.h[j] = P1.s[j] = P1.v[j] = 0;
        const int n = wi.walked;                      // frames walked (halo included)
        const int fbase = wi.f0 - 1 + wi.it_begin;    // frame index of k == 0
        int k = 0;
        uint32_t acc_first = sink0 + stage0 * 512;    // k == 0: no predecessor
#pragma unroll 1
        for (; k + U <= n; k += U) {
            const bool first_mine = active && (wi.it_begin + k >= 1);
            ws_step<F, 0>(a, sm, ad, parity, stage0, acc_first, first_mine, fbase + k, my_px, lane, zero, lut7, P0, P1);
            ws_step<F, 1>(a, sm, ad, parity, stage0, ad.acc, active, fbase + k + 1, my_px, lane, zero, lut7, P1, P0);
            ws_step<F, 2>(a, sm, ad, parity, stage0, ad.acc, active, fbase + k + 2, my_px, lane, zero, lut7, P0, P1);
            ws_step<F, 3>(a, sm, ad, parity, stage0, ad.acc, active, fbase + k + 3, my_px, lane, zero, lut7, P1, P0);
            next_body(acc0);
            acc_first = ad.acc;
        }
        if (k < n) {  // last, partial body of the item: real frames first, then the padding slots
            const int r = n - k;  // 1 .. U-1
            ws_step<F, 0>(a, sm, ad, parity, stage0, acc_first, active && (wi.it_begin + k >= 1), fbase + k, my_px,
                              lane, zero, lut7, P0, P1);
            if (r > 1) ws_step<F, 1>(a, sm, ad, parity, stage0, ad.acc, active, fbase + k + 1, my_px, lane, zero, lut7, P1, P0);
            else ws_null_step<1>(ad, parity, lane);
            if (r > 2) ws_step<F, 2>(a, sm, ad, parity, stage0, ad.acc, active, fbase + k + 2, my_px, lane, zero, lut7, P0, P1);
            else ws_null_step<2>(ad, parity, lane);
            ws_null_step<3>(ad, parity, lane);
            next_body(acc0);
        }
    }
}

// Number of time chunks: the walk costs (frames + 1 halo) per item and the launch ends when the most
// loaded SM is done, so minimise ceil(strips * C / grid) * (N / C + 1) over C.
static int pick_chunks(int n_frames, int n_strips, int grid) {
    long long best_cost = -1;
    int best = 1;
    const int c_max = n_frames < 4096 ? n_frames : 4096;
    for (int c = 1; c <= c_max; ++c) {
        const int longest = (n_frames + c - 1) / c;
        if (longest < 8 && c > 1) break;  // shorter walks only add halo frames
        const long long per_cta = ((long long)n_strips * c + grid - 1) / grid;
        const long long cost = per_cta * (longest + 1);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = c; }
    }
    return best;
}

template <uint32_t F>
static int launch_ws(ScoreArgs a, int n_ws_strips, cudaStream_t stream) {
    const int smem = (int)sizeof(WsSmem);
    static int sm_count = 0;
    if (sm_count == 0) {
        int dev = 0;
        PSD_CUDA(cudaGetDevice(&dev));
        PSD_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    }
    PSD_CUDA(cudaFuncSetAttribute(psd_score_ws_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    a.shift24 = 0x01000000u;
    a.features = F;
    a.n_strips = n_ws_strips;
    a.n_chunks = pick_chunks(a.n_frames, n_ws_strips, sm_count);
    if (a.n_chunks > a.n_frames) a.n_chunks = a.n_frames;
    const int64_t items = (int64_t)a.n_chunks * n_ws_strips;
    PSD_REQUIRE(items > 0 && items < 2147483647LL, "score work items out of range (%lld)", (long long)items);
    const int grid = (int)(items < sm_count ? items : sm_count);
    psd_score_ws_kernel<F><<<grid, kWsThreads, smem, stream>>>(a);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

static int dispatch_ws(const ScoreArgs& a, uint32_t f, int n_ws_strips, cudaStream_t s) {
    switch (f & 15u) {
#define CASE(F) case F: return launch_ws<F>(a, n_ws_strips, s);
        CASE(1) CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7)
        CASE(9) CASE(11) CASE(13) CASE(15)
#undef CASE
        default:
            set_error("unsupported feature mask 0x%x", f);
            return PSD_ERR_INVALID;
    }
}

// ---------------------------------------------------------------------------------------------
// Tail kernel: the last P - P16 (1 .. 15) pixels of every frame, one thread per frame.  The thread loads
// this frame's and the predecessor's tail bytes into zero-filled words and runs the warp-specialised kernel's
// HSV arithmetic on them; the zero padding is black in both frames, so the padded pixels add nothing to the
// SADs or the byte sum, and the histograms and the V plane only take the valid pixels.
// ---------------------------------------------------------------------------------------------
constexpr int kTailThreads = 128;
constexpr int kLutBytes = 256 * 64 * 4;

__device__ __forceinline__ void load_tail(const uint8_t* src, int n_bytes, uint32_t (&w)[12]) {
#pragma unroll
    for (int j = 0; j < 12; ++j) w[j] = 0;
#pragma unroll
    for (int k = 0; k < 48; ++k)
        if (k < n_bytes) w[k >> 2] |= (uint32_t)src[k] << ((k & 3) * 8);
}

__global__ void __launch_bounds__(kTailThreads) psd_score_tail_kernel(const ScoreArgs a) {
    extern __shared__ __align__(128) float lut[];
    const bool hsv = (a.features & PSD_F_HSV) != 0;
    if (hsv) lut_fill7(lut, threadIdx.x, blockDim.x);
    __syncthreads();
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= a.n_frames) return;
    const int p16 = a.n_pixels & ~15, n = a.n_pixels - p16;
    const uint8_t* prev = fi > 0 ? a.frames + (int64_t)(fi - 1) * a.frame_stride : a.prev;
    uint32_t w[12];
    load_tail(a.frames + (int64_t)fi * a.frame_stride + (int64_t)p16 * 3, 3 * n, w);
    unsigned long long* sums = reinterpret_cast<unsigned long long*>(&a.sums[fi]);
    if (hsv) {
        const LutView7 lut7 = make_lut7(smem_u32(lut), threadIdx.x & 31);
        Px16 cur;
        hsv16_v7(w, cur, lut7);
        if (prev) {
            uint32_t wp[12];
            load_tail(prev + (int64_t)p16 * 3, 3 * n, wp);
            Px16 pre;
            hsv16_v7(wp, pre, lut7);
            uint32_t sad_h = 0, sad_s = 0, sad_v = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                sad_h = __vsadu4(cur.h[j], pre.h[j]) + sad_h;
                sad_s = __vsadu4(cur.s[j], pre.s[j]) + sad_s;
                sad_v = __vsadu4(cur.v[j], pre.v[j]) + sad_v;
            }
            atomicAdd(sums + 0, (unsigned long long)sad_h);
            atomicAdd(sums + 1, (unsigned long long)sad_s);
            atomicAdd(sums + 2, (unsigned long long)sad_v);
        }
        if (a.features & PSD_F_EDGES) {
            uint8_t* vp = a.vplane + (int64_t)fi * a.n_pixels + p16;
            for (int p = 0; p < n; ++p) {
                const uint32_t v = (cur.v[p >> 2] >> ((p & 3) * 8)) & 0xFFu;
                vp[p] = (uint8_t)v;
                atomicAdd(&a.vhist[(int64_t)fi * 256 + v], 1u);
            }
        }
    }
    if (a.features & PSD_F_BGRSUM) {
        uint32_t bsum = 0;
#pragma unroll
        for (int j = 0; j < 12; ++j) bsum = __dp4a(w[j], 0x01010101u, bsum);
        atomicAdd(sums + 4, (unsigned long long)bsum);
    }
    if (a.features & PSD_F_YHIST) {
        for (int p = 0; p < n; ++p)
            atomicAdd(&a.yhist[(int64_t)fi * 256 + y_px(byte_of(w, 3 * p), byte_of(w, 3 * p + 1), byte_of(w, 3 * p + 2))],
                      1u);
    }
    if (p16 == 0) a.sums[fi].has_prev = (fi > 0 || a.prev != nullptr) ? 1ull : 0ull;  // else the ws kernel writes it
}

static int launch_tail(ScoreArgs a, uint32_t features, cudaStream_t stream) {
    PSD_CUDA(cudaFuncSetAttribute(psd_score_tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLutBytes));
    a.features = features;
    const int grid = (a.n_frames + kTailThreads - 1) / kTailThreads;
    psd_score_tail_kernel<<<grid, kTailThreads, (features & PSD_F_HSV) ? kLutBytes : 0, stream>>>(a);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

int launch_score(const ScoreArgs& a, uint32_t features, cudaStream_t stream) {
    if (features & PSD_F_EDGES) features |= PSD_F_HSV;
    PSD_REQUIRE(a.n_frames > 0 && a.n_pixels > 0, "empty score launch");
    const uintptr_t al = reinterpret_cast<uintptr_t>(a.frames) | (uintptr_t)a.frame_stride |
                         reinterpret_cast<uintptr_t>(a.prev);
    PSD_REQUIRE((al & 15) == 0, "score pass input is not 16-byte aligned");
    const int p16 = a.n_pixels & ~15;
    if (p16 > 0) {
        const int rc = dispatch_ws(a, features, (p16 + kWsStripPx - 1) / kWsStripPx, stream);
        if (rc) return rc;
    }
    if (p16 < a.n_pixels) return launch_tail(a, features, stream);
    return PSD_OK;
}

// ---- test hook: the fused pass's device functions on a flat pixel array ----
__global__ void psd_test_hsv_kernel(const uint8_t* bgr, int64_t n_groups, uint8_t* h, uint8_t* s,
                                    uint8_t* v, uint8_t* y) {
    extern __shared__ __align__(128) float lutmem[];
    lut_fill7(lutmem, threadIdx.x, blockDim.x);
    const LutView7 lut7 = make_lut7(smem_u32(lutmem), threadIdx.x & 31);
    __syncthreads();
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_groups;
         g += (int64_t)gridDim.x * blockDim.x) {
        uint32_t w[12];
        const uint4* p = reinterpret_cast<const uint4*>(bgr + g * 48);
        const uint4 q0 = p[0], q1 = p[1], q2 = p[2];
        w[0] = q0.x; w[1] = q0.y; w[2] = q0.z; w[3] = q0.w;
        w[4] = q1.x; w[5] = q1.y; w[6] = q1.z; w[7] = q1.w;
        w[8] = q2.x; w[9] = q2.y; w[10] = q2.z; w[11] = q2.w;
        Px16 o;
        hsv16_v7(w, o, lut7);
        *reinterpret_cast<uint4*>(h + g * 16) = make_uint4(o.h[0], o.h[1], o.h[2], o.h[3]);
        *reinterpret_cast<uint4*>(s + g * 16) = make_uint4(o.s[0], o.s[1], o.s[2], o.s[3]);
        *reinterpret_cast<uint4*>(v + g * 16) = make_uint4(o.v[0], o.v[1], o.v[2], o.v[3]);
        for (int px = 0; px < 16; ++px)
            y[g * 16 + px] = (uint8_t)y_px(byte_of(w, 3 * px), byte_of(w, 3 * px + 1), byte_of(w, 3 * px + 2));
    }
}

}  // namespace psd

extern "C" int psd_test_hsv(int device, const uint8_t* bgr_host, int64_t n_pixels, uint8_t* h_out,
                            uint8_t* s_out, uint8_t* v_out, uint8_t* y_out) {
    using namespace psd;
    PSD_REQUIRE(n_pixels > 0 && (n_pixels % 16) == 0, "n_pixels must be a positive multiple of 16");
    PSD_CUDA(cudaSetDevice(device));
    int sm_count = 0;
    PSD_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
    uint8_t *d_bgr = nullptr, *d_out = nullptr;
    PSD_CUDA(cudaMalloc(&d_bgr, (size_t)n_pixels * 3));
    PSD_CUDA(cudaMalloc(&d_out, (size_t)n_pixels * 4));
    PSD_CUDA(cudaMemcpy(d_bgr, bgr_host, (size_t)n_pixels * 3, cudaMemcpyHostToDevice));
    uint8_t* dh = d_out;
    uint8_t* ds = d_out + n_pixels;
    uint8_t* dv = d_out + 2 * n_pixels;
    uint8_t* dy = d_out + 3 * n_pixels;
    PSD_CUDA(cudaFuncSetAttribute(psd_test_hsv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLutBytes));
    psd_test_hsv_kernel<<<sm_count * 2, 256, kLutBytes>>>(d_bgr, n_pixels / 16, dh, ds, dv, dy);
    PSD_CHECK_LAUNCH();
    count_launch();
    PSD_CUDA(cudaDeviceSynchronize());
    PSD_CUDA(cudaMemcpy(h_out, dh, (size_t)n_pixels, cudaMemcpyDeviceToHost));
    PSD_CUDA(cudaMemcpy(s_out, ds, (size_t)n_pixels, cudaMemcpyDeviceToHost));
    PSD_CUDA(cudaMemcpy(v_out, dv, (size_t)n_pixels, cudaMemcpyDeviceToHost));
    PSD_CUDA(cudaMemcpy(y_out, dy, (size_t)n_pixels, cudaMemcpyDeviceToHost));
    cudaFree(d_bgr);
    cudaFree(d_out);
    return PSD_OK;
}
