// Edge component of ContentDetector (content_detector.py:213-239):
//   median = numpy.median(V);  low/high = int(max(0,(1-s)*median)), int(min(255,(1+s)*median)), s = 1/3
//   edges  = cv2.dilate(cv2.Canny(V, low, high), ones(k,k))
//   delta_edges = mean |edges_t - edges_{t-1}|                       (content_detector.py:171-175)
// Canny is restated from OpenCV's algorithm (aperture 3, L1 gradient): Sobel 3x3 with
// BORDER_REPLICATE, fixed-point non-maximum suppression (TG22 = 13573), double threshold with
// strict '>' and 8-connected hysteresis.  oracle/intmath.py:canny is the CPU twin pinned
// against cv2.Canny.
//
// Everything after the gradient stage works on BIT-PACKED maps (32 pixels per word, bit i of word
// (y, wq) = pixel 32 wq + i; padding bits are 0), 1/8 byte per pixel and plane:
//   thresholds (V histogram of the fused pass)                                   [1 launch]
//   -> classify: Sobel / L1 magnitude / NMS / double threshold straight into two bit planes,
//      E = strong pixels, C = candidates (weak or strong), both tile-major      [1 launch]
//   -> hysteresis: E grows inside C until nothing changes, bit-parallel          [1 cooperative launch]
//   -> k x k max on the bits in one pass (k <= 17) or two separable passes (k >= 19),
//      popcount SAD against the previous frame                                   [2 - 3 launches]
// (the first version kept a byte class map, 4-byte union-find labels per pixel and 12 launches per
// batch).
#include <cooperative_groups.h>

#include "canny_pairs.cuh"
#include "psd_common.cuh"

namespace cg = cooperative_groups;

// classify launch shape: 128 threads x 3 CTAs per SM = 163 registers, no spills (256 x 2 caps at 128 registers
// and spills ~50 words; measured 3-4 % slower)
constexpr int kClassifyBlock = 128;

namespace psd {

// ---- 1. per-frame Canny thresholds from the V histogram ----
// one warp per frame: lane l owns bins 8l .. 8l+7; an inclusive warp scan of the lane totals locates the two
// order statistics
__global__ void psd_edge_thresholds_kernel(const uint32_t* __restrict__ vhist, int n, int64_t n_pixels,
                                           int32_t* __restrict__ thr) {
    const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (f >= n) return;
    const uint4* h4 = reinterpret_cast<const uint4*>(vhist + (int64_t)f * 256) + 2 * lane;
    const uint4 a = h4[0], b = h4[1];
    const uint32_t bins[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t own = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) own += bins[i];
    uint32_t incl = own;   // a frame has fewer than 2^32 pixels
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl += up;
    }
    // numpy.median: mean of the order statistics (n-1)//2 and n//2 (0-based)
    const int64_t r_lo = (n_pixels - 1) / 2 + 1, r_hi = n_pixels / 2 + 1;
    int64_t cum = (int64_t)incl - own;
    int lo_l = -1, hi_l = -1;   // first bin of this lane whose cumulative count reaches the rank
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t before = cum;
        cum += bins[i];
        if (before < r_lo && cum >= r_lo) lo_l = 8 * lane + i;
        if (before < r_hi && cum >= r_hi) hi_l = 8 * lane + i;
    }
    // exactly one lane sees each crossing
    const int lo = __reduce_max_sync(0xFFFFFFFFu, lo_l), hi = __reduce_max_sync(0xFFFFFFFFu, hi_l);
    if (lane != 0) return;
    const double median = __ddiv_rn((double)(lo + hi), 2.0);
    const double sigma = __ddiv_rn(1.0, 3.0);
    const double lo_d = __dmul_rn(__dsub_rn(1.0, sigma), median);
    const double hi_d = __dmul_rn(__dadd_rn(1.0, sigma), median);
    int low = (int)(lo_d > 0.0 ? lo_d : 0.0);       // int(max(0, x)) truncates
    int high = (int)(hi_d < 255.0 ? hi_d : 255.0);  // int(min(255, x))
    if (low > high) { const int t = low; low = high; high = t; }  // cv2.Canny swaps
    thr[2 * f] = low;
    thr[2 * f + 1] = high;
}

// ---- 2. Sobel + L1 magnitude + NMS + double threshold -> bit planes ----
// One thread owns 8 consecutive columns (one byte of each bit plane per row) and marches down a band of
// kBandRows rows; everything it needs from neighbouring rows stays in registers.  The arithmetic is done on
// pixel PAIRS, two 16-bit lanes per register (canny_pairs.cuh).  No shared memory, no shuffles, no barrier;
// neighbouring threads re-read overlapping words from L1.  (Round 2's first version of this kernel kept one
// pixel per 32-bit register - IDP4A row sums, integer NMS: 476 instructions per 8-pixel row against 281,
// earlier A/B runs.)
//
// The two planes it writes are TILE-MAJOR: tile (ty, tx) = rows 32 ty .. 32 ty + 31 x columns 64 tx .. 64 tx + 63
// is 64 consecutive words, row r of the tile at words 2 r and 2 r + 1.  A warp of the hysteresis kernel then
// pulls its whole tile with one 256-byte request instead of 32 row fragments 4 Wq bytes apart.  Words and
// rows beyond the image are never written by anyone and stay 0 from the allocation.
constexpr int kBandRows = 32;   // == kHystTileH: a band of the classify kernel is one tile row of the hysteresis
constexpr int kTileWords = 64;  // 32 rows x 2 words

template <bool ALIGNED>
__global__ void __launch_bounds__(kClassifyBlock, 3) psd_canny_classify_pairs_kernel(
    const uint8_t* __restrict__ vplane, const int32_t* __restrict__ thr, uint32_t* __restrict__ edge_bits,
    uint32_t* __restrict__ cand_bits, uint8_t* __restrict__ tile_dirty, int W, int H, int Wq, int strips,
    int bands, int64_t n_threads) {
    const int64_t gid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (gid >= n_threads) return;
    const int sx = (int)(gid % strips);
    const int by = (int)((gid / strips) % bands);
    const int64_t f = gid / ((int64_t)strips * bands);
    const int64_t P = (int64_t)W * H;
    const uint8_t* src = vplane + f * P;
    // this band's tile of the planes: byte (sx & 7) of each of its 32 rows (8 bytes per row)
    const int tiles_x = (Wq + 1) / 2;
    const int64_t tile = (f * bands + by) * (int64_t)tiles_x + (sx >> 3);
    const int yb = by * kBandRows, ye = min(yb + kBandRows, H);
    uint8_t* eout = reinterpret_cast<uint8_t*>(edge_bits + tile * kTileWords) + (sx & 7) - (int64_t)yb * 8;
    uint8_t* cout = reinterpret_cast<uint8_t*>(cand_bits + tile * kTileWords) + (sx & 7) - (int64_t)yb * 8;
    const uint32_t low1 = cp::scaled2(thr[2 * f] + 1), high1 = cp::scaled2(thr[2 * f + 1] + 1);
    const int x0 = sx * 8;
    // lanes of the pairs that lie inside the image (gradients outside are zero: cv2 pads the magnitude buffer)
    uint32_t inO[4], inL[5];
#pragma unroll
    for (int k = 0; k < 4; ++k)
        inO[k] = (x0 + 2 * k < W ? 0x0000FFFFu : 0u) | (x0 + 2 * k + 1 < W ? 0xFFFF0000u : 0u);
#pragma unroll
    for (int k = 0; k < 5; ++k)
        inL[k] = ((x0 + 2 * k - 1 >= 0 && x0 + 2 * k - 1 < W) ? 0x0000FFFFu : 0u) | (x0 + 2 * k < W ? 0xFFFF0000u : 0u);

    // the 16 bytes x0-4 .. x0+11 of row y (BORDER_REPLICATE in both directions)
    auto load_window = [&](int y, uint32_t (&w)[4]) {
        const int yc = min(max(y, 0), H - 1);
        const uint8_t* row = src + (int64_t)yc * W;
        if (ALIGNED) {  // W % 8 == 0: every strip is whole, words are 4-byte aligned
            const uint2 mid = *reinterpret_cast<const uint2*>(row + x0);
            const uint32_t* rw = reinterpret_cast<const uint32_t*>(row) + 2 * sx;
            w[1] = mid.x;
            w[2] = mid.y;
            w[0] = (sx > 0) ? rw[-1] : __byte_perm(w[1], 0, 0x0000);        // replicate column 0
            w[3] = (x0 + 8 < W) ? rw[2] : __byte_perm(w[2], 0, 0x3333);     // replicate column W-1
        } else {
            w[0] = w[1] = w[2] = w[3] = 0;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const int x = min(max(x0 - 4 + k, 0), W - 1);
                w[k >> 2] |= (uint32_t)row[x] << (8 * (k & 3));
            }
        }
    };
    // Row yy+1 arrives: magnitudes (and, if asked, sectors) of row yy from the sums of rows yy-1 (`so`,
    // replaced by row yy+1 on the way out), yy (`sm`) and yy+1.
    uint32_t wn[4];   // the window of the next row to arrive, loaded one row early
    auto advance = [&](int yy, cp::Sums& so, const cp::Sums& sm, cp::Mags& r, bool want_sectors) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) w[i] = wn[i];
        load_window(yy + 2, wn);
        // the first touch of a row goes to L2 / HBM and four warps per scheduler cannot hide that: pull the line
        // of the row two further down into L1 now (no register, no dependency; +4 % on the edge path)
        if (yy + 3 < H) asm volatile("prefetch.global.L1 [%0];" ::"l"(src + (int64_t)(yy + 3) * W + x0));
        cp::Sums sn;
        cp::row_sums(w, sn);
        uint32_t gxO[4], gyO[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            gxO[k] = cp::hadd(cp::hfma(sm.cO[k], cp::kTwo, so.cO[k]), sn.cO[k]);
            gyO[k] = cp::hsub(sn.hO[k], so.hO[k]);
            r.mO[k] = cp::habs_sum(gxO[k], gyO[k]);
            if (!ALIGNED) r.mO[k] &= inO[k];
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const uint32_t gx = cp::hadd(cp::hfma(sm.cL[k], cp::kTwo, so.cL[k]), sn.cL[k]);
            const uint32_t gy = cp::hsub(sn.hL[k], so.hL[k]);
            r.mL[k] = cp::habs_sum(gx, gy);
            if (!ALIGNED || k == 0 || k == 4) r.mL[k] &= inL[k];
        }
        if (yy < 0 || yy >= H) {   // rows above / below the image
#pragma unroll
            for (int k = 0; k < 4; ++k) r.mO[k] = 0;
#pragma unroll
            for (int k = 0; k < 5; ++k) r.mL[k] = 0;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) r.pO[k] = cp::hadd(r.mO[k], cp::kOne);
#pragma unroll
        for (int k = 0; k < 5; ++k) r.pL[k] = cp::hadd(r.mL[k], cp::kOne);
        so = sn;
        const uint32_t top = cp::umax3(cp::umax3(r.pO[0], r.pO[1], r.pO[2]), r.pO[3], 0u);
        r.any = cp::hgt_mask(top, low1) != 0u;
        if (want_sectors && r.any) {
#pragma unroll
            for (int k = 0; k < 4; ++k) cp::sector(gxO[k], gyO[k], r.dlo[k], r.dhi[k]);
        }
    };
    uint32_t weak_seen = 0;   // some candidate of this band is not strong: its tile needs hysteresis
    // output row y from the magnitude rows y-1 (`u`), y (`c`), y+1 (`d`)
    auto emit = [&](int y, const cp::Mags& u, const cp::Mags& c, const cp::Mags& d) {
        uint32_t ebyte = 0, cbyte = 0;
        if (c.any) {
            uint32_t acc_c = 0, acc_e = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t n_h = cp::umax3(c.pL[k], c.mL[k + 1], low1);      // m > left,  m >= right
                const uint32_t n_v = cp::umax3(u.pO[k], d.mO[k], low1);          // m > above, m >= below
                const uint32_t n_d1 = cp::umax3(u.pL[k], d.pL[k + 1], low1);     // (y-1,x-1) / (y+1,x+1)
                const uint32_t n_d2 = cp::umax3(u.pL[k + 1], d.pL[k], low1);     // (y-1,x+1) / (y+1,x-1)
                const uint32_t n = cp::bitsel(c.dhi[k], cp::bitsel(c.dlo[k], n_d2, n_d1),
                                              cp::bitsel(c.dlo[k], n_v, n_h));
                const uint32_t keep = cp::hgt_mask(c.pO[k], n);
                const uint32_t strong = keep & cp::hgt_mask(c.pO[k], high1);
                const uint32_t wk = (1u << (2 * k)) | (2u << (2 * k + 8));       // bit 2k for lane 0, 2k+1 for lane 1
                acc_c = __dp2a_lo(keep, wk, acc_c);                              // += 65535 * bit
                acc_e = __dp2a_lo(strong, wk, acc_e);
            }
            cbyte = (0u - acc_c) & 0xFFu;   // 65535 b = -b (mod 2^16)
            ebyte = (0u - acc_e) & 0xFFu;
        }
        eout[y * 8] = (uint8_t)ebyte;
        cout[y * 8] = (uint8_t)cbyte;
        weak_seen |= cbyte & ~ebyte;
    };

    cp::Sums sa, sb;        // sums of the two most recent rows (roles alternate)
    cp::Mags r0, r1, r2;    // magnitude rows (roles rotate)
    {
        uint32_t w[4];
        load_window(yb - 2, w);
        cp::row_sums(w, sa);
        load_window(yb - 1, w);
        cp::row_sums(w, sb);
        load_window(yb, wn);
        advance(yb - 1, sa, sb, r0, false);   // sa: yb-2 -> yb
        advance(yb, sb, sa, r1, true);        // sb: yb-1 -> yb+1
    }
    // entering row y: sa = row y, sb = row y+1, r0 = row y-1, r1 = row y.  Six rows per trip so that the
    // roles of the two sum sets and the three magnitude rows come back to where they started.
#pragma unroll 1
    for (int y = yb; y < ye; y += 6) {
        advance(y + 1, sa, sb, r2, true);
        emit(y, r0, r1, r2);
        if (y + 1 >= ye) break;
        advance(y + 2, sb, sa, r0, true);
        emit(y + 1, r1, r2, r0);
        if (y + 2 >= ye) break;
        advance(y + 3, sa, sb, r1, true);
        emit(y + 2, r2, r0, r1);
        if (y + 3 >= ye) break;
        advance(y + 4, sb, sa, r2, true);
        emit(y + 3, r0, r1, r2);
        if (y + 4 >= ye) break;
        advance(y + 5, sa, sb, r0, true);
        emit(y + 4, r1, r2, r0);
        if (y + 5 >= ye) break;
        advance(y + 6, sb, sa, r1, true);
        emit(y + 5, r2, r0, r1);
    }
    if (weak_seen) tile_dirty[tile] = 1;
}

// ---- 3. hysteresis on the bit planes ----
// "Weak pixels 8-connected to an edge pixel become edges" = grow E inside C until nothing changes.
// A warp owns a 64 x 32 tile: lane r holds row r as one 64-bit word of C and of E.  One step ORs the
// rows above and below (shifted by -1, 0, +1) into the row, masks with C and then fills every horizontal
// run of C that received a bit - the run fill is two additions ((c + t) ^ c walks a carry up the run; the
// same on the bit-reversed words walks down).  The tile iterates in registers until it is stable, taking
// the one-pixel ring around it from the neighbouring tiles' E words.  Tiles whose ring may have changed are
// revisited in the next round; rounds are separated by a grid-wide barrier of a cooperative launch, so a
// batch costs ONE launch however long the weak chains are (a chain advances at least one tile per round).
constexpr int kHystTileH = 32;  // tiles are 64 columns (two words) x 32 rows

__device__ __forceinline__ unsigned long long run_fill(unsigned long long t, unsigned long long c) {
    // t subset of c: every maximal run of 1-bits of c that contains a bit of t, completely
    const unsigned long long up = (((c + t) ^ c) & c) | t;
    const unsigned long long cr = __brevll(c), tr = __brevll(t);
    const unsigned long long dn = __brevll((((cr + tr) ^ cr) & cr) | tr);
    return up | dn;
}

__global__ void __launch_bounds__(256, 5) psd_hyst_bits_kernel(uint32_t* __restrict__ edge_bits,
                                                            const uint32_t* __restrict__ cand_bits,
                                                            uint8_t* __restrict__ dirty /* [2][n_tiles] */,
                                                            int32_t* __restrict__ flags /* [3] */, int W, int H,
                                                            int Wq, int tiles_x, int tiles_y, int64_t n_tiles) {
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t per_frame_tiles = (int64_t)tiles_x * tiles_y;
    // Tiles are dealt to the warps in runs of 32 (their dirty bytes are read 32 at a time, one per lane, and a
    // warp visits the dirty ones of a run one after the other, so a change walks along the run within the round).
    // Round-robin over the runs: the heavy frames of a batch are spread over all warps.  (A compacted work list
    // per round - perfectly even counts, but neighbouring tiles visited by different warps at the same time -
    // took twice as long.)
    const int64_t t_begin = warp0 * 32, t_end = n_tiles, t_step = n_warps * 32;

    for (int round = 0; round < 100000; ++round) {
        uint8_t* dcur = dirty + (int64_t)(round & 1) * n_tiles;
        uint8_t* dnext = dirty + (int64_t)((round + 1) & 1) * n_tiles;
        if (blockIdx.x == 0 && threadIdx.x == 0) flags[(round + 1) % 3] = 0;
        bool warp_changed = false;
        for (int64_t base = t_begin; base < t_end; base += t_step) {
            uint32_t todo;  // bit l: tile base + l needs a visit this round
            {
                const int64_t mine = base + lane;
                bool need = mine < t_end;
                if (need) {  // round 0: the classify kernel flagged the tiles that hold weak candidates
                    need = dcur[mine] != 0;
                    if (need) dcur[mine] = 0;
                }
                todo = __ballot_sync(0xFFFFFFFFu, need);
            }
            while (todo) {
                const int64_t t = base + __ffs(todo) - 1;
                todo &= todo - 1;
                const int64_t f = t / per_frame_tiles;
                const int tt = (int)(t - f * per_frame_tiles);
                const int ty = tt / tiles_x, tx = tt - ty * tiles_x;
                uint32_t* Et = edge_bits + t * kTileWords;            // tile-major planes: 64 words per tile
                const uint32_t* Ct = cand_bits + t * kTileWords;
                const bool has_left = tx > 0, has_right = tx + 1 < tiles_x;
                // every load of the tile and of its ring is issued before the first use.  Rows beyond the image
                // and the second word of a last odd column hold 0 in both planes.
                const uint2 cw = reinterpret_cast<const uint2*>(Ct)[lane];
                const uint2 ew = reinterpret_cast<const uint2*>(Et)[lane];
                const uint32_t c_lo = cw.x, c_hi = cw.y, e_lo = ew.x, e_hi = ew.y;
                const uint32_t e_l = has_left ? Et[-kTileWords + 2 * lane + 1] : 0u;   // word 1 of the left tile
                const uint32_t e_r = has_right ? Et[kTileWords + 2 * lane] : 0u;       // word 0 of the right tile
                // ring rows above / below the tile: lane 0 / lane 31 fetch them (row 31 of the tile above,
                // row 0 of the tile below)
                const bool ring_in = (lane == 0 && ty > 0) || (lane == 31 && ty + 1 < tiles_y);
                uint32_t g_lo = 0, g_hi = 0, g_l = 0, g_r = 0;
                if (ring_in) {
                    const uint32_t* pe = (lane == 0) ? Et - (int64_t)tiles_x * kTileWords + 62
                                                     : Et + (int64_t)tiles_x * kTileWords;
                    g_lo = pe[0];
                    g_hi = pe[1];
                    if (has_left) g_l = pe[-kTileWords + 1];
                    if (has_right) g_r = pe[kTileWords];
                }
                const unsigned long long c = (unsigned long long)c_lo | ((unsigned long long)c_hi << 32);
                unsigned long long e = (unsigned long long)e_lo | ((unsigned long long)e_hi << 32);
                // weak pixels left in this tile?  (warp-uniform exit: nothing can change)
                if (__ballot_sync(0xFFFFFFFFu, (c & ~e) != 0ull) == 0u) continue;
                const uint32_t lbit = e_l >> 31, rbit = e_r & 1u;  // E left of column 0 / right of column 63, this row
                const unsigned long long e_ring = (unsigned long long)g_lo | ((unsigned long long)g_hi << 32);
                // the side columns do not change while the tile iterates: fold them into two seed bits per row
                uint32_t lu = __shfl_up_sync(0xFFFFFFFFu, lbit, 1), ld = __shfl_down_sync(0xFFFFFFFFu, lbit, 1);
                uint32_t ru = __shfl_up_sync(0xFFFFFFFFu, rbit, 1), rd = __shfl_down_sync(0xFFFFFFFFu, rbit, 1);
                if (lane == 0) { lu = g_l >> 31; ru = g_r & 1u; }
                if (lane == 31) { ld = g_l >> 31; rd = g_r & 1u; }
                unsigned long long side_seed = 0;
                if (lu | lbit | ld) side_seed |= 1ull;
                if (ru | rbit | rd) side_seed |= 1ull << 63;
                const unsigned long long e_in = e;
                while (true) {
                    unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, e, 1), d = __shfl_down_sync(0xFFFFFFFFu, e, 1);
                    if (lane == 0) u = e_ring;
                    if (lane == 31) d = e_ring;
                    const unsigned long long v = u | d;
                    const unsigned long long nb = v | (v << 1) | (v >> 1) | side_seed;
                    const unsigned long long t2 = (nb & c) | e;
                    const unsigned long long e2 = run_fill(t2, c);
                    const bool ch = e2 != e;
                    e = e2;
                    if (__ballot_sync(0xFFFFFFFFu, ch) == 0u) break;
                }
                const bool changed = e != e_in;
                if (changed) reinterpret_cast<uint2*>(Et)[lane] = make_uint2((uint32_t)e, (uint32_t)(e >> 32));
                if (__ballot_sync(0xFFFFFFFFu, changed) != 0u) {
                    warp_changed = true;
                    // the ring of the 8 neighbours may have changed: they look again next round
                    if (lane < 9 && lane != 4) {
                        const int ny = ty + lane / 3 - 1, nx = tx + lane % 3 - 1;
                        if (ny >= 0 && ny < tiles_y && nx >= 0 && nx < tiles_x)
                            dnext[f * per_frame_tiles + (int64_t)ny * tiles_x + nx] = 1;
                    }
                }
            }
        }
        if (warp_changed && lane == 0) atomicOr(&flags[round % 3], 1);
        __threadfence();
        grid.sync();
        if (*(volatile int32_t*)&flags[round % 3] == 0) break;
    }
}

// ---- 4. dilate on the bit-packed edge maps, SAD ----
// The edge plane arrives tile-major (section 2); the dilated plane is row-major [n][H][Wq].
__device__ __forceinline__ uint32_t tiled_word(const uint32_t* __restrict__ plane, int tiles_x, int y, int wq) {
    return plane[((int64_t)(y >> 5) * tiles_x + (wq >> 1)) * kTileWords + ((y & 31) << 1) + (wq & 1)];
}

// the usual kernel sizes (k = 2 R + 1 <= 17): a thread owns one word column of a band of kDilBand rows and
// marches down it with the last 2 R + 1 horizontally dilated rows in registers (the row loop is unrolled
// 2 R + 1 times so the ring slots are register names).  Consecutive lanes own consecutive word columns of the
// same band, so the left / right neighbour words come from the neighbouring LANES (two shuffles) and only the
// first and last lane of a warp load theirs: one load per output word (a tile-major load touches 16 sectors
// per warp, three of them per row cost more than the row-major version of this kernel did).  Every lane runs
// the same kDilBand + 2 R steps; rows and lanes outside the image are predicates, not branches.
constexpr int kDilBand = 64;   // rows per thread: 2 R halo rows on top of them (bands of 32: 0.6 % slower)

template <int R>
__global__ void __launch_bounds__(256) psd_edge_dilate_bits_kernel(const uint32_t* __restrict__ in,
                                                                   uint32_t* __restrict__ out, int H, int Wq,
                                                                   int tiles_x, int64_t tile_words_per_frame,
                                                                   int bands, int64_t n_threads,
                                                                   uint32_t last_word_mask) {
    const int64_t gid0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool active = gid0 < n_threads;
    const int64_t gid = active ? gid0 : n_threads - 1;   // idle lanes shadow the last thread and store nothing
    const int lane = threadIdx.x & 31;
    const int wq = (int)(gid % Wq);
    const int band = (int)((gid / Wq) % bands);
    const int64_t f = gid / ((int64_t)Wq * bands);
    const uint32_t* src = in + f * tile_words_per_frame;
    uint32_t* dst = out + f * (int64_t)H * Wq + wq;
    const uint32_t keep = (wq == Wq - 1) ? last_word_mask : 0xFFFFFFFFu;   // columns >= W stay 0
    const bool has_prv = wq > 0, has_nxt = wq + 1 < Wq;
    const bool load_prv = has_prv && lane == 0, load_nxt = has_nxt && lane == 31;
    auto hdil = [&](int y) -> uint32_t {
        const bool row_in = y >= 0 && y < H;
        const uint32_t cur = row_in ? tiled_word(src, tiles_x, y, wq) : 0u;
        uint32_t prv = __shfl_up_sync(0xFFFFFFFFu, cur, 1), nxt = __shfl_down_sync(0xFFFFFFFFu, cur, 1);
        if (load_prv) prv = row_in ? tiled_word(src, tiles_x, y, wq - 1) : 0u;
        if (load_nxt) nxt = row_in ? tiled_word(src, tiles_x, y, wq + 1) : 0u;
        if (!has_prv) prv = 0u;
        if (!has_nxt) nxt = 0u;
        uint32_t o = cur;
#pragma unroll
        for (int s = 1; s <= R; ++s) o |= __funnelshift_r(cur, nxt, s) | __funnelshift_l(prv, cur, s);
        return o & keep;
    };
    constexpr int K = 2 * R + 1;
    uint32_t ring[K];
    const int y0 = band * kDilBand;
#pragma unroll
    for (int i = 0; i < K - 1; ++i) ring[i] = hdil(y0 - R + i);
#pragma unroll 1
    for (int yo = 0; yo < kDilBand; yo += K) {
#pragma unroll
        for (int j = 0; j < K; ++j) {
            if (yo + j < kDilBand) {
                const int y = y0 + yo + j;
                ring[(K - 1 + j) % K] = hdil(y + R);
                uint32_t o = 0;
#pragma unroll
                for (int i = 0; i < K; ++i) o |= ring[i];
                if (active && y < H) dst[(int64_t)y * Wq] = o;
            }
        }
    }
}

// every larger kernel size (r >= kLargeMinR): the k x k box is separable, a horizontal window-OR of radius r into
// the row-major plane `hdil`, then a vertical one into the dilated plane.  Neither pass does work that grows with k
// beyond log2 k per word.  Radii are clamped to W - 1 / H - 1 first: a window that covers the whole row or column
// from every pixel is saturated, and taps outside the image contribute nothing (cv2.dilate's default border).
// (It replaced a one-thread-per-word kernel for k = 19 .. 63 that ORed (2 r + 1) rows x (2 r + 1) shifts per word:
// on an H100 at 1980 MHz that took 6.3 - 34 us per 1080p frame against 1.0 - 1.2 us for the two passes, and
// 27 - 137 us per 4K frame against 3.8 - 5.1 us; bench_dilate.py.)
constexpr int kLargeMinR = 9;    // k >= 19
constexpr int kHdilRows = 8;     // rows per CTA of the horizontal pass (a warp per row), fewer for very wide rows

// 32 bits of a shared-memory row starting at bit `bit` (>= 0); words at or past `len` read as 0
__device__ __forceinline__ uint32_t row_bits(const uint32_t* row, int len, int bit) {
    const int w = bit >> 5;
    const uint32_t lo = w < len ? row[w] : 0u;
    const uint32_t hi = w + 1 < len ? row[w + 1] : 0u;
    return __funnelshift_r(lo, hi, bit & 31);
}

// Horizontal pass.  A CTA takes `rows` consecutive rows of one frame (they lie in one tile row, and each tile holds
// them as 2 x rows consecutive words, so the load is contiguous per tile) into shared memory, each behind `pad`
// zero words that stand for bit positions -32 pad .. -1.  A warp then doubles windows on its row,
// W_2l(x) = W_l(x) | W_l(x + l) with W_1 = the row, up to the largest power of two L <= k = 2 r + 1, and writes
// out(x) = W_L(x - r) | W_L(x + r - L + 1): two windows of length L that together cover exactly [x - r, x + r]
// (pad = ceil(r / 32) keeps every position read >= -32 pad).  Columns >= W of the last word stay 0.
__global__ void __launch_bounds__(32 * kHdilRows) psd_edge_hdil_rows_kernel(
    const uint32_t* __restrict__ in, uint32_t* __restrict__ hdil, int H, int Wq, int tiles_x,
    int64_t tile_words_per_frame, int rows, int pad, int r, int L, uint32_t last_word_mask) {
    extern __shared__ uint32_t srow[];
    const int len = pad + 2 * tiles_x;   // words of one row buffer
    const int64_t f = blockIdx.y;
    const int y0 = blockIdx.x * rows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t* src = in + f * tile_words_per_frame + (int64_t)(y0 >> 5) * tiles_x * kTileWords + 2 * (y0 & 31);
    const int per_tile = 2 * rows;
    for (int i = threadIdx.x; i < per_tile * tiles_x; i += blockDim.x) {
        const int tx = i / per_tile, j = i - tx * per_tile;   // word j of this tile's slice: row j / 2, word j % 2
        srow[(j >> 1) * 2 * len + pad + 2 * tx + (j & 1)] = src[(int64_t)tx * kTileWords + j];
    }
    for (int i = threadIdx.x; i < rows * pad; i += blockDim.x) srow[(i / pad) * 2 * len + i % pad] = 0u;
    __syncthreads();
    const int y = y0 + warp;
    if (y >= H) return;
    uint32_t* a = srow + warp * 2 * len;
    uint32_t* b = a + len;
    for (int l = 1; l < L; l <<= 1) {
        for (int w = lane; w < len; w += 32) b[w] = a[w] | row_bits(a, len, 32 * w + l);
        __syncwarp();   // b complete; every read of a is done before the next step overwrites it
        uint32_t* t = a; a = b; b = t;
    }
    uint32_t* dst = hdil + (f * H + y) * (int64_t)Wq;
    for (int w = lane; w < Wq; w += 32) {
        const int x = 32 * (pad + w);
        uint32_t o = row_bits(a, len, x - r) | row_bits(a, len, x + r - L + 1);
        if (w == Wq - 1) o &= last_word_mask;
        dst[w] = o;
    }
}

// Vertical pass: van Herk / Gil-Werman.  Pad the column with r zero rows on either side; output row y then ORs the
// padded rows y .. y + k - 1.  Cut the padded column into blocks of k rows: that window is the suffix of block
// b = y / k from row y on and the prefix of block b + 1 up to row y + k - 1.  A thread owns one word column of one
// block of output rows: it marches up block b storing the suffix ORs, then down block b + 1 ORing the running
// prefix in - 3 ORs and 5 accesses per word whatever k is.
__global__ void __launch_bounds__(256) psd_edge_vdil_cols_kernel(const uint32_t* __restrict__ hdil,
                                                                 uint32_t* __restrict__ out, int H, int Wq, int r,
                                                                 int blocks, int64_t n_threads) {
    const int64_t gid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (gid >= n_threads) return;
    const int wq = (int)(gid % Wq);
    const int b = (int)((gid / Wq) % blocks);
    const int64_t f = gid / ((int64_t)Wq * blocks);
    const int k = 2 * r + 1;
    const uint32_t* src = hdil + f * H * (int64_t)Wq + wq;   // padded row q is image row q - r
    uint32_t* dst = out + f * H * (int64_t)Wq + wq;
    const int q0 = b * k, y_end = min(q0 + k, H);
    uint32_t acc = 0;
#pragma unroll 4
    for (int q = min(q0 + k - 1, r + H - 1); q >= q0; --q) {   // padded rows >= r + H are 0
        if (q >= r) acc |= src[(int64_t)(q - r) * Wq];
        if (q < H) dst[(int64_t)q * Wq] = acc;
    }
    acc = 0;
#pragma unroll 4
    for (int y = q0; y < y_end; ++y) {   // padded row y + k of block b + 1 (> r always)
        if (y > q0) dst[(int64_t)y * Wq] |= acc;
        if (y + k < r + H) acc |= src[(int64_t)(y + k - r) * Wq];
    }
}

static int hdil_smem_bytes(int rows, int pad, int tiles_x) { return rows * 2 * (pad + 2 * tiles_x) * 4; }

static int max_smem_optin() {
    static int optin = 0;
    if (optin == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
            optin = 48 * 1024;
    }
    return optin;
}

// rows per CTA of the horizontal pass for a frame width and kernel size, 0 if one row does not fit
static int hdil_rows(int W, int ksize) {
    const int Wq = (W + 31) / 32, tiles_x = (Wq + 1) / 2;
    const int r = min(ksize / 2, W - 1), pad = (r + 31) / 32;
    int rows = kHdilRows;
    while (rows > 0 && hdil_smem_bytes(rows, pad, tiles_x) > max_smem_optin()) rows >>= 1;
    return rows;
}

// this kernel size dilates in two passes through EdgeBuffers::bits_hdil
static bool edge_dilate_separable(int ksize) { return ksize / 2 >= kLargeMinR; }

// words per frame of a tile-major bit plane
static int64_t edge_tile_words(int W, int H) {
    const int Wq = (W + 31) / 32;
    return (int64_t)((Wq + 1) / 2) * ((H + kHystTileH - 1) / kHystTileH) * kTileWords;
}

int edge_dilate_check(int W, int ksize) {
    if (!edge_dilate_separable(ksize)) return PSD_OK;
    PSD_REQUIRE(hdil_rows(W, ksize) > 0, "frame width %d is too wide for the kernel size %d dilation (one row and "
                "its padding must fit in %d bytes of shared memory)", W, ksize, max_smem_optin());
    return PSD_OK;
}

static int launch_dilate_separable(const uint32_t* in, uint32_t* hdil, uint32_t* out, int n, int W, int H, int ksize,
                                   uint32_t mask, cudaStream_t stream) {
    const int Wq = (W + 31) / 32, tiles_x = (Wq + 1) / 2;
    const int rh = min(ksize / 2, W - 1), rv = min(ksize / 2, H - 1);
    const int pad = (rh + 31) / 32;
    int L = 1;
    while (2 * L <= 2 * rh + 1) L *= 2;
    const int rows = hdil_rows(W, ksize);
    PSD_REQUIRE(rows > 0, "frame width %d is too wide for the kernel size %d dilation", W, ksize);
    const int smem = hdil_smem_bytes(rows, pad, tiles_x);
    if (smem > 48 * 1024) {
        static int raised = 0;   // the attribute is a ceiling, not a reservation: raise it once to the device limit
        if (!raised) {
            PSD_CUDA(cudaFuncSetAttribute(psd_edge_hdil_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          max_smem_optin()));
            raised = 1;
        }
    }
    // rows per CTA divide 32, so a CTA never straddles two tile rows; rows past H load the planes' zero padding
    dim3 hg((unsigned)((H + rows - 1) / rows), (unsigned)n);
    psd_edge_hdil_rows_kernel<<<hg, 32 * rows, smem, stream>>>(in, hdil, H, Wq, tiles_x, edge_tile_words(W, H), rows,
                                                             pad, rh, L, mask);
    PSD_CHECK_LAUNCH();
    const int k = 2 * rv + 1, blocks = (H + k - 1) / k;
    const int64_t n_threads = (int64_t)Wq * blocks * n;
    psd_edge_vdil_cols_kernel<<<(unsigned)((n_threads + 255) / 256), 256, 0, stream>>>(hdil, out, H, Wq, rv, blocks,
                                                                                      n_threads);
    return PSD_OK;
}

template <int R>
static void launch_dilate(const uint32_t* in, uint32_t* out, int n, int H, int Wq, uint32_t mask, cudaStream_t stream) {
    const int bands = (H + kDilBand - 1) / kDilBand;
    const int tiles_x = (Wq + 1) / 2;
    const int64_t tile_words = (int64_t)tiles_x * ((H + kHystTileH - 1) / kHystTileH) * kTileWords;
    const int64_t n_threads = (int64_t)Wq * bands * n;
    psd_edge_dilate_bits_kernel<R><<<(unsigned)((n_threads + 255) / 256), 256, 0, stream>>>(
        in, out, H, Wq, tiles_x, tile_words, bands, n_threads, mask);
}

// frame f's SAD is added to sad[f * sad_stride] (psd_frame_sums::sad_edges of slot 0, or an edge slot's own array)
__global__ void __launch_bounds__(256) psd_edge_sad_bits_kernel(const uint32_t* __restrict__ dil,
                                                                const uint32_t* __restrict__ carry,
                                                                int64_t per_frame, int have_prev,
                                                                uint64_t* __restrict__ sad, int64_t sad_stride) {
    const int64_t f = blockIdx.y;
    if (f == 0 && !have_prev) return;
    const uint32_t* cur = dil + f * per_frame;
    const uint32_t* prv = (f == 0) ? carry : dil + (f - 1) * per_frame;
    uint32_t cnt = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < per_frame;
         i += (int64_t)gridDim.x * blockDim.x)
        cnt += __popc(cur[i] ^ prv[i]);
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    __shared__ uint32_t part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; ++w) t += part[w];
        if (t) atomicAdd(reinterpret_cast<unsigned long long*>(sad + f * sad_stride), 255ull * t);
    }
}

// debug/test tap: bit-packed map (row-major, or tile-major if tiles_x > 0) -> 0/255 bytes
__global__ void psd_edge_unpack_kernel(const uint32_t* __restrict__ bits, uint8_t* __restrict__ out, int W,
                                       int H, int Wq, int tiles_x) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)W * H) return;
    const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
    const uint32_t w = tiles_x > 0 ? tiled_word(bits, tiles_x, y, x >> 5) : bits[(int64_t)y * Wq + (x >> 5)];
    out[i] = ((w >> (x & 31)) & 1u) ? 255 : 0;
}

int edge_unpack(const EdgeBuffers& b, int64_t index, bool canny_map, int W, int H, cudaStream_t stream) {
    const int Wq = (W + 31) / 32;
    const uint32_t* bits = canny_map ? b.bits_in + index * edge_tile_words(W, H) : b.bits_dil + index * H * (int64_t)Wq;
    psd_edge_unpack_kernel<<<(unsigned)(((int64_t)W * H + 255) / 256), 256, 0, stream>>>(bits, b.tmp, W, H, Wq,
                                                                                         canny_map ? (Wq + 1) / 2 : 0);
    PSD_CHECK_LAUNCH();
    return PSD_OK;
}

int edge_buffers_create(EdgeBuffers* b, int W, int H, int max_batch, int ksize) {
    const size_t P = (size_t)W * H, words = (size_t)H * ((W + 31) / 32);
    PSD_CUDA(cudaMalloc(&b->vplane, P * max_batch));
    // the two planes of the hysteresis are tile-major and padded to whole 64 x 32 tiles; the padding is never
    // written, so it is zeroed once here
    const size_t tiled = (size_t)edge_tile_words(W, H) * 4 * max_batch;
    PSD_CUDA(cudaMalloc(&b->cand, tiled)); PSD_CUDA(cudaMalloc(&b->bits_in, tiled));
    PSD_CUDA(cudaMemset(b->cand, 0, tiled)); PSD_CUDA(cudaMemset(b->bits_in, 0, tiled));
    PSD_CUDA(cudaMalloc(&b->tmp, P));
    PSD_CUDA(cudaMalloc(&b->bits_dil, words * 4 * max_batch));
    PSD_CUDA(cudaMalloc(&b->vhist, (size_t)max_batch * 256 * 4));
    PSD_CUDA(cudaMalloc(&b->thresholds, (size_t)max_batch * 2 * 4));
    PSD_CUDA(cudaMalloc(&b->hyst_flags, 64));
    const size_t n_tiles = (size_t)max_batch * ((W + 63) / 64) * ((H + 31) / 32);
    PSD_CUDA(cudaMalloc(&b->dirty, 2 * n_tiles));
    return edge_buffers_add_ksize(b, W, H, max_batch, ksize);
}

int edge_buffers_add_ksize(EdgeBuffers* b, int W, int H, int max_batch, int ksize) {
    if (edge_dilate_separable(ksize) && !b->bits_hdil)
        PSD_CUDA(cudaMalloc(&b->bits_hdil, (size_t)H * ((W + 31) / 32) * 4 * max_batch));
    return PSD_OK;
}

void edge_buffers_destroy(EdgeBuffers* b) {
    cudaFree(b->vplane); cudaFree(b->vhist); cudaFree(b->thresholds); cudaFree(b->cand); cudaFree(b->bits_in);
    cudaFree(b->bits_dil); cudaFree(b->bits_hdil); cudaFree(b->tmp); cudaFree(b->dirty); cudaFree(b->hyst_flags);
    *b = EdgeBuffers{};
}

int launch_edges(const EdgeBuffers& b, int n, int W, int H, const EdgeSlot* slots, int n_slots, int64_t first,
                 bool have_prev, cudaStream_t stream) {
    PSD_REQUIRE(n > 0 && n <= 65535, "edge batch out of range");
    const int64_t P = (int64_t)W * H;
    const int Wq = (W + 31) / 32;
    const int64_t per_frame = (int64_t)H * Wq;
    psd_edge_thresholds_kernel<<<(n + 7) / 8, 256, 0, stream>>>(b.vhist, n, P, b.thresholds);
    PSD_CHECK_LAUNCH();
    // classify: one thread per 8 columns x kBandRows rows
    {
        const int strips = (W + 7) / 8, bands = (H + kBandRows - 1) / kBandRows;
        const int64_t n_threads = (int64_t)strips * bands * n;
        const unsigned cblock = kClassifyBlock;
        const unsigned blocks = (unsigned)((n_threads + cblock - 1) / cblock);
        // (bytes of the planes that no strip writes - beyond the last strip, below the last row - were zeroed
        // when the planes were allocated and nothing ever sets them)
        const int64_t n_tiles0 = (int64_t)((Wq + 1) / 2) * bands * n;  // bands == hysteresis tile rows
        PSD_CUDA(cudaMemsetAsync(b.dirty, 0, (size_t)2 * n_tiles0, stream));
        if ((W & 7) == 0)
            psd_canny_classify_pairs_kernel<true><<<blocks, cblock, 0, stream>>>(b.vplane, b.thresholds, b.bits_in, b.cand,
                                                                              b.dirty, W, H, Wq, strips, bands, n_threads);
        else
            psd_canny_classify_pairs_kernel<false><<<blocks, cblock, 0, stream>>>(b.vplane, b.thresholds, b.bits_in, b.cand,
                                                                               b.dirty, W, H, Wq, strips, bands, n_threads);
        PSD_CHECK_LAUNCH();
    }
    // hysteresis: one cooperative launch (grid = what is co-resident on the device)
    {
        int tiles_x = (Wq + 1) / 2, tiles_y = (H + kHystTileH - 1) / kHystTileH;
        int64_t n_tiles = (int64_t)tiles_x * tiles_y * n;
        PSD_CUDA(cudaMemsetAsync(b.hyst_flags, 0, 3 * sizeof(int32_t), stream));
        static int grid_cap = 0;
        if (grid_cap == 0) {
            int dev = 0, sms = 0, per_sm = 0;
            PSD_CUDA(cudaGetDevice(&dev));
            PSD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            PSD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, psd_hyst_bits_kernel, 256, 0));
            PSD_REQUIRE(per_sm > 0, "psd_hyst_bits_kernel does not fit on an SM");
            grid_cap = sms * per_sm;
        }
        const int64_t want = (n_tiles + 7) / 8;  // 8 warps per CTA, at least one tile per warp
        const int grid = (int)(want < grid_cap ? (want > 0 ? want : 1) : grid_cap);
        uint32_t* e_ptr = b.bits_in;
        const uint32_t* c_ptr = b.cand;
        uint8_t* d_ptr = b.dirty;
        int32_t* f_ptr = b.hyst_flags;
        int w_ = W, h_ = H, wq_ = Wq;
        void* args[] = {&e_ptr, &c_ptr, &d_ptr, &f_ptr, &w_, &h_, &wq_, &tiles_x, &tiles_y, &n_tiles};
        PSD_CUDA(cudaLaunchCooperativeKernel((const void*)psd_hyst_bits_kernel, dim3(grid), dim3(256), args, 0, stream));
    }
    count_launch(3);
    // one dilation + SAD per kernel size, in stream order through the one bits_dil plane
    const uint32_t last_mask = (W & 31) ? ((1u << (W & 31)) - 1u) : 0xFFFFFFFFu;
    for (int s = 0; s < n_slots; ++s) {
        const int ksize = slots[s].ksize, r = ksize / 2;
        if (edge_dilate_separable(ksize)) {   // k >= 19
            const int rc = launch_dilate_separable(b.bits_in, b.bits_hdil, b.bits_dil, n, W, H, ksize, last_mask, stream);
            if (rc) return rc;
            count_launch(1);   // the second pass
        } else switch (r) {
            case 1: launch_dilate<1>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 2: launch_dilate<2>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 3: launch_dilate<3>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 4: launch_dilate<4>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 5: launch_dilate<5>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 6: launch_dilate<6>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 7: launch_dilate<7>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            case 8: launch_dilate<8>(b.bits_in, b.bits_dil, n, H, Wq, last_mask, stream); break;
            default: PSD_REQUIRE(false, "edge kernel size %d has no dilation kernel", ksize);
        }
        PSD_CHECK_LAUNCH();
        dim3 sg((unsigned)min((int64_t)64, (per_frame + 255) / 256), (unsigned)n);
        const FrameRows& sads = slots[s].sads;
        psd_edge_sad_bits_kernel<<<sg, 256, 0, stream>>>(b.bits_dil, slots[s].carry_bits, per_frame, have_prev ? 1 : 0,
                                                         sads.at<uint64_t>(first), sads.row_bytes / 8);
        PSD_CHECK_LAUNCH();
        count_launch(2);
        PSD_CUDA(cudaMemcpyAsync(slots[s].carry_bits, b.bits_dil + (int64_t)(n - 1) * per_frame,
                                 (size_t)per_frame * 4, cudaMemcpyDeviceToDevice, stream));
    }
    return PSD_OK;
}

}  // namespace psd
