// HashDetector's perceptual hash (hash_detector.py:124-158) for every frame of a batch:
//   gray = cv2.cvtColor(BGR2GRAY)                      15-bit fixed point, exact
//   r    = cv2.resize(gray, (n, n), INTER_AREA)        n = size * lowpass; exact restatement of OpenCV's two paths
//   x    = float32(r) / max(r)                         float32 division
//   D    = cv2.dct(x)[:size, :size]                    float64 here (cv2: float32 through IPP) - the one stage
//                                                      with a tolerance: a bit can differ only where a coefficient
//                                                      lies within rounding distance of the median
//   hash = D > numpy.median(D)                         float32 compare; median of an even count = float32 mean
// INTER_AREA (imgproc/resize.cpp): integer scale factors in both directions -> integer block sums times
// float32(1/area), rounded (2x2: (sum + 2) >> 2); otherwise per destination cell a float32 accumulation
// `buf += S * alpha` along each source row (separate multiply and add, source order) and `sum += beta * buf`
// down the rows.  oracle/intmath.py:resize_area is the CPU twin, pinned against cv2.
#include <math.h>

#include <vector>

#include "psd_common.cuh"

namespace psd {

__device__ __forceinline__ uint32_t gray_bgr(uint32_t b, uint32_t g, uint32_t r) {
    return (b * 3735u + g * 19235u + r * 9798u + 16384u) >> 15;
}
// the same from a register holding (B, G, R, x) bytes: two IDP4A on the weights' high and low bytes
// (3735 = 14 * 256 + 151, 19235 = 75 * 256 + 35, 9798 = 38 * 256 + 70; 64 * 256 = the rounding constant)
__device__ __forceinline__ uint32_t gray_word(uint32_t px) {
    const uint32_t hi = __dp4a(px, 0x00264B0Eu, 64u);
    return (__dp4a(px, 0x00462397u, hi << 8)) >> 15;
}
// byte -> float32 without the conversion unit: 0x4B000000 | g is 2^23 + g
__device__ __forceinline__ float byte_to_float(uint32_t g) { return __fadd_rn(__uint_as_float(0x4B000000u | g), -8388608.0f); }

// The horizontal pass.  A CTA takes a block of consecutive source rows of one frame (max(1, 256 / n) of them, fewer
// if their gray bytes would not fit kHashRowsSmemBytes):
//   1. all threads pull the block - it is contiguous in memory - 16 pixels (three 16-byte loads) at a time,
//      convert to gray and park the gray bytes in shared memory (row pitch W rounded up + 4: two rows of a
//      1920-wide frame would otherwise sit in the same banks);
//   2. thread (row, destination column) walks its taps in shared memory: the integer block sum if both scale
//      factors are integers, else OpenCV's float32 `buf += S * alpha` in source order (separate multiply and
//      add: the order and the roundings decide the last bit, so this chain stays sequential).  For one geometry
//      with n <= 256 every thread has at most one (row, column); for n > 256 the CTA owns one row and loops over
//      columns.  With several geometries the block height follows the smallest n and threads loop as needed.
// (The first version had one thread per (row, column) read its 3 x 120 bytes straight from global memory, 32
// lanes 360 bytes apart: 0.085 of the HBM roofline.)
// One launch serves up to kHashRowsMaxGeo hash geometries (an engine's hash slots): step 1 runs once, step 2 once
// per geometry, each with its own taps and row buffer.  A geometry's row buffer does not depend on the block of rows
// a CTA takes or on the other geometries, so it is bit-identical to what a one-geometry launch writes.
constexpr int kHashRowsMaxGeo = 8;
struct HashRowsGeo {
    const int32_t* xstart;
    const int32_t* xsi;
    const float* xalpha;
    const int32_t* xmid;
    float* rowbuf;   // [frames][H][n]
    int n, fast;
};
struct HashRowsArgs {
    HashRowsGeo g[kHashRowsMaxGeo];
    int count;
};

__global__ void __launch_bounds__(256) psd_hash_rows_kernel(const uint8_t* __restrict__ frames, int64_t frame_stride,
                                                            int W, int H, int rows_per_cta, int pitch,
                                                            const __grid_constant__ HashRowsArgs geo) {
    extern __shared__ __align__(16) uint8_t sgray[];   // [rows_per_cta][pitch]
    const int tid = threadIdx.x;
    const int64_t f = blockIdx.y;
    const int sy0 = blockIdx.x * rows_per_cta;
    const int rows = min(rows_per_cta, H - sy0);
    const uint8_t* blk = frames + f * frame_stride + (int64_t)sy0 * W * 3;
    const int n_px = rows * W;
    // ---- 1. gray bytes of the block ----
    if ((W & 15) == 0 && ((reinterpret_cast<uintptr_t>(blk) & 15) == 0)) {
        for (int q = tid * 16; q < n_px; q += 256 * 16) {   // a group of 16 pixels never straddles a row
            const uint4* p = reinterpret_cast<const uint4*>(blk + (int64_t)q * 3);
            const uint4 a = p[0], b = p[1], c = p[2];
            const uint32_t w[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
            const int r = q / W, x = q - r * W;
            uint32_t* dst = reinterpret_cast<uint32_t*>(sgray + r * pitch + x);
#pragma unroll
            for (int g4 = 0; g4 < 4; ++g4) {   // 4 pixels = 12 bytes = words 3 g4 .. 3 g4 + 2
                const uint32_t w0 = w[3 * g4], w1 = w[3 * g4 + 1], w2 = w[3 * g4 + 2];
                const uint32_t g0 = gray_word(w0);                              // bytes 0 1 2 (3 ignored: weight 0)
                const uint32_t g1 = gray_word(__byte_perm(w0, w1, 0x0543));     // bytes 3 4 5
                const uint32_t g2 = gray_word(__byte_perm(w1, w2, 0x0432));     // bytes 6 7 8
                const uint32_t g3 = gray_word(w2 >> 8);                         // bytes 9 10 11
                dst[g4] = g0 | (g1 << 8) | (g2 << 16) | (g3 << 24);
            }
        }
    } else {
        for (int q = tid; q < n_px; q += 256) {
            const int r = q / W, x = q - r * W;
            const uint8_t* p = blk + (int64_t)q * 3;
            sgray[r * pitch + x] = (uint8_t)gray_bgr(p[0], p[1], p[2]);
        }
    }
    __syncthreads();
    // ---- 2. (row, destination column) pairs of every geometry ----
    for (int gi = 0; gi < geo.count; ++gi) {
        const HashRowsGeo& g = geo.g[gi];
        const int n = g.n;
        const int32_t* __restrict__ xstart = g.xstart;
        const int32_t* __restrict__ xsi = g.xsi;
        const float* __restrict__ xalpha = g.xalpha;
        const int32_t* __restrict__ xmid = g.xmid;
        for (int c = tid; c < rows * n; c += 256) {
            const int r = c / n, dx = c - r * n;
            const uint8_t* srow = sgray + r * pitch;
            float* out = g.rowbuf + (f * H + sy0 + r) * (int64_t)n + dx;
            if (g.fast) {  // integer scale: exact integer sum of the block's columns
                const int sxw = W / n;
                uint32_t s = 0;
                for (int x = dx * sxw; x < (dx + 1) * sxw; ++x) s += srow[x];
                *out = __uint_as_float(s);
            } else {
                // first (partial) tap, the run of whole pixels, last (partial) tap - in source order
                float buf = 0.0f;
                const int k0 = __ldg(xstart + dx), k1 = __ldg(xstart + dx + 1);
                const int km = __ldg(xmid + 2 * dx), nm = __ldg(xmid + 2 * dx + 1);
                for (int k = k0; k < km; ++k)
                    buf = __fadd_rn(buf, __fmul_rn(byte_to_float(srow[__ldg(xsi + k)]), __ldg(xalpha + k)));
                if (nm > 0) {
                    const uint8_t* sp = srow + __ldg(xsi + km);
                    const float am = __ldg(xalpha + km);
#pragma unroll 8
                    for (int i = 0; i < nm; ++i) buf = __fadd_rn(buf, __fmul_rn(byte_to_float(sp[i]), am));
                }
                for (int k = km + nm; k < k1; ++k)
                    buf = __fadd_rn(buf, __fmul_rn(byte_to_float(srow[__ldg(xsi + k)]), __ldg(xalpha + k)));
                *out = buf;
            }
        }
    }
}

// 1-D DCT-II (unnormalised) coefficient u of a vector, computed the way fast DCTs do: the vector is folded
// (s[i] = a[i] + a[len-1-i]) as long as its length is even; an even frequency is the half frequency of the folded
// vector, an odd frequency is a sum over DIFFERENCES a[i] - a[len-1-i].  Constant and mirror-symmetric inputs
// therefore give exact zeros where the exact transform is zero (a plain sum of products leaves rounding noise of
// random sign, and the hash is `coefficient > median`).  `lev` holds the folded levels back to back
// (level k at lev + off[k], length len[k]; level 0 is the vector itself).  oracle/intmath.py:dct_fold_1d is the twin.
struct FoldPlan {
    int levels;        // number of levels including level 0
    int len[8], off[8];
};

__device__ __forceinline__ double fold_coef(const double* v0, int stride0, const double* lev, int lstride,
                                            const FoldPlan& fp, int n, int u, const double* costab) {
    int k = 0;
    if (u == 0) k = fp.levels - 1;
    else while (k + 1 < fp.levels && (u & ((2 << k) - 1)) == 0) ++k;
    const double* a = (k == 0) ? v0 : lev + (int64_t)fp.off[k] * lstride;
    const int st = (k == 0) ? stride0 : lstride;
    const int nk = fp.len[k];
    double acc = 0.0;
    if ((nk & 1) == 0 && ((u >> k) & 1)) {
        for (int i = 0; i < nk / 2; ++i) {
            const double d = __dsub_rn(a[(int64_t)i * st], a[(int64_t)(nk - 1 - i) * st]);
            acc = __dadd_rn(acc, __dmul_rn(d, costab[((2 * i + 1) * u) % (4 * n)]));
        }
    } else {
        for (int i = 0; i < nk; ++i)
            acc = __dadd_rn(acc, __dmul_rn(a[(int64_t)i * st], costab[((2 * i + 1) * u) % (4 * n)]));
    }
    return acc;
}

// Order-preserving keys of float32: key(a) < key(b) exactly when a < b (-0.0 sorts just below +0.0, which
// compare equal, so the selected value compares like numpy's).
__device__ __forceinline__ uint32_t float_key(float a) {
    const uint32_t b = __float_as_uint(a);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// The k-th smallest (0-based) of v[0..m) by a CTA of 256 threads: a radix select over the keys, 8 bits a pass from
// the top.  Each pass histograms the digit of the keys that share the prefix found so far; warp 0 scans the 256
// counts (8 per lane) and picks the bin that holds rank k.  hist[256] and sel[2] are shared scratch.
__device__ float cta_select(const float* v, int m, int k, uint32_t* hist, uint32_t* sel) {
    const int tid = threadIdx.x;
    uint32_t prefix = 0, mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        hist[tid] = 0;
        __syncthreads();
        for (int c = tid; c < m; c += 256) {
            const uint32_t key = float_key(v[c]);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {
            uint32_t s = 0;
#pragma unroll
            for (int b = 0; b < 8; ++b) s += hist[tid * 8 + b];
            uint32_t incl = s;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
                if (tid >= d) incl += y;
            }
            uint32_t below = incl - s;
            if (below <= (uint32_t)k && (uint32_t)k < incl) {
                int b = tid * 8;
                while (below + hist[b] <= (uint32_t)k) below += hist[b++];
                sel[0] = (uint32_t)b;
                sel[1] = below;
            }
        }
        __syncthreads();
        prefix |= sel[0] << shift;
        mask |= 255u << shift;
        k -= (int)sel[1];
        __syncthreads();
    }
    return key_float(prefix);
}

// One CTA per frame: vertical pass, normalisation, DCT low band, median, bits.  The working set (image, folded
// levels, low band) sits in dynamic shared memory, or for large hash images (kGlobal) in the frame's slice of a
// global workspace - the same code on the same values either way.
template <bool kGlobal>
__global__ void __launch_bounds__(256, 2) psd_hash_finish_kernel(const float* __restrict__ rowbuf, int H, int n, int size,
                                                              int fast, int area_w, int area_h,
                                                              const int32_t* __restrict__ ystart,
                                                              const int32_t* __restrict__ ysi,
                                                              const float* __restrict__ ybeta,
                                                              const double* __restrict__ costab /* [4n] cos(pi k / 2n) */,
                                                              FoldPlan fp, double* __restrict__ ws, int64_t ws_doubles,
                                                              int words,
                                                              uint64_t* __restrict__ hashes /* [frames][words] */) {
    extern __shared__ __align__(16) double dsm[];
    const int64_t f = blockIdx.x;
    double* x = kGlobal ? ws + f * ws_doubles : dsm;   // [n][n] normalised image (row i, column j)
    double* lev = x + n * n;            // [n][n]: folded levels of every column j (element e of column j at lev[e*n + j])
    double* t = lev + n * n;            // [size][n]: vertical transform, t[u][j]
    double* lev2 = t + size * n;        // [n][size]: folded levels of every t[u][.] (element e of row u at lev2[e*size + u])
    float* low = reinterpret_cast<float*>(lev2 + (int64_t)n * size);   // [size][size] low band
    __shared__ uint32_t mx;
    __shared__ uint32_t hist[256], sel[2];
    const int tid = threadIdx.x;
    const float* rb = rowbuf + f * (int64_t)H * n;
    if (tid == 0) mx = 0;
    __syncthreads();
    uint32_t my_max = 0;
    for (int c = tid; c < n * n; c += 256) {
        const int dy = c / n, dx = c - dy * n;
        uint32_t v;
        if (fast) {
            uint32_t s = 0;
            for (int sy = dy * area_h; sy < (dy + 1) * area_h; ++sy) s += __float_as_uint(rb[(int64_t)sy * n + dx]);
            if (area_w == 2 && area_h == 2) v = (s + 2u) >> 2;
            else if (area_w == 1 && area_h == 1) v = s;
            else v = (uint32_t)min(max(__float2int_rn(__fmul_rn((float)s, __fdiv_rn(1.0f, (float)(area_w * area_h)))), 0), 255);
        } else {
            float sum = 0.0f;
            for (int k = ystart[dy]; k < ystart[dy + 1]; ++k) {
                const float term = __fmul_rn(ybeta[k], rb[(int64_t)ysi[k] * n + dx]);
                sum = (k == ystart[dy]) ? term : __fadd_rn(sum, term);
            }
            v = (uint32_t)min(max(__float2int_rn(sum), 0), 255);
        }
        x[c] = (double)v;
        my_max = max(my_max, v);
    }
    atomicMax(&mx, my_max);
    __syncthreads();
    const float denom = (float)(mx ? mx : 1u);
    for (int c = tid; c < n * n; c += 256) x[c] = (double)__fdiv_rn((float)x[c], denom);
    __syncthreads();
    // folded levels of every column (level k from level k-1)
    for (int k = 1; k < fp.levels; ++k) {
        const int len = fp.len[k], plen = fp.len[k - 1];
        for (int c = tid; c < len * n; c += 256) {
            const int e = c / n, j = c - e * n;
            const double* prev = (k == 1) ? x : lev + (int64_t)fp.off[k - 1] * n;
            lev[(int64_t)(fp.off[k] + e) * n + j] = __dadd_rn(prev[(int64_t)e * n + j], prev[(int64_t)(plen - 1 - e) * n + j]);
        }
        __syncthreads();
    }
    // vertical transform: t[u][j] = sum_i x[i][j] cos(pi (2i+1) u / 2n), u < size
    for (int c = tid; c < size * n; c += 256) {
        const int u = c / n, j = c - u * n;
        t[c] = fold_coef(x + j, n, lev + j, n, fp, n, u, costab);
    }
    __syncthreads();
    for (int k = 1; k < fp.levels; ++k) {
        const int len = fp.len[k], plen = fp.len[k - 1];
        for (int c = tid; c < len * size; c += 256) {
            const int e = c / size, u = c - e * size;
            double pa, pb;
            if (k == 1) { pa = t[u * n + e]; pb = t[u * n + plen - 1 - e]; }
            else { pa = lev2[(int64_t)(fp.off[k - 1] + e) * size + u]; pb = lev2[(int64_t)(fp.off[k - 1] + plen - 1 - e) * size + u]; }
            lev2[(int64_t)(fp.off[k] + e) * size + u] = __dadd_rn(pa, pb);
        }
        __syncthreads();
    }
    // horizontal transform + orthonormal scale: D[u][v] = s(u) s(v) sum_j t[u][j] cos(pi (2j+1) v / 2n)
    const int m = size * size;
    const double s0 = sqrt(1.0 / n), s1 = sqrt(2.0 / n);
    for (int c = tid; c < m; c += 256) {
        const int u = c / size, v = c - u * size;
        const double acc = fold_coef(t + u * n, 1, lev2 + u, size, fp, n, v, costab);
        low[c] = (float)__dmul_rn(__dmul_rn(acc, u ? s1 : s0), v ? s1 : s0);
    }
    __syncthreads();
    // numpy.median: the middle value, or the float32 mean of the two middle values
    float med = cta_select(low, m, m / 2, hist, sel);
    if ((m & 1) == 0) med = __fmul_rn(__fadd_rn(cta_select(low, m, m / 2 - 1, hist, sel), med), 0.5f);
    // bit c = low[c] > med; word w holds bits 64 w .. 64 w + 63 (words past the low band stay 0)
    const int warp = tid >> 5, lane = tid & 31;
    for (int w = warp; w < words; w += 8) {
        const int c0 = w * 64 + lane, c1 = c0 + 32;
        const uint32_t lo = __ballot_sync(0xFFFFFFFFu, c0 < m && low[c0] > med);
        const uint32_t hi = __ballot_sync(0xFFFFFFFFu, c1 < m && low[c1] > med);
        if (lane == 0) hashes[f * words + w] = ((uint64_t)hi << 32) | lo;
    }
}

// hash_detector.py:95-99: Hamming distance to the previous frame's hash, divided by size * size.  One warp per
// frame; hashes are `words` apart.
__global__ void psd_scan_hash_dist_kernel(const uint64_t* __restrict__ hashes, int64_t n, int words, double size_sq,
                                          const uint64_t* __restrict__ prev_hash, double* __restrict__ out) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint64_t* cur = hashes + i * words;
    const uint64_t* prv = (i > 0) ? cur - words : prev_hash;
    if (prv == nullptr) { if (lane == 0) out[i] = __longlong_as_double(0x7FF8000000000000LL); return; }
    int cnt = 0;
    for (int w = lane; w < words; w += 32) cnt += __popcll(cur[w] ^ prv[w]);
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    if (lane == 0) out[i] = __ddiv_rn((double)cnt, size_sq);
}

// ---- host side: OpenCV's computeResizeAreaTab, the cosine table ----
static void area_tab(int ssize, int dsize, std::vector<int32_t>& start, std::vector<int32_t>& si, std::vector<float>& alpha) {
    const double scale = (double)ssize / dsize;
    start.assign(dsize + 1, 0);
    si.clear(); alpha.clear();
    for (int dx = 0; dx < dsize; ++dx) {
        start[dx] = (int32_t)si.size();
        const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        const double cell = std::min(scale, ssize - fsx1);
        int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
        sx2 = std::min(sx2, ssize - 1);
        sx1 = std::min(sx1, sx2);
        if (sx1 - fsx1 > 1e-3) { si.push_back(sx1 - 1); alpha.push_back((float)((sx1 - fsx1) / cell)); }
        for (int sx = sx1; sx < sx2; ++sx) { si.push_back(sx); alpha.push_back((float)(1.0 / cell)); }
        if (fsx2 - sx2 > 1e-3) { si.push_back(sx2); alpha.push_back((float)(std::min(std::min(fsx2 - sx2, 1.0), cell) / cell)); }
    }
    start[dsize] = (int32_t)si.size();
}

template <typename T>
static int upload(const std::vector<T>& v, T** out) {
    PSD_CUDA(cudaMalloc(out, std::max<size_t>(1, v.size()) * sizeof(T)));
    if (!v.empty()) PSD_CUDA(cudaMemcpy(*out, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return PSD_OK;
}

constexpr int kHashStaticSmem = 2048;                       // the finish kernel's static shared memory, rounded up
constexpr int64_t kHashWorkspaceBytes = (int64_t)512 << 20;  // row buffer + finish workspace of one sub-batch
constexpr int kHashRowsSmemBytes = 200 * 1024;              // the rows kernel's gray block (rows_per_cta * pitch)

int hash_plan_create(HashPlan* p, int W, int H, int size, int lowpass, int max_batch, bool force_global_ws) {
    PSD_REQUIRE(size >= 1 && lowpass >= 1, "HashDetector needs size >= 1 and lowpass >= 1");
    const int64_t n64 = (int64_t)size * lowpass;
    PSD_REQUIRE(W >= n64 && H >= n64, "frames smaller than the %lldx%lld hash image are not supported",
                (long long)n64, (long long)n64);
    const int n = (int)n64;
    p->n = n; p->size = size;
    p->words = PSD_HASH_WORDS_FOR(size);
    p->fast = (W % n == 0 && H % n == 0) ? 1 : 0;
    p->area_w = W / n; p->area_h = H / n;
    std::vector<int32_t> st, si; std::vector<float> al;
    area_tab(W, n, st, si, al);
    int rc = upload(st, &p->xstart); if (rc) return rc;
    rc = upload(si, &p->xsi); if (rc) return rc;
    rc = upload(al, &p->xalpha); if (rc) return rc;
    {   // the whole-pixel taps of a column are consecutive source pixels with one common weight
        std::vector<int32_t> mid((size_t)2 * n);
        const double scale = (double)W / n;
        for (int dx = 0; dx < n; ++dx) {
            const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
            int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
            sx2 = std::min(sx2, W - 1);
            sx1 = std::min(sx1, sx2);
            mid[2 * dx] = st[dx] + ((sx1 - fsx1 > 1e-3) ? 1 : 0);
            mid[2 * dx + 1] = std::max(0, sx2 - sx1);
        }
        rc = upload(mid, &p->xmid); if (rc) return rc;
    }
    area_tab(H, n, st, si, al);
    rc = upload(st, &p->ystart); if (rc) return rc;
    rc = upload(si, &p->ysi); if (rc) return rc;
    rc = upload(al, &p->ybeta); if (rc) return rc;
    std::vector<double> c((size_t)4 * n);
    const double pi = 3.141592653589793;
    for (int k = 0; k < 4 * n; ++k) c[k] = cos(pi * k / (2.0 * n));   // numpy: cos(pi * k / (2 n)), same expression
    rc = upload(c, &p->cosn); if (rc) return rc;
    // folded levels: level k+1 exists while level k has even length
    p->levels = 1; p->len[0] = n; p->off[0] = 0;
    int off = 0;
    while ((p->len[p->levels - 1] & 1) == 0 && p->len[p->levels - 1] > 1 && p->levels < 8) {
        p->len[p->levels] = p->len[p->levels - 1] / 2;
        p->off[p->levels] = off;
        off += p->len[p->levels];
        p->levels += 1;
    }
    // the finish kernel's working set per frame: image and column levels (2 n^2), t and its levels (2 size n),
    // the low band (size^2 floats); in shared memory while it fits, else in a global workspace
    const int64_t m = (int64_t)size * size;
    p->ws_doubles = ((2 * n64 * n64 + 2 * (int64_t)size * n64 + (m + 1) / 2) + 1) & ~(int64_t)1;
    int dev = 0, smem_optin = 0;
    PSD_CUDA(cudaGetDevice(&dev));
    PSD_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    p->global_ws = force_global_ws || (size_t)p->ws_doubles * sizeof(double) > (size_t)smem_optin - kHashStaticSmem;
    // frames per sub-batch: the row buffer and the workspace together stay within kHashWorkspaceBytes
    // (or one frame's worth, if that is larger)
    const int64_t per_frame = (int64_t)H * n * (int64_t)sizeof(float) +
                              (p->global_ws ? p->ws_doubles * (int64_t)sizeof(double) : 0);
    p->batch = (int)std::max<int64_t>(1, std::min<int64_t>(max_batch, kHashWorkspaceBytes / per_frame));
    PSD_CUDA(cudaMalloc(&p->rowbuf, (size_t)p->batch * H * n * sizeof(float)));
    if (p->global_ws) PSD_CUDA(cudaMalloc(&p->ws, (size_t)p->batch * p->ws_doubles * sizeof(double)));
    return PSD_OK;
}

void hash_plan_destroy(HashPlan* p) {
    cudaFree(p->xstart); cudaFree(p->xsi); cudaFree(p->xmid); cudaFree(p->xalpha); cudaFree(p->ystart); cudaFree(p->ysi);
    cudaFree(p->ybeta); cudaFree(p->cosn); cudaFree(p->rowbuf); cudaFree(p->ws);
    *p = HashPlan{};
}

static int launch_hash_finish(const HashPlan& p, int nb, int H, uint64_t* out, cudaStream_t stream) {
    FoldPlan fp{};
    fp.levels = p.levels;
    for (int k = 0; k < 8; ++k) { fp.len[k] = p.len[k]; fp.off[k] = p.off[k]; }
    const size_t smem = p.global_ws ? 0 : (size_t)p.ws_doubles * sizeof(double);
    if (p.global_ws) {
        psd_hash_finish_kernel<true><<<(unsigned)nb, 256, 0, stream>>>(
            p.rowbuf, H, p.n, p.size, p.fast, p.area_w, p.area_h, p.ystart, p.ysi, p.ybeta, p.cosn, fp, p.ws,
            p.ws_doubles, p.words, out);
    } else {
        PSD_CUDA(cudaFuncSetAttribute(psd_hash_finish_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        psd_hash_finish_kernel<false><<<(unsigned)nb, 256, smem, stream>>>(
            p.rowbuf, H, p.n, p.size, p.fast, p.area_w, p.area_h, p.ystart, p.ysi, p.ybeta, p.cosn, fp, nullptr, 0,
            p.words, out);
    }
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

int launch_hash(const HashPlan* plans, int n_plans, const uint8_t* frames, int64_t frame_stride, int n_frames, int W,
                int H, uint64_t* const* hashes, cudaStream_t stream) {
    PSD_REQUIRE(n_plans >= 1, "launch_hash: no hash plan");
    // rows kernel: max(1, 256 / n) source rows per CTA for the smallest hash image n, as many as fit
    // kHashRowsSmemBytes of gray bytes in shared memory (a small n on a wide frame: 256 rows of 1920 would not);
    // the row buffers do not depend on the block height.  A sub-batch fits every plan's row buffer and workspace.
    int n_min = plans[0].n, batch = plans[0].batch;
    for (int g = 1; g < n_plans; ++g) { n_min = std::min(n_min, plans[g].n); batch = std::min(batch, plans[g].batch); }
    const int pitch = ((W + 3) & ~3) + 4;
    PSD_REQUIRE(pitch <= kHashRowsSmemBytes, "frame too wide for the hash rows kernel (%d columns)", W);
    const int rows_per_cta = std::max(1, std::min(256 / n_min, kHashRowsSmemBytes / pitch));
    const size_t smem_rows = (size_t)rows_per_cta * pitch;
    PSD_CUDA(cudaFuncSetAttribute(psd_hash_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rows));
    for (int f0 = 0; f0 < n_frames; f0 += batch) {   // sub-batches share the row buffers and the workspaces
        const int nb = std::min(batch, n_frames - f0);
        dim3 rgrid((unsigned)((H + rows_per_cta - 1) / rows_per_cta), (unsigned)nb);
        for (int g0 = 0; g0 < n_plans; g0 += kHashRowsMaxGeo) {
            HashRowsArgs geo{};
            geo.count = std::min(kHashRowsMaxGeo, n_plans - g0);
            for (int i = 0; i < geo.count; ++i) {
                const HashPlan& p = plans[g0 + i];
                geo.g[i] = HashRowsGeo{p.xstart, p.xsi, p.xalpha, p.xmid, p.rowbuf, p.n, p.fast};
            }
            psd_hash_rows_kernel<<<rgrid, 256, smem_rows, stream>>>(frames + f0 * frame_stride, frame_stride, W, H,
                                                                    rows_per_cta, pitch, geo);
            PSD_CHECK_LAUNCH();
            count_launch();
        }
        for (int g = 0; g < n_plans; ++g) {
            const int rc = launch_hash_finish(plans[g], nb, H, hashes[g] + (int64_t)f0 * plans[g].words, stream);
            if (rc) return rc;
        }
    }
    return PSD_OK;
}

int launch_hash_dist(const uint64_t* hashes, int64_t n, int size, const uint64_t* prev_hash, double* out,
                     cudaStream_t stream) {
    if (n <= 0) return PSD_OK;
    psd_scan_hash_dist_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(hashes, n, PSD_HASH_WORDS_FOR(size),
                                                                          (double)size * size, prev_hash, out);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

}  // namespace psd

// ---- test hook: every stage of the hash pass through the production kernels ----
extern "C" int psd_test_hash_stages(int device, const void* frames, int64_t n_frames, int32_t width, int32_t height,
                                    int64_t frame_stride, const int32_t* geometries, int32_t n_geo, float* rowbuf_out,
                                    uint64_t* hash_out, double* image_out, float* low_out) {
    using namespace psd;
    PSD_REQUIRE(frames && geometries && hash_out, "psd_test_hash_stages: null argument");
    PSD_REQUIRE(n_frames >= 1 && n_frames <= (1 << 30), "psd_test_hash_stages: bad frame count %lld", (long long)n_frames);
    PSD_REQUIRE(n_geo >= 1 && n_geo <= 16, "psd_test_hash_stages: 1 to 16 geometries, not %d", n_geo);
    PSD_REQUIRE(width >= 1 && height >= 1 && frame_stride >= (int64_t)width * height * 3,
                "psd_test_hash_stages: bad frame size or stride");
    PSD_CUDA(cudaSetDevice(device));
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, frames) != cudaSuccess) cudaGetLastError();
    PSD_REQUIRE((at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == device,
                "psd_test_hash_stages: frames are not memory of device %d", device);
    const bool force_global = image_out || low_out;
    struct Owned {   // released on every return
        std::vector<HashPlan> plans;
        uint64_t* d_hash = nullptr;
        ~Owned() { for (HashPlan& p : plans) hash_plan_destroy(&p); cudaFree(d_hash); }
    } o;
    o.plans.resize(n_geo);
    int64_t words_total = 0;
    for (int g = 0; g < n_geo; ++g) {
        HashPlan& p = o.plans[g];
        const int rc = hash_plan_create(&p, width, height, geometries[2 * g], geometries[2 * g + 1], (int)n_frames,
                                        force_global);
        if (rc) return rc;
        PSD_REQUIRE(!(rowbuf_out || force_global) || p.batch >= n_frames,
                    "psd_test_hash_stages: the stages of %lld frames need %lld frames per sub-batch, geometry %d has %d",
                    (long long)n_frames, (long long)n_frames, g, p.batch);
        words_total += n_frames * p.words;
    }
    PSD_CUDA(cudaMalloc(&o.d_hash, (size_t)words_total * sizeof(uint64_t)));
    std::vector<uint64_t*> outs(n_geo);
    for (int64_t g = 0, w = 0; g < n_geo; w += n_frames * o.plans[g].words, ++g) outs[g] = o.d_hash + w;
    int rc = launch_hash(o.plans.data(), n_geo, (const uint8_t*)frames, frame_stride, (int)n_frames, width, height,
                         outs.data(), 0);
    if (rc) return rc;
    PSD_CUDA(cudaDeviceSynchronize());
    PSD_CUDA(cudaMemcpy(hash_out, o.d_hash, (size_t)words_total * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    for (const HashPlan& p : o.plans) {
        const int64_t n2 = (int64_t)p.n * p.n, m = (int64_t)p.size * p.size;
        if (rowbuf_out) {
            const int64_t cnt = n_frames * height * p.n;
            PSD_CUDA(cudaMemcpy(rowbuf_out, p.rowbuf, (size_t)cnt * sizeof(float), cudaMemcpyDeviceToHost));
            rowbuf_out += cnt;
        }
        for (int64_t f = 0; f < n_frames && force_global; ++f) {
            const double* ws = p.ws + f * p.ws_doubles;   // x [n][n] at 0, the low band after 2 n^2 + 2 size n
            if (image_out)
                PSD_CUDA(cudaMemcpy(image_out + f * n2, ws, (size_t)n2 * sizeof(double), cudaMemcpyDeviceToHost));
            if (low_out)
                PSD_CUDA(cudaMemcpy(low_out + f * m, ws + 2 * n2 + 2 * (int64_t)p.size * p.n, (size_t)m * sizeof(float),
                                    cudaMemcpyDeviceToHost));
        }
        if (image_out) image_out += n_frames * n2;
        if (low_out) low_out += n_frames * m;
    }
    return PSD_OK;
}
