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

// The horizontal pass.  A CTA takes a block of consecutive source rows of one frame (256 / n of them):
//   1. all threads pull the block - it is contiguous in memory - 16 pixels (three 16-byte loads) at a time,
//      convert to gray and park the gray bytes in shared memory (row pitch W rounded up + 4: two rows of a
//      1920-wide frame would otherwise sit in the same banks);
//   2. thread (row, destination column) walks its taps in shared memory: the integer block sum if both scale
//      factors are integers, else OpenCV's float32 `buf += S * alpha` in source order (separate multiply and
//      add: the order and the roundings decide the last bit, so this chain stays sequential).
// (The first version had one thread per (row, column) read its 3 x 120 bytes straight from global memory, 32
// lanes 360 bytes apart: 0.085 of the HBM roofline.)
__global__ void __launch_bounds__(256) psd_hash_rows_kernel(const uint8_t* __restrict__ frames, int64_t frame_stride,
                                                            int W, int H, int n, int rows_per_cta, int pitch, int fast,
                                                            const int32_t* __restrict__ xstart,
                                                            const int32_t* __restrict__ xsi,
                                                            const float* __restrict__ xalpha,
                                                            const int32_t* __restrict__ xmid,
                                                            float* __restrict__ rowbuf) {
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
    // ---- 2. one thread per (row, destination column) ----
    const int r = tid / n, dx = tid - r * n;
    if (r >= rows) return;
    const uint8_t* srow = sgray + r * pitch;
    float* out = rowbuf + (f * H + sy0 + r) * (int64_t)n + dx;
    if (fast) {  // integer scale: exact integer sum of the block's columns
        const int sxw = W / n;
        uint32_t s = 0;
        for (int x = dx * sxw; x < (dx + 1) * sxw; ++x) s += srow[x];
        *out = __uint_as_float(s);
    } else {
        // first (partial) tap, the run of whole pixels, last (partial) tap - in source order
        float buf = 0.0f;
        const int k0 = xstart[dx], k1 = xstart[dx + 1];
        const int km = xmid[2 * dx], nm = xmid[2 * dx + 1];
        for (int k = k0; k < km; ++k) buf = __fadd_rn(buf, __fmul_rn(byte_to_float(srow[xsi[k]]), xalpha[k]));
        if (nm > 0) {
            const uint8_t* sp = srow + xsi[km];
            const float am = xalpha[km];
#pragma unroll 8
            for (int i = 0; i < nm; ++i) buf = __fadd_rn(buf, __fmul_rn(byte_to_float(sp[i]), am));
        }
        for (int k = km + nm; k < k1; ++k) buf = __fadd_rn(buf, __fmul_rn(byte_to_float(srow[xsi[k]]), xalpha[k]));
        *out = buf;
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

// one CTA per frame: vertical pass, normalisation, DCT low band, median, bits
constexpr int kHashMaxN = 64, kHashMaxSize = 16;
__global__ void __launch_bounds__(256) psd_hash_finish_kernel(const float* __restrict__ rowbuf, int H, int n, int size,
                                                              int fast, int area_w, int area_h,
                                                              const int32_t* __restrict__ ystart,
                                                              const int32_t* __restrict__ ysi,
                                                              const float* __restrict__ ybeta,
                                                              const double* __restrict__ costab /* [4n] cos(pi k / 2n) */,
                                                              FoldPlan fp,
                                                              uint64_t* __restrict__ hashes /* [frames][PSD_HASH_WORDS] */) {
    extern __shared__ __align__(16) double dsm[];
    double* x = dsm;                    // [n][n] normalised image (row i, column j)
    double* lev = x + n * n;            // [n][n]: folded levels of every column j (element e of column j at lev[e*n + j])
    double* t = lev + n * n;            // [size][n]: vertical transform, t[u][j]
    double* lev2 = t + size * n;        // [n][size]: folded levels of every t[u][.] (element e of row u at lev2[e*size + u])
    __shared__ float low[kHashMaxSize * kHashMaxSize];
    __shared__ uint32_t mx;
    __shared__ float med;
    __shared__ float mid[2];
    __shared__ unsigned long long bits[PSD_HASH_WORDS];
    const int tid = threadIdx.x;
    const int64_t f = blockIdx.x;
    const float* rb = rowbuf + f * (int64_t)H * n;
    if (tid == 0) mx = 0;
    if (tid < PSD_HASH_WORDS) bits[tid] = 0ull;
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
    // numpy.median: rank every element (ties broken by index), pick the middle one / the float32 mean of the two
    for (int c = tid; c < m; c += 256) {
        const float a = low[c];
        int rank = 0;
        for (int k = 0; k < m; ++k) rank += (low[k] < a) || (low[k] == a && k < c);
        if (m & 1) { if (rank == m / 2) mid[0] = mid[1] = a; }
        else { if (rank == m / 2 - 1) mid[0] = a; if (rank == m / 2) mid[1] = a; }
    }
    __syncthreads();
    if (tid == 0) med = (m & 1) ? mid[0] : __fmul_rn(__fadd_rn(mid[0], mid[1]), 0.5f);
    __syncthreads();
    for (int c = tid; c < m; c += 256)
        if (low[c] > med) atomicOr(&bits[c >> 6], 1ull << (c & 63));
    __syncthreads();
    if (tid < PSD_HASH_WORDS) hashes[f * PSD_HASH_WORDS + tid] = bits[tid];
}

// hash_detector.py:95-99: Hamming distance to the previous frame's hash, divided by size * size
__global__ void psd_scan_hash_dist_kernel(const uint64_t* __restrict__ hashes, int64_t n, double size_sq,
                                          const uint64_t* __restrict__ prev_hash, double* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t* cur = hashes + i * PSD_HASH_WORDS;
    const uint64_t* prv = (i > 0) ? cur - PSD_HASH_WORDS : prev_hash;
    if (prv == nullptr) { out[i] = __longlong_as_double(0x7FF8000000000000LL); return; }
    int cnt = 0;
#pragma unroll
    for (int w = 0; w < PSD_HASH_WORDS; ++w) cnt += __popcll(cur[w] ^ prv[w]);
    out[i] = __ddiv_rn((double)cnt, size_sq);
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

int hash_plan_create(HashPlan* p, int W, int H, int size, int lowpass, int max_batch) {
    PSD_REQUIRE(size >= 1 && size <= kHashMaxSize && lowpass >= 1 && size * lowpass <= kHashMaxN,
                "HashDetector on the GPU needs size <= %d and size * lowpass <= %d", kHashMaxSize, kHashMaxN);
    const int n = size * lowpass;
    PSD_REQUIRE(W >= n && H >= n, "frames smaller than the %dx%d hash image are not supported", n, n);
    p->n = n; p->size = size;
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
    PSD_CUDA(cudaMalloc(&p->rowbuf, (size_t)max_batch * H * n * sizeof(float)));
    return PSD_OK;
}

void hash_plan_destroy(HashPlan* p) {
    cudaFree(p->xstart); cudaFree(p->xsi); cudaFree(p->xmid); cudaFree(p->xalpha); cudaFree(p->ystart); cudaFree(p->ysi);
    cudaFree(p->ybeta); cudaFree(p->cosn); cudaFree(p->rowbuf);
    *p = HashPlan{};
}

int launch_hash(const HashPlan& p, const uint8_t* frames, int64_t frame_stride, int n_frames, int W, int H,
                uint64_t* hashes, cudaStream_t stream) {
    // rows kernel: 256 / n source rows per CTA, their gray bytes in shared memory
    const int rows_per_cta = 256 / p.n;
    const int pitch = ((W + 3) & ~3) + 4;
    const size_t smem_rows = (size_t)rows_per_cta * pitch;
    PSD_REQUIRE(smem_rows <= 200 * 1024, "frame too wide for the hash rows kernel (%d columns)", W);
    PSD_CUDA(cudaFuncSetAttribute(psd_hash_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rows));
    dim3 rgrid((unsigned)((H + rows_per_cta - 1) / rows_per_cta), (unsigned)n_frames);
    psd_hash_rows_kernel<<<rgrid, 256, smem_rows, stream>>>(frames, frame_stride, W, H, p.n, rows_per_cta, pitch, p.fast,
                                                            p.xstart, p.xsi, p.xalpha, p.xmid, p.rowbuf);
    PSD_CHECK_LAUNCH();
    FoldPlan fp{};
    fp.levels = p.levels;
    for (int k = 0; k < 8; ++k) { fp.len[k] = p.len[k]; fp.off[k] = p.off[k]; }
    const size_t smem = ((size_t)2 * p.n * p.n + (size_t)p.size * p.n + (size_t)p.n * p.size) * sizeof(double);
    PSD_CUDA(cudaFuncSetAttribute(psd_hash_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    psd_hash_finish_kernel<<<(unsigned)n_frames, 256, smem, stream>>>(p.rowbuf, H, p.n, p.size, p.fast, p.area_w, p.area_h,
                                                                     p.ystart, p.ysi, p.ybeta, p.cosn, fp, hashes);
    PSD_CHECK_LAUNCH();
    count_launch(2);
    return PSD_OK;
}

int launch_hash_dist(const uint64_t* hashes, int64_t n, int size, const uint64_t* prev_hash, double* out,
                     cudaStream_t stream) {
    if (n <= 0) return PSD_OK;
    psd_scan_hash_dist_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(hashes, n, (double)(size * size), prev_hash, out);
    PSD_CHECK_LAUNCH();
    count_launch();
    return PSD_OK;
}

}  // namespace psd
