// psd_jpeg_decode: BGR images of a batch of baseline JPEG files, the bytes cv2.imread(path, IMREAD_COLOR) gives
// (libjpeg-turbo: jdhuff.c, jidctint.c islow, jdsample.c fancy upsampling, jdcolor.c ycc_rgb_convert), and
// psd_jpeg_probe, the host-side marker parser that says which files it takes.
//
// Every step is the library's integer arithmetic (tests/jpeg_decode_twin.py restates each one).  Per sub-batch of
// files, on one stream:
//   jd_destuff_kernel (count)   one thread per 256 bytes of a file's entropy-coded data: bytes kept once stuffed zeros,
//                               RSTn markers and fill bytes are dropped; psd_clip_scan_kernel -> offsets
//   jd_destuff_kernel (write)   the kept bytes, packed per file; the restart bitmap marks the bytes that begin an
//                               interval; any other marker inside the data is a bitstream error
//   jd_sync_init_kernel         self-synchronising Huffman decoding (Weissenberger & Schmidt, ICPP 2018): thread k
//                               decodes subsequence k (256 bytes of packed data) from its first bit, as if a block of
//                               MCU position 0 started there, and records the first block start at or past its end
//   jd_sync_check_kernel        (kSyncRounds parallel update rounds first, see the kernel) thread k decodes
//                               subsequence k again from the state its predecessor recorded; where the
//                               exit state differs from the one recorded for k + 1, that state is marked unsynchronised
//   jd_sync_fix_kernel          one warp per file walks the marked states in order and re-decodes until they agree
//                               (almost never needed: a decode from a wrong start meets the true one within a few
//                               blocks); every subsequence then knows its true start and its block count
//   psd_clip_scan_kernel        block counts -> each subsequence's first block
//   jd_write_kernel             thread k decodes its blocks once more and writes their coefficients (DC differences)
//   jd_dc_kernel                one CTA per (file, component): DC differences -> DCs, restarting every interval
//   jd_idct_kernel              one thread per block: dequantise, jidctint.c islow, range_limit -> component planes
//   jd_color_kernel             one thread per pixel: h2v1 / h2v2 fancy upsampling, ycc_rgb_convert, written B, G, R
//                               through the output's psd_frame_layout
// A file whose data does not decode (a bad code, a coefficient past 63, a missing or misplaced restart marker, the
// wrong number of blocks) gets a nonzero error flag; the kernels never read outside the file's bytes.
#include <string.h>

#include <algorithm>
#include <vector>

#include "psd_common.cuh"

namespace psd {
namespace jdec {

constexpr int kSubBytes = 256;       // packed bytes per subsequence of the entropy decode
constexpr int kStuffBytes = 256;     // raw bytes per thread of the destuffing pass
constexpr int kThreads = 128;
constexpr int kLut = 9;              // bits of the first-level Huffman lookup
constexpr int kSyncRounds = 2;       // parallel rounds of start-state updates ahead of the check

constexpr uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t kNat[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// jdhuff.c jpeg_make_d_derived_tbl: a first-level table of kLut bits (length << 8 | symbol, 0 where the code is
// longer), then maxcode / valoffset per length and the symbols
struct Huff {
    uint16_t lut[1 << kLut];
    int32_t maxcode[18];
    int32_t valoffset[18];
    uint8_t vals[256];
};

struct Img {
    const uint8_t* src;          // the file (device)
    int64_t scan0, scan1;        // its entropy-coded data: bytes [scan0, scan1)
    int64_t stuff0, n_stuff;     // its destuffing threads in the sub-batch
    int64_t sub0, n_sub;         // its subsequences in the sub-batch
    int64_t packed0;             // its packed data in Batch::packed (a multiple of 16 bytes)
    int64_t coef0;               // its first block in Batch::coefs
    int64_t plane0[3];           // its component planes in Batch::planes
    int32_t plane_w[3], plane_h[3];  // their sizes: whole blocks
    int32_t width, height, ncomp, bpm, mcus_x, mcus_y, restart;
    int32_t hmax, vmax;          // luma sampling factors
    int32_t n_blocks;            // mcus_x * mcus_y * bpm
    int8_t comp_of[6], dx_of[6], dy_of[6];  // MCU block position -> component, block column and row in the MCU
    uint16_t quant[3][64];       // natural order
    Huff dc[3], ac[3];           // by component
    uint8_t* out;                // B of pixel (0, 0)
    int64_t row_stride, pixel_stride, channel_stride;
};

struct Batch {
    const Img* images;
    const int32_t* stuff_image;  // [n_stuff]
    const int32_t* sub_image;    // [n_sub]
    int64_t* stuff_off;          // [n_stuff + 1] kept bytes per thread, then their offsets
    uint8_t* packed;             // the packed data of every image
    uint32_t* rst;               // restart bitmap over `packed`: bit b = an interval starts at packed byte b
    int64_t* start;              // [n_sub] start state of every subsequence (pos << 3 | MCU position)
    uint8_t* unsynced;           // [n_sub] start[k] was not confirmed by its predecessor's decode
    int32_t* any_unsynced;       // [n_images]
    int64_t* counts;             // [n_sub + 1] blocks per subsequence, then their offsets
    int16_t* coefs;              // [blocks][64] natural order
    uint8_t* planes;
    int32_t* errors;             // [n_images] of the sub-batch
};

__device__ __forceinline__ int64_t packed_bytes(const Batch& bt, const Img& im) {
    return bt.stuff_off[im.stuff0 + im.n_stuff] - bt.stuff_off[im.stuff0];
}

// ---- destuffing ----
// Raw byte i of the data is kept unless it is a stuffed 0x00, either byte of an RSTn marker or a fill 0xFF; a marker
// other than RSTn inside the data is an error.  Decisions read only bytes i - 1 and i + 1.
enum { kKeep = 0, kDrop = 1, kRst = 2, kBad = 3 };
__device__ __forceinline__ int classify(const uint8_t* d, int64_t i, int64_t lo, int64_t hi) {
    const uint8_t b = d[i];
    const uint8_t prev = i > lo ? d[i - 1] : 0;
    if (b == 0xFF) {
        const uint8_t nx = i + 1 < hi ? d[i + 1] : 0xFF;
        if (nx == 0x00) return kKeep;
        if (nx >= 0xD0 && nx <= 0xD7) return kRst;
        if (nx == 0xFF) return kDrop;
        return kBad;
    }
    if (prev == 0xFF && (b == 0x00 || (b >= 0xD0 && b <= 0xD7))) return kDrop;
    return kKeep;
}

template <bool WRITE>
__global__ void __launch_bounds__(kThreads) jd_destuff_kernel(Batch bt, int64_t n_stuff) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_stuff) return;
    const int i = bt.stuff_image[t];
    const Img& im = bt.images[i];
    const int64_t lo = im.scan0, hi = im.scan1;
    const int64_t b0 = lo + (t - im.stuff0) * kStuffBytes, b1 = min(b0 + kStuffBytes, hi);
    const uint8_t* d = im.src;
    if (!WRITE) {
        int64_t n = 0;
        for (int64_t b = b0; b < b1; ++b) n += classify(d, b, lo, hi) == kKeep;
        bt.stuff_off[t] = n;
        return;
    }
    int64_t o = bt.stuff_off[t] - bt.stuff_off[im.stuff0];
    uint8_t* out = bt.packed + im.packed0;
    bool bad = false;
    for (int64_t b = b0; b < b1; ++b) {
        const int c = classify(d, b, lo, hi);
        if (c == kKeep) out[o++] = d[b];
        else if (c == kRst) {
            const int64_t bit = im.packed0 + o;
            atomicOr(bt.rst + (bit >> 5), 1u << (bit & 31));
        } else if (c == kBad) bad = true;
    }
    if (bad) bt.errors[i] = 1;
}

// ---- Huffman decoding ----
struct Reader {
    const uint8_t* p;  // the image's packed bytes
    int64_t nbits;     // 8 * packed bytes
    // 32 bits from bit pos, MSB first; 1-bits past the end
    __device__ __forceinline__ uint32_t peek(int64_t pos) const {
        const int64_t byte = pos >> 3;
        uint64_t w = 0;
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int64_t b = byte + k;
            w = (w << 8) | (b * 8 < nbits ? p[b] : 0xFFu);
        }
        return (uint32_t)(w >> (8 - (pos & 7)));
    }
};

// one Huffman symbol at pos: the symbol (pos advanced), or -1 for a code the table lacks (pos advanced by 1)
__device__ __forceinline__ int huff_decode(const Huff& h, const Reader& r, int64_t& pos) {
    const uint32_t bits = r.peek(pos);
    const uint32_t e = h.lut[bits >> (32 - kLut)];
    if (e) {
        pos += e >> 8;
        return e & 255;
    }
    for (int l = kLut + 1; l <= 16; ++l) {
        const int32_t code = (int32_t)(bits >> (32 - l));
        if (code <= h.maxcode[l]) {
            pos += l;
            return h.vals[(code + h.valoffset[l]) & 255];
        }
    }
    pos += 1;
    return -1;
}

__device__ __forceinline__ int extend(uint32_t v, int s) {
    return s == 0 ? 0 : (v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v);
}

// jdhuff.c decode_mcu for one block of MCU position blk from pos: coefficients (the DC as its difference) into out
// if given.  False on a bitstream error (a code the table lacks, a coefficient past 63).
__device__ __forceinline__ bool decode_block(const Img& im, const Reader& r, int64_t& pos, int blk, int16_t* out) {
    const int c = im.comp_of[blk];
    int s = huff_decode(im.dc[c], r, pos);
    if (s < 0 || s > 15) return false;
    const int dc = extend(s ? r.peek(pos) >> (32 - s) : 0, s);
    pos += s;
    if (out) out[0] = (int16_t)dc;
    for (int k = 1; k < 64;) {
        const int rs = huff_decode(im.ac[c], r, pos);
        if (rs < 0) return false;
        const int run = rs >> 4, size = rs & 15;
        if (size) {
            k += run;
            if (k > 63) return false;
            const int v = extend(r.peek(pos) >> (32 - size), size);
            pos += size;
            if (out) out[kNat[k]] = (int16_t)v;
            ++k;
        } else if (run == 15) {
            k += 16;
        } else {
            break;
        }
    }
    return true;
}

// At an MCU start: padding 1-bits up to a byte where a restart interval (or the data) begins are skipped
__device__ __forceinline__ bool skip_padding(const Batch& bt, const Img& im, const Reader& r, int64_t& pos) {
    const int64_t byte = (pos + 7) >> 3;
    const int pad = (int)(8 * byte - pos);
    if (pad && (r.peek(pos) >> (32 - pad)) != (1u << pad) - 1) return false;
    const int64_t bit = im.packed0 + byte;
    const bool at_rst = 8 * byte < r.nbits && ((bt.rst[bit >> 5] >> (bit & 31)) & 1u);
    if (at_rst || 8 * byte >= r.nbits) {
        pos = 8 * byte;
        return at_rst;
    }
    return false;
}

struct SubResult {
    int64_t exit;   // state at the first block start at or past the subsequence's end
    int64_t count;  // blocks that start inside it
    bool ok;        // no bitstream error on the way
};

// Decodes subsequence k of image im from `state` (pos << 3 | MCU position).  WRITE: blocks go to the image's
// coefficients from block `first` on, checked against the MCU positions and restart intervals they must have.
template <bool WRITE>
__device__ __forceinline__ SubResult decode_sub(const Batch& bt, const Img& im, int64_t k, int64_t state, int64_t first) {
    const Reader r{bt.packed + im.packed0, 8 * packed_bytes(bt, im)};
    const int64_t end = min((k + 1) * kSubBytes * 8, r.nbits);
    int64_t pos = state >> 3;
    int blk = (int)(state & 7);
    SubResult res{0, 0, true};
    while (pos < end) {
        bool rst = false;
        if (blk == 0) {
            rst = skip_padding(bt, im, r, pos);
            if (pos >= end) break;
        }
        if (WRITE) {
            const int64_t b = first + res.count;
            const int64_t mcu = b / im.bpm;
            const bool want_rst = im.restart && mcu > 0 && mcu % im.restart == 0 && blk == 0;
            if (b >= im.n_blocks || b % im.bpm != blk || rst != want_rst) {
                res.ok = false;
                break;
            }
            if (!decode_block(im, r, pos, blk, bt.coefs + (im.coef0 + b) * 64)) {
                res.ok = false;
                break;
            }
        } else if (!decode_block(im, r, pos, blk, nullptr)) {
            res.ok = false;
        }
        ++res.count;
        blk = blk + 1 == im.bpm ? 0 : blk + 1;
    }
    // a block that reads past the data: libjpeg-turbo would decode it from zero bits, this reader gave it 1-bits
    if (WRITE && pos > r.nbits) res.ok = false;
    if (pos >= r.nbits) {
        pos = r.nbits;
        blk = 0;
    }
    res.exit = pos << 3 | blk;
    return res;
}

__global__ void __launch_bounds__(kThreads) jd_sync_init_kernel(Batch bt, int64_t n_sub) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_sub) return;
    const int i = bt.sub_image[t];
    const Img& im = bt.images[i];
    const int64_t k = t - im.sub0;
    const int64_t nbits = 8 * packed_bytes(bt, im);
    const int64_t pos0 = min(k * kSubBytes * 8, nbits);
    if (k == 0) bt.start[t] = 0;
    if (k + 1 < im.n_sub) bt.start[t + 1] = decode_sub<false>(bt, im, k, pos0 << 3, 0).exit;
}

// UPDATE: a round of the iteration start[k + 1] = exit(k, start[k]) for every k at once, for the states a subsequence
// was too short to synchronise (start[k] may be rewritten by thread k - 1 meanwhile: at a fixed point every start is
// its predecessor's exit, so the rounds only shorten the serial walk of jd_sync_fix_kernel).  Otherwise the check.
template <bool UPDATE>
__global__ void __launch_bounds__(kThreads, 8) jd_sync_check_kernel(Batch bt, int64_t n_sub) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_sub) return;
    const int i = bt.sub_image[t];
    const Img& im = bt.images[i];
    const int64_t k = t - im.sub0;
    const SubResult r = decode_sub<false>(bt, im, k, ((volatile int64_t*)bt.start)[t], 0);
    if (UPDATE) {
        if (k + 1 < im.n_sub && r.exit != bt.start[t + 1]) bt.start[t + 1] = r.exit;
        return;
    }
    bt.counts[t] = r.count;
    const bool bad = k + 1 < im.n_sub && r.exit != bt.start[t + 1];
    if (k + 1 < im.n_sub) bt.unsynced[t + 1] = bad;
    if (bad) bt.any_unsynced[i] = 1;
}

// one warp per image: start[k] for every k whose predecessor's decode disagreed, in order, until they agree again
__global__ void __launch_bounds__(32) jd_sync_fix_kernel(Batch bt) {
    const int i = blockIdx.x;
    const Img& im = bt.images[i];
    if (!bt.any_unsynced[i]) return;
    const int lane = threadIdx.x;
    int64_t k = 1;
    while (k < im.n_sub) {
        // the next marked state at or after k
        const int64_t j = k + lane;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, j < im.n_sub && bt.unsynced[im.sub0 + j]);
        if (!m) {
            k += 32;
            continue;
        }
        k += __ffs(m) - 1;
        if (lane == 0) {
            // start[k - 1] is true: decode k - 1 from it; while the exit changes the next start, go on
            for (;; ++k) {
                const int64_t t = im.sub0 + k - 1;
                const SubResult r = decode_sub<false>(bt, im, k - 1, bt.start[t], 0);
                bt.counts[t] = r.count;
                if (k == im.n_sub || r.exit == bt.start[t + 1]) break;
                bt.start[t + 1] = r.exit;
            }
        }
        k = __shfl_sync(0xFFFFFFFFu, k, 0) + 1;
    }
}

__global__ void __launch_bounds__(kThreads) jd_write_kernel(Batch bt, int64_t n_sub) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_sub) return;
    const int i = bt.sub_image[t];
    const Img& im = bt.images[i];
    const int64_t k = t - im.sub0;
    const int64_t first = bt.counts[t] - bt.counts[im.sub0];
    if (k + 1 == im.n_sub && bt.counts[t + 1] - bt.counts[im.sub0] != im.n_blocks) bt.errors[i] = 1;
    if (!decode_sub<true>(bt, im, k, bt.start[t], first).ok) bt.errors[i] = 1;
}

// DC differences -> DCs of component c of image i (blockIdx.x = 3 * i + c), restarting at every restart interval:
// a segmented scan over the component's blocks in scan order, int32 sums stored as int16 ((JCOEF)s)
__global__ void __launch_bounds__(256) jd_dc_kernel(Batch bt) {
    const int i = blockIdx.x / 3, c = blockIdx.x % 3;
    const Img& im = bt.images[i];
    if (c >= im.ncomp) return;
    __shared__ int32_t wsum[8];
    __shared__ int32_t wflag[8];
    __shared__ int32_t carry_s;
    int nc = 0, off = 0;
    for (int b = 0; b < im.bpm; ++b) {
        if (im.comp_of[b] == c) {
            if (!nc) off = b;
            ++nc;
        }
    }
    const int64_t n = (int64_t)im.mcus_x * im.mcus_y * nc;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int32_t carry = 0;
    for (int64_t base = 0; base < n; base += 256) {
        const int64_t e = base + threadIdx.x;
        int32_t v = 0, f = 0;
        int16_t* p = nullptr;
        if (e < n) {
            const int64_t mcu = e / nc;
            const int j = (int)(e % nc);
            p = bt.coefs + (im.coef0 + mcu * im.bpm + off + j) * 64;
            v = *p;
            f = (j == 0 && im.restart && mcu % im.restart == 0) ? 1 : 0;
        }
        // inclusive segmented scan within the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t v2 = __shfl_up_sync(0xFFFFFFFFu, v, o);
            const int32_t f2 = __shfl_up_sync(0xFFFFFFFFu, f, o);
            if (lane >= o) {
                if (!f) v += v2;
                f |= f2;
            }
        }
        if (lane == 31) {
            wsum[w] = v;
            wflag[w] = f;
        }
        __syncthreads();
        // prefix of the warps before this one, and the carry from the previous tile, unless a segment starts between
        int32_t pre = carry;
        for (int k = 0; k < w; ++k) pre = wflag[k] ? wsum[k] : pre + wsum[k];
        if (!f) v += pre;
        if (p) *p = (int16_t)v;
        if (threadIdx.x == 255) carry_s = v;
        __syncthreads();
        carry = carry_s;
        __syncthreads();
    }
}

// jidctint.c jpeg_idct_islow: one block per thread, dequantised with the component's table, into its plane
__global__ void __launch_bounds__(kThreads) jd_idct_kernel(Batch bt, int64_t n_blocks, const int32_t* block_image) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_blocks) return;
    const int i = block_image[g];
    const Img& im = bt.images[i];
    const int64_t b = g - im.coef0;
    if (b >= im.n_blocks) return;
    const int64_t mcu = b / im.bpm;
    const int blk = (int)(b % im.bpm);
    const int c = im.comp_of[blk];
    const int hc = c == 0 ? im.hmax : 1, vc = c == 0 ? im.vmax : 1;
    const int64_t bx = (mcu % im.mcus_x) * hc + im.dx_of[blk], by = (mcu / im.mcus_x) * vc + im.dy_of[blk];
    const int16_t* in = bt.coefs + g * 64;
    const uint16_t* q = im.quant[c];
    int ws[64];
    constexpr int kConst = 13, kPass1 = 2;
    // pass 1: columns
#pragma unroll
    for (int col = 0; col < 8; ++col) {
        int d[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) d[r] = (int)in[8 * r + col] * (int)q[8 * r + col];
        if (!(d[1] | d[2] | d[3] | d[4] | d[5] | d[6] | d[7])) {
            const int dc = d[0] * (1 << kPass1);
#pragma unroll
            for (int r = 0; r < 8; ++r) ws[8 * r + col] = dc;
            continue;
        }
        int z2 = d[2], z3 = d[6];
        int z1 = (z2 + z3) * 4433;
        const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
        const int tmp0 = (d[0] + d[4]) * (1 << kConst), tmp1 = (d[0] - d[4]) * (1 << kConst);
        const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        int t0 = d[7], t1 = d[5], t2 = d[3], t3 = d[1];
        z1 = t0 + t3;
        z2 = t1 + t2;
        z3 = t0 + t2;
        int z4 = t1 + t3;
        const int z5 = (z3 + z4) * 9633;
        t0 *= 2446;
        t1 *= 16819;
        t2 *= 25172;
        t3 *= 12299;
        z1 *= -7373;
        z2 *= -20995;
        z3 = z3 * -16069 + z5;
        z4 = z4 * -3196 + z5;
        t0 += z1 + z3;
        t1 += z2 + z4;
        t2 += z2 + z3;
        t3 += z1 + z4;
        constexpr int n = kConst - kPass1;
        ws[col] = (tmp10 + t3 + (1 << (n - 1))) >> n;
        ws[56 + col] = (tmp10 - t3 + (1 << (n - 1))) >> n;
        ws[8 + col] = (tmp11 + t2 + (1 << (n - 1))) >> n;
        ws[48 + col] = (tmp11 - t2 + (1 << (n - 1))) >> n;
        ws[16 + col] = (tmp12 + t1 + (1 << (n - 1))) >> n;
        ws[40 + col] = (tmp12 - t1 + (1 << (n - 1))) >> n;
        ws[24 + col] = (tmp13 + t0 + (1 << (n - 1))) >> n;
        ws[32 + col] = (tmp13 - t0 + (1 << (n - 1))) >> n;
    }
    // pass 2: rows; range_limit[x & 1023] = clamp(x as a signed 10-bit value + 128)
    auto limit = [](int x) {
        const int s = ((x & 1023) ^ 512) - 512;
        return (uint32_t)min(max(s + 128, 0), 255);
    };
    uint8_t* plane = bt.planes + im.plane0[c] + by * 8 * im.plane_w[c] + bx * 8;
#pragma unroll
    for (int row = 0; row < 8; ++row) {
        const int* d = ws + 8 * row;
        uint32_t o[8];
        constexpr int n = kConst + kPass1 + 3;
        int z2 = d[2], z3 = d[6];
        int z1 = (z2 + z3) * 4433;
        const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
        const int tmp0 = (d[0] + d[4]) * (1 << kConst), tmp1 = (d[0] - d[4]) * (1 << kConst);
        const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        int t0 = d[7], t1 = d[5], t2 = d[3], t3 = d[1];
        z1 = t0 + t3;
        z2 = t1 + t2;
        z3 = t0 + t2;
        int z4 = t1 + t3;
        const int z5 = (z3 + z4) * 9633;
        t0 *= 2446;
        t1 *= 16819;
        t2 *= 25172;
        t3 *= 12299;
        z1 *= -7373;
        z2 *= -20995;
        z3 = z3 * -16069 + z5;
        z4 = z4 * -3196 + z5;
        t0 += z1 + z3;
        t1 += z2 + z4;
        t2 += z2 + z3;
        t3 += z1 + z4;
        // the all-zero-AC row shortcut DESCALE(d[0], PASS1_BITS + 3) equals this
        o[0] = limit((tmp10 + t3 + (1 << (n - 1))) >> n);
        o[7] = limit((tmp10 - t3 + (1 << (n - 1))) >> n);
        o[1] = limit((tmp11 + t2 + (1 << (n - 1))) >> n);
        o[6] = limit((tmp11 - t2 + (1 << (n - 1))) >> n);
        o[2] = limit((tmp12 + t1 + (1 << (n - 1))) >> n);
        o[5] = limit((tmp12 - t1 + (1 << (n - 1))) >> n);
        o[3] = limit((tmp13 + t0 + (1 << (n - 1))) >> n);
        o[4] = limit((tmp13 - t0 + (1 << (n - 1))) >> n);
        uint2 v;
        v.x = o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24;
        v.y = o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24;
        *reinterpret_cast<uint2*>(plane + (int64_t)row * im.plane_w[c]) = v;
    }
}

// jdsample.c upsampling of chroma plane p to output pixel (x, y): h2v1 / h2v2 fancy (triangle filters, biases 1 / 2
// and 8 / 7 alternating, edges replicated) when the downsampled width is above 2, else replication
__device__ __forceinline__ int chroma_at(const uint8_t* p, int pw, int dw, int dh, int h2, int v2, int x, int y) {
    if (!h2 && !v2) return p[(int64_t)y * pw + x];
    const int cx = h2 ? x >> 1 : x, cy = v2 ? y >> 1 : y;
    if (dw <= 2) return p[(int64_t)cy * pw + cx];
    const int nx = (x & 1) ? min(cx + 1, dw - 1) : max(cx - 1, 0);
    if (!v2) {
        const uint8_t* r = p + (int64_t)cy * pw;
        return (3 * r[cx] + r[nx] + 1 + (x & 1)) >> 2;
    }
    const int ny = (y & 1) ? min(cy + 1, dh - 1) : max(cy - 1, 0);
    const uint8_t* r0 = p + (int64_t)cy * pw;
    const uint8_t* r1 = p + (int64_t)ny * pw;
    const int t = 3 * r0[cx] + r1[cx], tn = 3 * r0[nx] + r1[nx];
    return (3 * t + tn + 8 - (x & 1)) >> 4;
}

__constant__ int32_t kCrR[256], kCbB[256], kCrG[256], kCbG[256];  // jdcolor.c build_ycc_rgb_table

__global__ void __launch_bounds__(256) jd_color_kernel(Batch bt, int64_t n_rows, const int32_t* row_image,
                                                       const int32_t* row_first) {
    const int64_t rr = blockIdx.x;
    if (rr >= n_rows) return;
    const int i = row_image[rr];
    const Img& im = bt.images[i];
    const int y = (int)(rr - row_first[rr]);
    const int x = blockIdx.y * blockDim.x + threadIdx.x;
    if (x >= im.width) return;
    const int Y = bt.planes[im.plane0[0] + (int64_t)y * im.plane_w[0] + x];
    int b = Y, g = Y, r = Y;
    if (im.ncomp == 3) {
        const int h2 = im.hmax == 2, v2 = im.vmax == 2;
        const int dw = (im.width + im.hmax - 1) / im.hmax, dh = (im.height + im.vmax - 1) / im.vmax;
        const int cb = chroma_at(bt.planes + im.plane0[1], im.plane_w[1], dw, dh, h2, v2, x, y);
        const int cr = chroma_at(bt.planes + im.plane0[2], im.plane_w[2], dw, dh, h2, v2, x, y);
        r = min(max(Y + kCrR[cr], 0), 255);
        g = min(max(Y + ((kCbG[cb] + kCrG[cr]) >> 16), 0), 255);
        b = min(max(Y + kCbB[cb], 0), 255);
    }
    uint8_t* o = im.out + (int64_t)y * im.row_stride + (int64_t)x * im.pixel_stride;
    o[0] = (uint8_t)b;
    o[im.channel_stride] = (uint8_t)g;
    o[2 * im.channel_stride] = (uint8_t)r;
}

// ---- host side ----
struct Parsed {
    psd_jpeg_info info;
    int ids[3], tq[3], td[3], ta[3];
    bool have_q[4], have_dc[4], have_ac[4];
    uint16_t q[4][64];
    uint8_t dc_bits[4][16], ac_bits[4][16];
    uint8_t dc_vals[4][256], ac_vals[4][256];
};

int exif_orientation(const uint8_t* s, int64_t n) {
    if (n < 14 || memcmp(s, "Exif\0\0", 6) != 0) return 1;
    const uint8_t* t = s + 6;
    const int64_t tn = n - 6;
    bool le;
    if (t[0] == 'I' && t[1] == 'I') le = true;
    else if (t[0] == 'M' && t[1] == 'M') le = false;
    else return 1;
    auto u16 = [&](int64_t o) { return le ? t[o] | t[o + 1] << 8 : t[o] << 8 | t[o + 1]; };
    auto u32 = [&](int64_t o) {
        return le ? (uint32_t)t[o] | (uint32_t)t[o + 1] << 8 | (uint32_t)t[o + 2] << 16 | (uint32_t)t[o + 3] << 24
                  : (uint32_t)t[o] << 24 | (uint32_t)t[o + 1] << 16 | (uint32_t)t[o + 2] << 8 | (uint32_t)t[o + 3];
    };
    const int64_t off = u32(4);
    if (off + 2 > tn) return 1;
    const int cnt = u16(off);
    for (int e = 0; e < cnt; ++e) {
        const int64_t p = off + 2 + 12 * (int64_t)e;
        if (p + 12 > tn) break;
        if (u16(p) == 0x0112 && u16(p + 2) == 3) return u16(p + 8);
    }
    return 1;
}

// the marker walk of tests/jpeg_decode_twin.py:probe
int parse(const uint8_t* d, int64_t n, Parsed& P) {
    memset(&P, 0, sizeof(P));
    psd_jpeg_info& I = P.info;
    auto refuse = [&](int code) { return I.refusal = code; };
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return refuse(PSD_JPEG_NOT_JPEG);
    int64_t p = 2;
    bool sof = false;
    int adobe = -1;
    bool jfif = false;
    for (;;) {
        while (p < n && d[p] != 0xFF) ++p;
        while (p < n && d[p] == 0xFF) ++p;
        if (p >= n) return refuse(PSD_JPEG_TRUNCATED);
        const int m = d[p++];
        if (m == 0xD9) return refuse(PSD_JPEG_TRUNCATED);
        if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
        if (p + 2 > n) return refuse(PSD_JPEG_TRUNCATED);
        const int64_t L = d[p] << 8 | d[p + 1];
        if (L < 2 || p + L > n) return refuse(PSD_JPEG_TRUNCATED);
        const uint8_t* s = d + p + 2;
        const int64_t sl = L - 2;
        if (m == 0xC0 || m == 0xC1) {
            if (sof) return refuse(PSD_JPEG_MULTI_SCAN);
            if (sl < 6) return refuse(PSD_JPEG_TRUNCATED);
            sof = true;
            if (s[0] != 8) return refuse(PSD_JPEG_PRECISION);
            I.height = s[1] << 8 | s[2];
            I.width = s[3] << 8 | s[4];
            I.components = s[5];
            if (I.components != 1 && I.components != 3) return refuse(PSD_JPEG_COMPONENTS);
            if (sl < 6 + 3 * I.components || I.width == 0 || I.height == 0) return refuse(PSD_JPEG_TRUNCATED);
            int hs[3], vs[3];
            for (int c = 0; c < I.components; ++c) {
                P.ids[c] = s[6 + 3 * c];
                hs[c] = s[7 + 3 * c] >> 4;
                vs[c] = s[7 + 3 * c] & 15;
                P.tq[c] = s[8 + 3 * c];
            }
            I.h_samp = I.v_samp = 1;
            if (I.components == 3) {
                if (hs[1] != 1 || vs[1] != 1 || hs[2] != 1 || vs[2] != 1 ||
                    !((hs[0] == 1 && vs[0] == 1) || (hs[0] == 2 && vs[0] == 1) || (hs[0] == 2 && vs[0] == 2)))
                    return refuse(PSD_JPEG_SAMPLING);
                I.h_samp = hs[0];
                I.v_samp = vs[0];
            }
        } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            return refuse(PSD_JPEG_PROCESS);
        } else if (m == 0xCC) {
            return refuse(PSD_JPEG_PROCESS);
        } else if (m == 0xC4) {
            int64_t q = 0;
            while (q < sl) {
                if (q + 17 > sl) return refuse(PSD_JPEG_TRUNCATED);
                const int tc = s[q] >> 4, th = s[q] & 15;
                int cnt = 0;
                for (int l = 0; l < 16; ++l) cnt += s[q + 1 + l];
                if (q + 17 + cnt > sl || tc > 1 || th > 3 || cnt > 256) return refuse(PSD_JPEG_TABLES);
                memcpy(tc ? P.ac_bits[th] : P.dc_bits[th], s + q + 1, 16);
                memcpy(tc ? P.ac_vals[th] : P.dc_vals[th], s + q + 17, (size_t)cnt);
                (tc ? P.have_ac : P.have_dc)[th] = true;
                q += 17 + cnt;
            }
        } else if (m == 0xDB) {
            int64_t q = 0;
            while (q < sl) {
                const int pq = s[q] >> 4, tq = s[q] & 15;
                const int64_t size = 64 * (pq ? 2 : 1);
                if (q + 1 + size > sl || tq > 3) return refuse(PSD_JPEG_TABLES);
                for (int z = 0; z < 64; ++z)
                    P.q[tq][kNatural[z]] = pq ? (uint16_t)(s[q + 1 + 2 * z] << 8 | s[q + 2 + 2 * z]) : s[q + 1 + z];
                P.have_q[tq] = true;
                q += 1 + size;
            }
        } else if (m == 0xDD) {
            if (sl < 2) return refuse(PSD_JPEG_TRUNCATED);
            I.restart_interval = s[0] << 8 | s[1];
        } else if (m == 0xE0) {
            if (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;   // jdmarker.c examine_app0
        } else if (m == 0xEE) {
            if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = s[11];
        } else if (m == 0xE1) {
            const int o = exif_orientation(s, sl);
            if (o != 0 && o != 1) return refuse(PSD_JPEG_ORIENTATION);
        } else if (m == 0xDA) {
            if (!sof) return refuse(PSD_JPEG_TRUNCATED);
            const int ns = sl >= 1 ? s[0] : 0;
            if (ns != I.components) return refuse(PSD_JPEG_MULTI_SCAN);
            if (sl < 1 + 2 * ns + 3) return refuse(PSD_JPEG_TRUNCATED);
            for (int c = 0; c < ns; ++c) {
                if (s[1 + 2 * c] != P.ids[c]) return refuse(PSD_JPEG_MULTI_SCAN);
                P.td[c] = s[2 + 2 * c] >> 4;
                P.ta[c] = s[2 + 2 * c] & 15;
                if (P.td[c] > 3 || P.ta[c] > 3 || P.tq[c] > 3 || !P.have_dc[P.td[c]] || !P.have_ac[P.ta[c]] ||
                    !P.have_q[P.tq[c]])
                    return refuse(PSD_JPEG_TABLES);
            }
            // jdapimin.c default_decompress_parms: without a JFIF marker, an Adobe transform of 0, or (no Adobe
            // marker) component ids 'R', 'G', 'B', make the file RGB, which libjpeg does not convert from YCbCr
            if (I.components == 3 && !jfif &&
                (adobe == 0 || (adobe < 0 && P.ids[0] == 'R' && P.ids[1] == 'G' && P.ids[2] == 'B')))
                return refuse(PSD_JPEG_COMPONENTS);
            I.scan_begin = p + L;
            int64_t e = n - 2;
            while (e >= I.scan_begin && !(d[e] == 0xFF && d[e + 1] == 0xD9)) --e;
            if (e < I.scan_begin) return refuse(PSD_JPEG_TRUNCATED);
            I.scan_end = e;
            return PSD_JPEG_OK;
        }
        p += L;
    }
}

// jdhuff.c jpeg_make_d_derived_tbl; false for an over-subscribed table
bool derive(const uint8_t* bits, const uint8_t* vals, bool dc, Huff& h) {
    memset(&h, 0, sizeof(h));
    int size[257], code[257], k = 0;
    for (int l = 1; l <= 16; ++l)
        for (int i = 0; i < bits[l - 1]; ++i) size[k++] = l;
    const int n = k;
    if (n == 0) return false;
    int c = 0, si = size[0];
    k = 0;
    while (k < n) {
        while (k < n && size[k] == si) code[k++] = c++;
        if (c >= (1 << si)) return false;
        c <<= 1;
        ++si;
    }
    int p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (bits[l - 1]) {
            h.valoffset[l] = p - code[p];
            p += bits[l - 1];
            h.maxcode[l] = code[p - 1];
        } else {
            h.maxcode[l] = -1;
        }
    }
    h.maxcode[17] = 0x7FFFFFFF;
    for (int i = 0; i < n; ++i) {
        h.vals[i] = vals[i];
        if (dc && vals[i] > 15) return false;
        if (size[i] <= kLut) {
            const int lo = code[i] << (kLut - size[i]), cnt = 1 << (kLut - size[i]);
            for (int j = 0; j < cnt; ++j) h.lut[lo + j] = (uint16_t)(size[i] << 8 | vals[i]);
        }
    }
    return true;
}

struct Sizes {
    int64_t stuff = 0, sub = 0, packed = 0, blocks = 0, planes = 0, rows = 0, images = 0;
    int64_t bytes() const {
        return stuff * (8 + 4) + 8 + packed + packed / 8 + 64 + sub * (8 + 1 + 8 + 4) + 8 + blocks * (128 + 4) +
               planes + rows * 8 + images * (int64_t)(sizeof(Img) + 8) + 16 * 16;
    }
};

bool g_tables = false;
int upload_color_tables() {
    if (g_tables) return PSD_OK;
    int32_t rr[256], bb[256], rg[256], bg[256];
    auto fix = [](double x) { return (int32_t)(x * 65536.0 + 0.5); };
    for (int i = 0; i < 256; ++i) {
        const int x = i - 128;
        rr[i] = (fix(1.40200) * x + 32768) >> 16;
        bb[i] = (fix(1.77200) * x + 32768) >> 16;
        rg[i] = -fix(0.71414) * x;
        bg[i] = -fix(0.34414) * x + 32768;
    }
    PSD_CUDA(cudaMemcpyToSymbol(kCrR, rr, sizeof(rr)));
    PSD_CUDA(cudaMemcpyToSymbol(kCbB, bb, sizeof(bb)));
    PSD_CUDA(cudaMemcpyToSymbol(kCrG, rg, sizeof(rg)));
    PSD_CUDA(cudaMemcpyToSymbol(kCbG, bg, sizeof(bg)));
    g_tables = true;
    return PSD_OK;
}

}  // namespace jdec
}  // namespace psd

using namespace psd;
using namespace psd::jdec;

extern "C" int psd_jpeg_probe(const uint8_t* data, int64_t size, psd_jpeg_info* info) {
    PSD_REQUIRE(info && (data || size == 0) && size >= 0, "psd_jpeg_probe: bad arguments");
    Parsed* P = new Parsed;
    parse(data, size, *P);
    if (P->info.refusal == PSD_JPEG_OK) {
        Huff h;
        for (int c = 0; c < P->info.components && P->info.refusal == PSD_JPEG_OK; ++c)
            if (!derive(P->dc_bits[P->td[c]], P->dc_vals[P->td[c]], true, h) ||
                !derive(P->ac_bits[P->ta[c]], P->ac_vals[P->ta[c]], false, h))
                P->info.refusal = PSD_JPEG_TABLES;
    }
    *info = P->info;
    delete P;
    return PSD_OK;
}

extern "C" int psd_jpeg_decode(int device, const psd_jpeg_source* srcs, int32_t n, const psd_jpeg_image* images,
                               int64_t workspace_cap, int32_t* error_flags, void* stream) {
    PSD_REQUIRE(n >= 0 && workspace_cap >= 0, "psd_jpeg_decode: bad image count or workspace_cap");
    PSD_REQUIRE(n == 0 || (srcs && images && error_flags), "psd_jpeg_decode: no sources, images or error_flags");
    PSD_CUDA(cudaSetDevice(device));
    cudaStream_t s = (cudaStream_t)stream;
    int rc = PSD_OK;
    if (n == 0) return PSD_OK;
    if ((rc = require_device_memory(error_flags, device, "psd_jpeg_decode error_flags"))) return rc;
    if ((rc = upload_color_tables())) return rc;
    std::vector<Img> im((size_t)n);
    std::vector<Parsed> parsed(1);
    for (int32_t i = 0; i < n; ++i) {
        const psd_jpeg_source& x = srcs[i];
        PSD_REQUIRE(x.host && x.device && x.size > 0, "psd_jpeg_decode: file %d has no bytes", i);
        char what[64];
        snprintf(what, sizeof(what), "psd_jpeg_decode file %d", i);
        if ((rc = require_device_memory(x.device, device, what))) return rc;
        Parsed& P = parsed[0];
        parse((const uint8_t*)x.host, x.size, P);
        const psd_jpeg_info& I = P.info;
        PSD_REQUIRE(I.refusal == PSD_JPEG_OK, "psd_jpeg_decode: file %d is not a JPEG this decoder takes (refusal %d)",
                    i, I.refusal);
        const psd_jpeg_image& o = images[i];
        PSD_REQUIRE(o.base, "psd_jpeg_decode: image %d has no pixels", i);
        PSD_REQUIRE(o.width == I.width && o.height == I.height,
                    "psd_jpeg_decode: image %d is %d x %d, its file %d x %d", i, o.width, o.height, I.width,
                    I.height);
        snprintf(what, sizeof(what), "psd_jpeg_decode image %d", i);
        if ((rc = require_device_memory(o.base, device, what))) return rc;
        Img& m = im[i];
        memset(&m, 0, sizeof(Img));
        m.src = (const uint8_t*)x.device;
        m.scan0 = I.scan_begin;
        m.scan1 = I.scan_end;
        m.width = I.width;
        m.height = I.height;
        m.ncomp = I.components;
        m.hmax = I.h_samp;
        m.vmax = I.v_samp;
        m.restart = I.restart_interval;
        m.mcus_x = (I.width + 8 * m.hmax - 1) / (8 * m.hmax);
        m.mcus_y = (I.height + 8 * m.vmax - 1) / (8 * m.vmax);
        int k = 0;
        for (int c = 0; c < m.ncomp; ++c) {
            const int hc = c ? 1 : m.hmax, vc = c ? 1 : m.vmax;
            for (int dy = 0; dy < vc; ++dy)
                for (int dx = 0; dx < hc; ++dx) {
                    m.comp_of[k] = (int8_t)c;
                    m.dx_of[k] = (int8_t)dx;
                    m.dy_of[k] = (int8_t)dy;
                    ++k;
                }
            m.plane_w[c] = 8 * m.mcus_x * hc;
            m.plane_h[c] = 8 * m.mcus_y * vc;
            memcpy(m.quant[c], P.q[P.tq[c]], sizeof(m.quant[c]));
            PSD_REQUIRE(derive(P.dc_bits[P.td[c]], P.dc_vals[P.td[c]], true, m.dc[c]) &&
                            derive(P.ac_bits[P.ta[c]], P.ac_vals[P.ta[c]], false, m.ac[c]),
                        "psd_jpeg_decode: file %d has a bad Huffman table", i);
        }
        m.bpm = k;
        m.n_blocks = m.mcus_x * m.mcus_y * m.bpm;
        const int64_t raw = m.scan1 - m.scan0;
        m.n_stuff = std::max<int64_t>(1, (raw + kStuffBytes - 1) / kStuffBytes);
        m.n_sub = std::max<int64_t>(1, (raw + kSubBytes - 1) / kSubBytes);
        m.out = (uint8_t*)o.base;
        m.row_stride = o.layout.row_stride;
        m.pixel_stride = o.layout.pixel_stride;
        m.channel_stride = o.layout.channel_stride;
    }
    auto need = [](const Img& m, Sizes& z) {
        z.stuff += m.n_stuff;
        z.sub += m.n_sub;
        z.packed += ((m.scan1 - m.scan0) + 16 + 127) & ~(int64_t)127;
        z.blocks += m.n_blocks;
        for (int c = 0; c < m.ncomp; ++c) z.planes += (((int64_t)m.plane_w[c] * m.plane_h[c]) + 15) & ~(int64_t)15;
        z.rows += m.height;
        z.images += 1;
    };
    const int64_t cap = workspace_cap ? workspace_cap : (int64_t)512 << 20;
    std::vector<int32_t> first = {0};
    Sizes big, cur;
    for (int32_t i = 0; i < n; ++i) {
        Sizes nx = cur;
        need(im[i], nx);
        if (cur.images > 0 && nx.bytes() > cap) {
            first.push_back(i);
            nx = Sizes{};
            need(im[i], nx);
        }
        cur = nx;
        big.stuff = std::max(big.stuff, cur.stuff);
        big.sub = std::max(big.sub, cur.sub);
        big.packed = std::max(big.packed, cur.packed);
        big.blocks = std::max(big.blocks, cur.blocks);
        big.planes = std::max(big.planes, cur.planes);
        big.rows = std::max(big.rows, cur.rows);
        big.images = std::max(big.images, cur.images);
    }
    first.push_back(n);
    uint8_t* ws = nullptr;
    PSD_CUDA(cudaMallocAsync((void**)&ws, (size_t)big.bytes(), s));
    struct Free {
        uint8_t* p;
        cudaStream_t s;
        ~Free() { cudaFreeAsync(p, s); }
    } owned{ws, s};
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = ws + off;
        off += (bytes + 15) & ~(size_t)15;
        return p;
    };
    Batch bt{};
    bt.stuff_off = (int64_t*)take((size_t)(big.stuff + 1) * 8);
    bt.packed = take((size_t)big.packed);
    bt.rst = (uint32_t*)take((size_t)big.packed / 8 + 16);
    bt.start = (int64_t*)take((size_t)big.sub * 8);
    bt.unsynced = take((size_t)big.sub);
    bt.counts = (int64_t*)take((size_t)(big.sub + 1) * 8);
    bt.any_unsynced = (int32_t*)take((size_t)big.images * 4);
    bt.coefs = (int16_t*)take((size_t)big.blocks * 128);
    bt.planes = take((size_t)big.planes);
    Img* d_images = (Img*)take((size_t)big.images * sizeof(Img));
    int32_t* d_stuff_image = (int32_t*)take((size_t)big.stuff * 4);
    int32_t* d_sub_image = (int32_t*)take((size_t)big.sub * 4);
    int32_t* d_block_image = (int32_t*)take((size_t)big.blocks * 4);
    int32_t* d_row_image = (int32_t*)take((size_t)big.rows * 4);
    int32_t* d_row_first = (int32_t*)take((size_t)big.rows * 4);
    bt.images = d_images;
    bt.stuff_image = d_stuff_image;
    bt.sub_image = d_sub_image;
    PSD_CUDA(cudaMemsetAsync(error_flags, 0, sizeof(int32_t) * (size_t)n, s));
    std::vector<int32_t> stuff_image, sub_image, block_image, row_image, row_first;
    for (size_t b = 0; b + 1 < first.size(); ++b) {
        const int32_t i0 = first[b], nb = first[b + 1] - first[b];
        stuff_image.clear();
        sub_image.clear();
        block_image.clear();
        row_image.clear();
        row_first.clear();
        int64_t packed = 0, planes = 0, max_w = 1;
        for (int32_t j = 0; j < nb; ++j) {
            Img& m = im[i0 + j];
            m.stuff0 = (int64_t)stuff_image.size();
            m.sub0 = (int64_t)sub_image.size();
            m.coef0 = (int64_t)block_image.size();
            m.packed0 = packed;
            packed += ((m.scan1 - m.scan0) + 16 + 127) & ~(int64_t)127;
            for (int c = 0; c < m.ncomp; ++c) {
                m.plane0[c] = planes;
                planes += (((int64_t)m.plane_w[c] * m.plane_h[c]) + 15) & ~(int64_t)15;
            }
            stuff_image.insert(stuff_image.end(), (size_t)m.n_stuff, j);
            sub_image.insert(sub_image.end(), (size_t)m.n_sub, j);
            block_image.insert(block_image.end(), (size_t)m.n_blocks, j);
            const int32_t r0 = (int32_t)row_image.size();
            row_image.insert(row_image.end(), (size_t)m.height, j);
            row_first.insert(row_first.end(), (size_t)m.height, r0);
            max_w = std::max<int64_t>(max_w, m.width);
        }
        const int64_t n_stuff = (int64_t)stuff_image.size(), n_sub = (int64_t)sub_image.size();
        const int64_t n_blocks = (int64_t)block_image.size(), n_rows = (int64_t)row_image.size();
        PSD_CUDA(cudaMemcpyAsync(d_images, &im[i0], sizeof(Img) * nb, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_stuff_image, stuff_image.data(), 4 * n_stuff, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_sub_image, sub_image.data(), 4 * n_sub, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_block_image, block_image.data(), 4 * n_blocks, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_row_image, row_image.data(), 4 * n_rows, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_row_first, row_first.data(), 4 * n_rows, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemsetAsync(bt.rst, 0, (size_t)packed / 8 + 16, s));
        PSD_CUDA(cudaMemsetAsync(bt.unsynced, 0, (size_t)n_sub, s));
        PSD_CUDA(cudaMemsetAsync(bt.any_unsynced, 0, 4 * (size_t)nb, s));
        PSD_CUDA(cudaMemsetAsync(bt.coefs, 0, (size_t)n_blocks * 128, s));
        bt.errors = error_flags + i0;
        auto grid = [](int64_t m) { return (unsigned)((m + kThreads - 1) / kThreads); };
        jd_destuff_kernel<false><<<grid(n_stuff), kThreads, 0, s>>>(bt, n_stuff);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(bt.stuff_off, n_stuff);
        PSD_CHECK_LAUNCH();
        jd_destuff_kernel<true><<<grid(n_stuff), kThreads, 0, s>>>(bt, n_stuff);
        PSD_CHECK_LAUNCH();
        jd_sync_init_kernel<<<grid(n_sub), kThreads, 0, s>>>(bt, n_sub);
        PSD_CHECK_LAUNCH();
        for (int round = 0; round < kSyncRounds; ++round) {
            jd_sync_check_kernel<true><<<grid(n_sub), kThreads, 0, s>>>(bt, n_sub);
            PSD_CHECK_LAUNCH();
        }
        jd_sync_check_kernel<false><<<grid(n_sub), kThreads, 0, s>>>(bt, n_sub);
        PSD_CHECK_LAUNCH();
        jd_sync_fix_kernel<<<(unsigned)nb, 32, 0, s>>>(bt);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(bt.counts, n_sub);
        PSD_CHECK_LAUNCH();
        jd_write_kernel<<<grid(n_sub), kThreads, 0, s>>>(bt, n_sub);
        PSD_CHECK_LAUNCH();
        jd_dc_kernel<<<(unsigned)(3 * nb), 256, 0, s>>>(bt);
        PSD_CHECK_LAUNCH();
        jd_idct_kernel<<<grid(n_blocks), kThreads, 0, s>>>(bt, n_blocks, d_block_image);
        PSD_CHECK_LAUNCH();
        const dim3 cg((unsigned)n_rows, (unsigned)((max_w + 255) / 256));
        jd_color_kernel<<<cg, 256, 0, s>>>(bt, n_rows, d_row_image, d_row_first);
        PSD_CHECK_LAUNCH();
        count_launch(11 + kSyncRounds);
    }
    return PSD_OK;
}
