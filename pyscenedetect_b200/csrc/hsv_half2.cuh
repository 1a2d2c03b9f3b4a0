// Per-pixel colour arithmetic of the fused score pass and the test hook.
//
// Exact restatement of OpenCV's 8-bit BGR->HSV (H in [0,180)) and BGR->YUV-Y, the arithmetic
// behind content_detector.py:155 and histogram_detector.py:156 (see oracle/intmath.py, which is
// pinned against cv2 over all 2^24 colours):
//   V = max(B,G,R), d = V - min(B,G,R)
//   S = (d * sdiv[V] + 2048) >> 12,           sdiv[i] = rint((255<<12) / i),     sdiv[0] = 0
//   h = (V==R) ? G-B : (V==G) ? B-R+2d : R-G+4d
//   H = (h * hdiv[d] + 2048) >> 12 (arithmetic), hdiv[i] = rint((180<<12) / (6 i)), hdiv[0] = 0
//   H += 180 if H < 0
//   Y = (R*4899 + G*9617 + B*1868 + 8192) >> 14
//
// HSV: the numerator stage runs on pixel PAIRS in packed 16-bit lanes, so most instructions serve
// two pixels.  ("variant 7" in DESIGN.md's history of formulations.)
//
// The fused pass is issue-bound (one warp instruction per clock per sub-partition), so the lever is
// the instruction COUNT per pixel; this formulation needs ~20:
//   * bytes are lifted straight into half2 "magic" lanes 0x6400 | x = 1024 + x (ulp 1), 8 PRMT/LOP3
//     per 4 pixels instead of 12 single-byte lifts;
//   * V = max3, mn = min3 are ONE VIMNMX3.U16x2 each per pair (the magic bit patterns order like the
//     bytes); d = V - mn is exact both as half2 (HADD2) and as integer lanes (plain IADD, no borrow);
//   * the three hue numerators G-B, B-R+2d, R-G+4d (|.| <= 1275 < 2048: exact in fp16) are
//     HADD2/HFMA2 on pairs; the R > G > B tie priority becomes two HSET2 lane masks + two LOP3
//     selects per pair;
//   * only the two table products stay per pixel and in fp32: HADD2.F32 lifts a lane of d / h,
//     yS = fma.rz(d, sdiv/4096, 32768.5), yH = fma.rm(h, hdiv/4096, 49152.5): the FMA is exact before its
//     single rounding, RZ / RM at ulp 2^-8 only drop fraction bits and the integer part lands in bits 8..15
//     (byte 1 of the result = S resp. H mod 256); each LUT row address is built by one IDP2A
//     (u16 lane x 128 + addend);
//   * "H += 180 if H < 0" is applied after packing, on four pixels at once: H mod 256 is either
//     0..179 or 226..255, so a byte is negative iff its bits 7 and 6 are both set, and adding 180
//     mod 256 equals subtracting 76 without a borrow.
// Every step is an exact integer identity; pinned over all 2^24 colours by tests/test_gpu_parity.py
// (psd_test_hsv) and restated in numpy by tests/v7_model.py, which
// tests/test_v7_model.py pins against the oracle over all 2^24 colours on the CPU.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

namespace psd {

struct Px16 {  // 16 pixels, planar, 4 pixels per 32-bit word (pixel 4j+i in byte i of word j)
    uint32_t h[4], s[4], v[4];
};

__device__ __forceinline__ uint32_t y_px(uint32_t b, uint32_t g, uint32_t r) {
    return (r * 4899u + g * 9617u + b * 1868u + 8192u) >> 14;
}

// Y of pixel P straight from the packed words with IDP4A: the 14-bit coefficients are split into
// (lo, hi) bytes, 1868 = 7*256+76, 9617 = 37*256+145, 4899 = 19*256+35, so
// Y = (dp4a(w, lo) + 256 * dp4a(w, hi) + 8192) >> 14 with per-byte-position coefficient words.
__host__ __device__ constexpr uint32_t y_coef_word(int word, int k0, int which) {
    // which: 0 = lo bytes (76,145,35 for B,G,R), 1 = hi bytes (7,37,19)
    uint32_t r = 0;
    for (int b = 0; b < 4; ++b) {
        const int g = 4 * word + b - k0;  // 0,1,2 -> B,G,R of this pixel
        uint32_t c = 0;
        if (g == 0) c = which ? 7u : 76u;
        if (g == 1) c = which ? 37u : 145u;
        if (g == 2) c = which ? 19u : 35u;
        r |= c << (8 * b);
    }
    return r;
}

template <int P>
__device__ __forceinline__ uint32_t y_of_pixel(const uint32_t (&w)[12]) {
    constexpr int k0 = 3 * P, j0 = k0 >> 2, j1 = (k0 + 2) >> 2;
    uint32_t lo = __dp4a(w[j0], y_coef_word(j0, k0, 0), 8192u);
    uint32_t hi = __dp4a(w[j0], y_coef_word(j0, k0, 1), 0u);
    if (j1 != j0) {
        lo = __dp4a(w[j1], y_coef_word(j1, k0, 0), lo);
        hi = __dp4a(w[j1], y_coef_word(j1, k0, 1), hi);
    }
    return (hi * 256u + lo) >> 14;
}

// byte k (0..47) of 12 packed words
__device__ __forceinline__ uint32_t byte_of(const uint32_t (&w)[12], int k) {
    return (w[k >> 2] >> ((k & 3) * 8)) & 0xFFu;
}

// The LUT is replicated per lane (32 copies of each of the 2 x 256 table values, 64 KB): rows of 128 B in two
// tables (sdiv | hdiv), lane l reads word l of a row, so any 32 lookups hit 32 distinct banks.
struct LutView7 {
    uint32_t cs;    // addend of the sdiv row address: (0x6400 + V) * 128 + cs = table + V * 128 + lane * 4
    uint32_t ch;    // addend of the hdiv row address: d * 128 + ch
};

__device__ __forceinline__ LutView7 make_lut7(uint32_t lut_smem_addr, int lane) {
    LutView7 l;
    l.cs = lut_smem_addr + (uint32_t)lane * 4u - 0x6400u * 128u;
    l.ch = lut_smem_addr + 32768u + (uint32_t)lane * 4u;  // hdiv table follows the sdiv table
    return l;
}

// fills the LUT: value = table integer / 4096 (exact in fp32: < 2^21 and a power-of-two divisor)
__device__ __forceinline__ void lut_fill7(float* lut, int tid, int nthreads) {
    for (int t = tid; t < 512; t += nthreads) {
        const int row = t >> 1, which = t & 1;
        float v = 0.0f;
        if (row) {
            const int q = which ? __double2int_rn(737280.0 / (6.0 * (double)row))
                                : __double2int_rn(1044480.0 / (double)row);
            v = (float)q * 0.000244140625f;
        }
        float4* dst = reinterpret_cast<float4*>(lut + which * 8192 + row * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[j] = make_float4(v, v, v, v);
    }
}

namespace v7 {

__device__ __forceinline__ __half2 as_h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
__device__ __forceinline__ uint32_t as_u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

__device__ __forceinline__ uint32_t hsub2u(uint32_t a, uint32_t b) { return as_u32(__hsub2(as_h2(a), as_h2(b))); }
__device__ __forceinline__ uint32_t hfma2u(uint32_t a, uint32_t b, uint32_t c) {
    return as_u32(__hfma2(as_h2(a), as_h2(b), as_h2(c)));
}
__device__ __forceinline__ uint32_t heq2m(uint32_t a, uint32_t b) { return __heq2_mask(as_h2(a), as_h2(b)); }
// m ? x : y per bit
__device__ __forceinline__ uint32_t bitsel(uint32_t m, uint32_t x, uint32_t y) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xCA;" : "=r"(r) : "r"(m), "r"(x), "r"(y));
    return r;
}
// (t & 0x00FF00FF) | 0x64006400
__device__ __forceinline__ uint32_t even_bytes_magic(uint32_t t) {
    uint32_t r;
    asm("lop3.b32 %0, %1, 0x00FF00FF, %2, 0xEA;" : "=r"(r) : "r"(t), "r"(0x64006400u));  // (a & b) | c
    return r;
}
__device__ __forceinline__ float lds(uint32_t addr) {
    float r;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(addr));
    return r;
}
__device__ __forceinline__ float fma_rz_(float a, float b, float c) {
    float r;
    asm("fma.rz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
}
__device__ __forceinline__ float fma_rm_(float a, float b, float c) {
    float r;
    asm("fma.rm.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
}

struct PairOut7 {
    uint32_t yh0, yh1, ys0, ys1;  // fp32 bit patterns, value in byte 1
    uint32_t vh;                  // half2 magic lanes: byte 0 = V of lane 0, byte 2 = V of lane 1
};

// Bh, Gh, Rh: magic half2 lanes of one pixel pair.
__device__ __forceinline__ void pair(uint32_t Bh, uint32_t Gh, uint32_t Rh, const LutView7& lut, PairOut7& o) {
    const uint32_t Vh = __vimax3_u16x2(Bh, Gh, Rh);
    const uint32_t mh = __vimin3_u16x2(Bh, Gh, Rh);
    const uint32_t dh = hsub2u(Vh, mh);  // half2 d, exact
    const uint32_t di = Vh - mh;         // integer d per 16-bit lane (each lane >= 0: no borrow)
    const uint32_t hR = hsub2u(Gh, Bh);
    const uint32_t hG = hfma2u(dh, 0x40004000u, hsub2u(Bh, Rh));  // 2 d + (B - R)
    const uint32_t hB = hfma2u(dh, 0x44004400u, hsub2u(Rh, Gh));  // 4 d + (R - G)
    const uint32_t eR = heq2m(Vh, Rh);
    const uint32_t eG = heq2m(Vh, Gh);
    const uint32_t hh = bitsel(eR, hR, bitsel(eG, hG, hB));
    // per-lane table products
    const float d0 = __low2float(as_h2(dh)), d1 = __high2float(as_h2(dh));
    const float h0 = __low2float(as_h2(hh)), h1 = __high2float(as_h2(hh));
    const uint32_t aS0 = __dp2a_lo(Vh, 0x00000080u, lut.cs), aS1 = __dp2a_lo(Vh, 0x00008000u, lut.cs);
    const uint32_t aH0 = __dp2a_lo(di, 0x00000080u, lut.ch), aH1 = __dp2a_lo(di, 0x00008000u, lut.ch);
    o.ys0 = __float_as_uint(fma_rz_(d0, lds(aS0), 32768.5f));
    o.ys1 = __float_as_uint(fma_rz_(d1, lds(aS1), 32768.5f));
    o.yh0 = __float_as_uint(fma_rm_(h0, lds(aH0), 49152.5f));
    o.yh1 = __float_as_uint(fma_rm_(h1, lds(aH1), 49152.5f));
    o.vh = Vh;
}

// packed "H += 180 where H < 0" on four H mod 256 bytes
__device__ __forceinline__ uint32_t fix_hue4(uint32_t hw) {
    uint32_t m;
    asm("lop3.b32 %0, %1, %2, 0x80808080, 0x80;" : "=r"(m) : "r"(hw), "r"(hw + hw));  // a & b & c
    return hw - (m >> 7) * 76u;
}

}  // namespace v7

__device__ __forceinline__ void hsv16_v7(const uint32_t (&w)[12], Px16& o, const LutView7& lut) {
    const uint32_t K = 0x64646464u;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const uint32_t wa = w[3 * g], wb = w[3 * g + 1], wc = w[3 * g + 2];
        // wa = B0 G0 R0 B1 | wb = G1 R1 B2 G2 | wc = R2 B3 G3 R3
        const uint32_t B01 = __byte_perm(wa, K, 0x4340);
        const uint32_t t01 = __byte_perm(wa, wb, 0x5421);  // G0 R0 G1 R1
        const uint32_t G01 = v7::even_bytes_magic(t01);
        const uint32_t R01 = __byte_perm(t01, K, 0x4341);
        const uint32_t R23 = __byte_perm(wc, K, 0x4340);
        const uint32_t t23 = __byte_perm(wb, wc, 0x6532);  // B2 G2 B3 G3
        const uint32_t B23 = v7::even_bytes_magic(t23);
        const uint32_t G23 = __byte_perm(t23, K, 0x4341);
        v7::PairOut7 p, q;
        v7::pair(B01, G01, R01, lut, p);
        v7::pair(B23, G23, R23, lut, q);
        const uint32_t hw = __byte_perm(__byte_perm(p.yh0, p.yh1, 0x0051), __byte_perm(q.yh0, q.yh1, 0x0051), 0x5410);
        o.h[g] = v7::fix_hue4(hw);
        o.s[g] = __byte_perm(__byte_perm(p.ys0, p.ys1, 0x0051), __byte_perm(q.ys0, q.ys1, 0x0051), 0x5410);
        o.v[g] = __byte_perm(p.vh, q.vh, 0x6420);
    }
}

}  // namespace psd
