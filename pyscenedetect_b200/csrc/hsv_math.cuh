// Per-pixel colour arithmetic shared by the fused score kernel and the test hook.
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
#pragma once

#include <stdint.h>

namespace psd {

struct Px16 {  // 16 pixels, planar, 4 pixels per 32-bit word (pixel 4j+i in byte i of word j)
    uint32_t h[4], s[4], v[4];
};

// ---- generic-path arithmetic: float-domain pipeline on pixel PAIRS ----
// (used by psd_score_kernel for strips the warp-specialised kernel cannot take: unaligned inputs, tails that
// are not a multiple of 16 pixels, frames smaller than a strip; the fast path is hsv_half2.cuh.)
// The table entries are regenerated with one MUFU.RCP each:
//   sdiv[V] = rint(1044480 / V):  q = 1044480 * rcp(V) has relative error <= 2^-23 * (1 + eps)
//   (rcp.approx.f32 is specified to 1 ulp), i.e. absolute error < 0.125 / V * 1.01, while the exact
//   quotient j/V is never closer than 1/(2V) to a rounding boundary k + 1/2 (1044480 = 2^12*255 has
//   no factor 2^13, so 2*1044480/V is never an odd integer).  Hence adding the 1.5*2^23 magic
//   constant inside the FMA rounds to exactly rint(1044480/V).  The same argument holds for
//   hdiv[d] = rint(122880 / d) (122880 = 2^13 * 15).
// Bytes are lifted to "magic" floats 2^23 + b by one PRMT each (mantissa ulp = 1, so integer
// add/sub/compare on them is exact and order-preserving).  The two fixed-point products use
// directed rounding so that only bits below the
// 4096 quantum are dropped before the >> 12:
//   S:  x = fma.rz(d, sdiv, 2048)  (x >= 0: truncation never crosses a multiple of 4096)
//       y = fma.rz(x, 2^-12, 2^23)            -> mantissa = floor(x / 4096) = S
//   H:  x = fma.rm(h, hdiv, 2048)  (h may be negative: round toward -inf == arithmetic shift)
//       y = fma.rm(x, 2^-12, 1.5 * 2^23)      -> mantissa = 2^22 + floor(x / 4096)
// |d * sdiv| < 2^28 and |h * hdiv| < 2^25, so the dropped bits are at most 2^4 resp. 2^1 wide and
// 4096 k is always representable: floor(x/4096) is unchanged.  Pinned by the exhaustive test.
// sm_90 has no packed FP32 instructions (f32x2 needs sm_100), so a pair is two scalar FP32 operations
// with the same rounding mode per lane: the results are the same bits.
struct f32x2_t {
    float lo, hi;
};

__device__ __forceinline__ f32x2_t pack2(float lo, float hi) { return {lo, hi}; }
__device__ __forceinline__ void unpack2(f32x2_t v, float& lo, float& hi) {
    lo = v.lo;
    hi = v.hi;
}
__device__ __forceinline__ f32x2_t add2(f32x2_t a, f32x2_t b) {
    return {__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)};
}
__device__ __forceinline__ f32x2_t sub2(f32x2_t a, f32x2_t b) {
    return {__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)};
}
__device__ __forceinline__ f32x2_t fma2_rn(f32x2_t a, f32x2_t b, f32x2_t c) {
    return {__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ f32x2_t fma2_rz(f32x2_t a, f32x2_t b, f32x2_t c) {
    return {__fmaf_rz(a.lo, b.lo, c.lo), __fmaf_rz(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ f32x2_t fma2_rm(f32x2_t a, f32x2_t b, f32x2_t c) {
    return {__fmaf_rd(a.lo, b.lo, c.lo), __fmaf_rd(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// byte j of word w -> float 2^23 + byte  (PRMT with the constant 0x4B000000 as second source)
template <int J>
__device__ __forceinline__ float magic_byte(uint32_t w) {
    return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440 | J));
}

struct PairOut {  // H, S, V of two pixels as magic-float bit patterns (value in the low byte)
    uint32_t h0, h1, s0, s1, v0, v1;
};

// bytes of pixels (P, P+1) inside the 12 packed words: pixel p occupies bytes 3p, 3p+1, 3p+2
template <int P>
__device__ __forceinline__ void hsv_pair_f32x2(const uint32_t (&w)[12], PairOut& o) {
    constexpr int kb0 = 3 * P, kb1 = 3 * P + 3;
    const float B0 = magic_byte<(kb0 + 0) & 3>(w[(kb0 + 0) >> 2]);
    const float G0 = magic_byte<(kb0 + 1) & 3>(w[(kb0 + 1) >> 2]);
    const float R0 = magic_byte<(kb0 + 2) & 3>(w[(kb0 + 2) >> 2]);
    const float B1 = magic_byte<(kb1 + 0) & 3>(w[(kb1 + 0) >> 2]);
    const float G1 = magic_byte<(kb1 + 1) & 3>(w[(kb1 + 1) >> 2]);
    const float R1 = magic_byte<(kb1 + 2) & 3>(w[(kb1 + 2) >> 2]);
    // max / min on the bit patterns (order-preserving for these positive floats)
    const uint32_t V0 = __vimax3_u32(__float_as_uint(B0), __float_as_uint(G0), __float_as_uint(R0));
    const uint32_t V1 = __vimax3_u32(__float_as_uint(B1), __float_as_uint(G1), __float_as_uint(R1));
    const uint32_t m0 = __vimin3_u32(__float_as_uint(B0), __float_as_uint(G0), __float_as_uint(R0));
    const uint32_t m1 = __vimin3_u32(__float_as_uint(B1), __float_as_uint(G1), __float_as_uint(R1));
    const f32x2_t Vm = pack2(__uint_as_float(V0), __uint_as_float(V1));
    const f32x2_t mn = pack2(__uint_as_float(m0), __uint_as_float(m1));
    const f32x2_t d2 = sub2(Vm, mn);  // plain floats 0..255 (exact)
    float d0, d1;
    unpack2(d2, d0, d1);
    // reciprocals of max(V,1), max(d,1): d == 0 whenever V == 0, and h == 0 whenever d == 0, so the
    // clamped entries are multiplied by zero exactly as the tables' zero entries would be
    const f32x2_t M23 = pack2(8388608.0f, 8388608.0f);
    const f32x2_t M15 = pack2(12582912.0f, 12582912.0f);
    const f32x2_t Vg = pack2(__uint_as_float(max(V0, 0x4B000001u)), __uint_as_float(max(V1, 0x4B000001u)));
    float Vp0, Vp1;
    unpack2(sub2(Vg, M23), Vp0, Vp1);
    const f32x2_t rV = pack2(rcp_approx(Vp0), rcp_approx(Vp1));
    const f32x2_t rd = pack2(rcp_approx(fmaxf(d0, 1.0f)), rcp_approx(fmaxf(d1, 1.0f)));
    const f32x2_t sdiv = sub2(fma2_rn(pack2(1044480.0f, 1044480.0f), rV, M15), M15);
    const f32x2_t hdiv = sub2(fma2_rn(pack2(122880.0f, 122880.0f), rd, M15), M15);
    const f32x2_t c2048 = pack2(2048.0f, 2048.0f);
    const f32x2_t cshift = pack2(0.000244140625f, 0.000244140625f);  // 2^-12
    const f32x2_t ys = fma2_rz(fma2_rz(d2, sdiv, c2048), cshift, M23);
    // hue numerators (differences of magic floats are exact small integers)
    const f32x2_t B2 = pack2(B0, B1), G2 = pack2(G0, G1), R2 = pack2(R0, R1);
    const f32x2_t hR = sub2(G2, B2);
    const f32x2_t hG = fma2_rn(d2, pack2(2.0f, 2.0f), sub2(B2, R2));
    const f32x2_t hB = fma2_rn(d2, pack2(4.0f, 4.0f), sub2(R2, G2));
    float hR0, hR1, hG0, hG1, hB0, hB1;
    unpack2(hR, hR0, hR1);
    unpack2(hG, hG0, hG1);
    unpack2(hB, hB0, hB1);
    const float h0 = (V0 == __float_as_uint(R0)) ? hR0 : ((V0 == __float_as_uint(G0)) ? hG0 : hB0);
    const float h1 = (V1 == __float_as_uint(R1)) ? hR1 : ((V1 == __float_as_uint(G1)) ? hG1 : hB1);
    float yh0, yh1;
    unpack2(fma2_rm(fma2_rm(pack2(h0, h1), hdiv, c2048), cshift, M15), yh0, yh1);
    if (yh0 < 12582912.0f) yh0 += 180.0f;
    if (yh1 < 12582912.0f) yh1 += 180.0f;
    float ys0, ys1;
    unpack2(ys, ys0, ys1);
    o.h0 = __float_as_uint(yh0); o.h1 = __float_as_uint(yh1);
    o.s0 = __float_as_uint(ys0); o.s1 = __float_as_uint(ys1);
    o.v0 = V0; o.v1 = V1;
}

// four magic words (value in the low byte) -> one planar word; the two IMADs run on the FMA pipe
__device__ __forceinline__ uint32_t pack4_low_bytes(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    const uint32_t lo = b * 256u + a;  // low 16 bits = [a.b0, b.b0] (a's upper bytes only reach bytes 2,3)
    const uint32_t hi = d * 256u + c;
    return __byte_perm(lo, hi, 0x5410);
}

__device__ __forceinline__ void hsv16_f32x2(const uint32_t (&w)[12], Px16& o) {
    PairOut p[8];
    hsv_pair_f32x2<0>(w, p[0]);
    hsv_pair_f32x2<2>(w, p[1]);
    hsv_pair_f32x2<4>(w, p[2]);
    hsv_pair_f32x2<6>(w, p[3]);
    hsv_pair_f32x2<8>(w, p[4]);
    hsv_pair_f32x2<10>(w, p[5]);
    hsv_pair_f32x2<12>(w, p[6]);
    hsv_pair_f32x2<14>(w, p[7]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        o.h[j] = pack4_low_bytes(p[2 * j].h0, p[2 * j].h1, p[2 * j + 1].h0, p[2 * j + 1].h1);
        o.s[j] = pack4_low_bytes(p[2 * j].s0, p[2 * j].s1, p[2 * j + 1].s0, p[2 * j + 1].s1);
        o.v[j] = pack4_low_bytes(p[2 * j].v0, p[2 * j].v1, p[2 * j + 1].v0, p[2 * j + 1].v1);
    }
}

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

}  // namespace psd
