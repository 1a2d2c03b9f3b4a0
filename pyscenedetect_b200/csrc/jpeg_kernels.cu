// psd_jpeg_encode: baseline JPEG files of a batch of BGR images, the bytes cv2.imencode(".jpg", img,
// [IMWRITE_JPEG_QUALITY, q]) writes (libjpeg-turbo: jpeg_set_quality with force_baseline, 4:2:0, the T.81 Annex K
// Huffman tables, no optimisation, no restart interval), for scenedetect/output/image.py:317-319.
//
// Every step is the library's integer arithmetic (tests/jpeg_twin.py restates each one), so the files are equal
// byte for byte.  Per sub-batch of images, on one stream:
//   jpeg_block_kernel   one CTA per tile of 32 MCUs of one image, one warp per block position of the MCU (Y00 Y01
//                       Y10 Y11 Cb Cr): reads its samples through the psd_frame_layout, jccolor.c YCbCr, edge
//                       replication and h2v2 downsampling (jcprepct.c / jcsample.c), jfdctint.c islow, jcdctmgr.c
//                       reciprocal quantisation, zigzag; writes the int16 coefficients and the block's Huffman bit
//                       length as an offset inside its tile, and the tile's total
//   psd_clip_scan_kernel   tile totals -> bit offsets (each image's stream has its own region of the largest size it
//                       can take, so every stream starts on 16 bytes)
//   jpeg_emit_kernel    every block ORs its codes into its image's bit stream, 32 bits at a time; the image's last
//                       block pads the last byte with 1-bits (jchuff.c flush_bits)
//   jpeg_ff_kernel      0xFF bytes per 8 KiB chunk of every stream, psd_clip_scan_kernel -> offsets
//   jpeg_size_kernel    each file's size, psd_clip_scan_kernel -> file offsets
//   jpeg_copy_kernel    the header (SOI, APP0, DQT, SOF0, DHT, SOS), the stream with 0x00 after every 0xFF, EOI
#include <string.h>

#include <vector>

#include "psd_common.cuh"

namespace psd {


constexpr int kTileMcus = 32;                 // MCUs per tile of the block and emit passes
constexpr int kTileBlocks = 6 * kTileMcus;    // = threads of a block-pass CTA
constexpr int kMaxBlockBits = 22 + 63 * 26;   // DC: 11-bit code + 11 bits; AC: 16-bit code + 10 bits each
constexpr int kBlockWords = (kMaxBlockBits + 31) / 32;
constexpr int kChunkBytes = 8192;             // raw stream bytes per CTA of the stuffing passes
constexpr int kChunkThreads = 256;
constexpr int kHeaderBytes = 623;
constexpr int kSofOffset = 2 + 18 + 2 * 69;   // the SOF0 segment: height at +5, width at +7

// ITU T.81 Annex K.3 (bits per code length, symbols): DC luma, AC luma, DC chroma, AC chroma
constexpr uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D};
constexpr uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
    0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72,
    0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37,
    0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
    0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3,
    0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
    0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA};
constexpr uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
constexpr uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
    0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1,
    0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36,
    0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
    0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A,
    0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A,
    0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA,
    0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
    0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA};
// Annex K.1 / K.2 quantisation tables, natural order
constexpr uint8_t kStdQuant[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
     47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
constexpr uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// zigzag index -> natural index, as a constant expression in unrolled device loops
__host__ __device__ constexpr int zigzag(int z) {
    constexpr uint8_t t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                               12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                               58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return t[z];
}

// Huffman code of every symbol (T.81 Annex C): code << 8 | length, 0 for symbols the table lacks
struct HuffTable {
    uint32_t c[256];
};
constexpr HuffTable make_huff(const uint8_t (&bits)[16], const uint8_t* vals) {
    HuffTable t{};
    uint32_t code = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int i = 0; i < bits[len - 1]; ++i) t.c[vals[k++]] = (code++ << 8) | (uint32_t)len;
        code <<= 1;
    }
    return t;
}
// [0] DC luma, [1] AC luma, [2] DC chroma, [3] AC chroma
__constant__ HuffTable kHuff[4] = {make_huff(kDcLumaBits, kDcVals), make_huff(kAcLumaBits, kAcLumaVals),
                                   make_huff(kDcChromaBits, kDcVals), make_huff(kAcChromaBits, kAcChromaVals)};

// jcdctmgr.c compute_reciprocal of every divisor 8 * quantval (16-bit DCTELEM): |x| -> ((|x| + corr) * recip) >> shift
struct Quant {
    uint16_t recip[2][64];
    uint16_t corr[2][64];
    uint8_t shift[2][64];
};

struct Image {            // one image of a sub-batch
    const uint8_t* base;  // channel B of pixel (0, 0)
    int64_t row_stride, pixel_stride, channel_stride;
    int32_t width, height;
    int32_t mcus_x, n_mcu;   // MCUs per row, MCUs
    int32_t wib, hib;        // luma blocks per row and per column: ceil(width / 8), ceil(height / 8)
    int64_t tile0, n_tiles;  // its tiles in the sub-batch
    int64_t raw0;            // the first word of its stream in Batch::raw (a multiple of 4)
    int64_t chunk0, n_chunks;// its stuffing chunks (enough for the largest stream it can have)
};

struct Batch {
    const Image* images;
    const int32_t* tile_image;   // [n_tiles]
    const int32_t* chunk_image;  // [n_chunks]
    int32_t n_images;
    int16_t* coefs;        // [n_tiles * kTileBlocks][64] zigzag order; block b of a tile = warp b / 32, lane b % 32
    int32_t* block_off;    // [n_tiles * kTileBlocks] bit offset inside the tile
    int64_t* tile_bits;    // [n_tiles + 1] tile lengths, then their offsets
    uint32_t* raw;         // bit streams, byte order in memory
    int64_t* chunk_ff;     // [n_chunks + 1] 0xFF counts, then offsets
    int64_t* sizes;        // [n_images + 1] file sizes, then offsets inside the sub-batch
    const uint8_t* header; // [kHeaderBytes] with height and width 0
};

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// Component sample (i, j) of block position k (0-3 luma Y00 Y01 Y10 Y11, 4 Cb, 5 Cr) of MCU (mx, my), with the
// edge replication libjpeg applies.  Luma: rows and columns clamped to the image.  Chroma: the downsampled row index
// clamped to ceil(h / 2) - 1 (jcprepct.c repeats the last downsampled row), then h2v2 over full-resolution rows and
// columns clamped to the image, bias 1, 2 alternating along the row (jcsample.c).  A luma block outside the
// component (a dummy block) reads its source block: see source_block.
__device__ __forceinline__ int rgb_y(int b, int g, int r) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int rgb_c(int b, int g, int r, int k) {
    return k == 4 ? (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16
                  : (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}
__device__ __forceinline__ void pixel(const Image& im, int x, int y, int& b, int& g, int& r) {
    const uint8_t* p = im.base + (int64_t)y * im.row_stride + (int64_t)x * im.pixel_stride;
    b = p[0];
    g = p[im.channel_stride];
    r = p[2 * im.channel_stride];
}

// jccoefct.c: a luma block right of the component takes the DC of its left neighbour, one below it the DC of the
// MCU's Y01 (itself Y00's when Y01 is right of the component): the block whose pixels give that DC.  Real blocks are
// their own source.
__device__ __forceinline__ void source_block(const Image& im, int k, int mx, int my, int& bx, int& by) {
    const int r = k >> 1, c = k & 1;
    if (2 * my + r < im.hib) {
        by = 2 * my + r;
        bx = min(2 * mx + c, im.wib - 1);
    } else {
        by = 2 * my;
        bx = min(2 * mx + 1, im.wib - 1);
    }
}

__device__ __forceinline__ int luma_sample(const Image& im, int bx, int by, int i, int j) {
    int b, g, r;
    pixel(im, min(8 * bx + j, im.width - 1), min(8 * by + i, im.height - 1), b, g, r);
    return rgb_y(b, g, r);
}
__device__ __forceinline__ int chroma_sample(const Image& im, int k, int mx, int my, int i, int j) {
    const int cy = min(8 * my + i, (im.height + 1) / 2 - 1), cx = 8 * mx + j;
    const int y0 = min(2 * cy, im.height - 1), y1 = min(2 * cy + 1, im.height - 1);
    const int x0 = min(2 * cx, im.width - 1), x1 = min(2 * cx + 1, im.width - 1);
    int b, g, r, s;
    pixel(im, x0, y0, b, g, r);
    s = rgb_c(b, g, r, k);
    pixel(im, x1, y0, b, g, r);
    s += rgb_c(b, g, r, k);
    pixel(im, x0, y1, b, g, r);
    s += rgb_c(b, g, r, k);
    pixel(im, x1, y1, b, g, r);
    s += rgb_c(b, g, r, k);
    return (s + 1 + (j & 1)) >> 2;
}

__device__ __forceinline__ int quantize(int v, const Quant& q, int t, int i) {
    const uint32_t a = (uint32_t)(v < 0 ? -v : v);
    const int m = (int)(((a + q.corr[t][i]) * (uint32_t)q.recip[t][i]) >> q.shift[t][i]);
    return v < 0 ? -m : m;
}

// The quantised DC of block position k of MCU m (a dummy block's included): islow's DC is the sum of the 64
// centred samples
__device__ int block_dc(const Image& im, int k, int m, const Quant& q) {
    const int mx = m % im.mcus_x, my = m / im.mcus_x;
    int s = 0;
    if (k < 4) {
        int bx, by;
        source_block(im, k, mx, my, bx, by);
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 8; ++j) s += luma_sample(im, bx, by, i, j);
    } else {
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 8; ++j) s += chroma_sample(im, k, mx, my, i, j);
    }
    return quantize(s - 64 * 128, q, k < 4 ? 0 : 1, 0);
}

// jfdctint.c jpeg_fdct_islow on one row (STRIDE 1) or column (STRIDE 8) of d
template <int STRIDE, bool COLUMN>
__device__ __forceinline__ void fdct_1d(int* d) {
    constexpr int kPass1 = 2, kConst = 13;
    constexpr int n = COLUMN ? kConst + kPass1 : kConst - kPass1;
    auto descale = [](int x, int s) { return (x + (1 << (s - 1))) >> s; };
    const int tmp0 = d[0] + d[7 * STRIDE], tmp7 = d[0] - d[7 * STRIDE];
    const int tmp1 = d[STRIDE] + d[6 * STRIDE], tmp6 = d[STRIDE] - d[6 * STRIDE];
    const int tmp2 = d[2 * STRIDE] + d[5 * STRIDE], tmp5 = d[2 * STRIDE] - d[5 * STRIDE];
    const int tmp3 = d[3 * STRIDE] + d[4 * STRIDE], tmp4 = d[3 * STRIDE] - d[4 * STRIDE];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    if (COLUMN) {
        d[0] = descale(tmp10 + tmp11, kPass1);
        d[4 * STRIDE] = descale(tmp10 - tmp11, kPass1);
    } else {
        d[0] = (tmp10 + tmp11) * (1 << kPass1);
        d[4 * STRIDE] = (tmp10 - tmp11) * (1 << kPass1);
    }
    int z1 = (tmp12 + tmp13) * 4433;
    d[2 * STRIDE] = descale(z1 + tmp13 * 6270, n);
    d[6 * STRIDE] = descale(z1 - tmp12 * 15137, n);
    z1 = tmp4 + tmp7;
    int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int z5 = (z3 + z4) * 9633;
    const int t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
    z1 *= -7373;
    z2 *= -20995;
    z3 = z3 * -16069 + z5;
    z4 = z4 * -3196 + z5;
    d[7 * STRIDE] = descale(t4 + z1 + z3, n);
    d[5 * STRIDE] = descale(t5 + z2 + z4, n);
    d[3 * STRIDE] = descale(t6 + z2 + z3, n);
    d[STRIDE] = descale(t7 + z1 + z4, n);
}

// Walks one block's codes in stream order (jchuff.c encode_one_block): put(code, length) for the DC difference,
// then the ACs (a ZRL per 16 zeros ahead of a coefficient), then EOB unless coefficient 63 is nonzero.  c is the
// block's zigzag coefficients, nz the mask of its nonzero ACs (bit z for coefficient z).
template <class Put>
__device__ __forceinline__ void walk(const int16_t* c, uint64_t nz, int dc_diff, const uint32_t* dc_tab,
                                     const uint32_t* ac_tab, Put put) {
    int s = nbits(dc_diff);
    uint32_t e = dc_tab[s];
    put(e >> 8, e & 255);
    if (s) put((uint32_t)(dc_diff < 0 ? dc_diff - 1 : dc_diff) & ((1u << s) - 1), s);
    int last = 0;
    while (nz) {
        const int z = __ffsll((long long)nz) - 1;
        nz &= nz - 1;
        int run = z - last - 1;
        last = z;
        for (; run > 15; run -= 16) {
            e = ac_tab[0xF0];
            put(e >> 8, e & 255);
        }
        const int v = c[z];
        s = nbits(v);
        e = ac_tab[(run << 4) | s];
        put(e >> 8, e & 255);
        put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1), s);
    }
    if (last != 63) {
        e = ac_tab[0];
        put(e >> 8, e & 255);
    }
}

__device__ __forceinline__ void load_tables(uint32_t (*tab)[256]) {
    for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) tab[i >> 8][i & 255] = kHuff[i >> 8].c[i & 255];
}

// A block's place: tile t, position k (= warp), MCU lane; its image; -1 when the tile's MCU does not exist
struct BlockAt {
    int img, k, lane, m;  // m: MCU index in the image
    int64_t g;            // block index in the sub-batch
};
__device__ __forceinline__ BlockAt block_at(const Batch& bt, int64_t tile) {
    BlockAt a;
    a.img = bt.tile_image[tile];
    a.k = threadIdx.x >> 5;
    a.lane = threadIdx.x & 31;
    const int64_t m = (tile - bt.images[a.img].tile0) * kTileMcus + a.lane;
    a.m = m < bt.images[a.img].n_mcu ? (int)m : -1;
    a.g = tile * kTileBlocks + threadIdx.x;
    return a;
}

// Exclusive scan of v over the 192 threads of a tile CTA in stream order (MCU by MCU: Y00 Y01 Y10 Y11 Cb Cr), where
// thread (warp k, lane l) holds block k of MCU l; *total receives the sum
__device__ __forceinline__ int64_t tile_scan(int64_t v, int64_t* sh, int64_t* total) {
    __shared__ int64_t warp_sum[6];
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    sh[lane * 6 + k] = v;
    __syncthreads();
    const int64_t x = sh[threadIdx.x];  // stream position threadIdx.x
    int64_t s = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += y;
    }
    if (lane == 31) warp_sum[k] = s;
    __syncthreads();
    int64_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < 6; ++w) {
        before += w < k ? warp_sum[w] : 0;
        all += warp_sum[w];
    }
    sh[threadIdx.x] = before + s - x;
    __syncthreads();
    const int64_t r = sh[lane * 6 + k];
    *total = all;
    return r;
}

// nonzero mask of the ACs of a block's 64 zigzag coefficients
__device__ __forceinline__ uint64_t ac_mask(const int16_t* c) {
    uint64_t nz = 0;
    const uint4* c4 = reinterpret_cast<const uint4*>(c);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint4 v = c4[i];
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int h = 0; h < 8; ++h)
            if ((w[h >> 1] >> (16 * (h & 1))) & 0xFFFFu) nz |= 1ull << (8 * i + h);
    }
    return nz & ~1ull;
}

__global__ void __launch_bounds__(kTileBlocks) jpeg_block_kernel(Batch bt, Quant q) {
    __shared__ uint32_t tab[4][256];
    __shared__ int dc[6][kTileMcus];
    __shared__ int64_t scan[kTileBlocks];
    load_tables(tab);
    const int64_t tile = blockIdx.x;
    const BlockAt a = block_at(bt, tile);
    const Image& im = bt.images[a.img];
    const int t = a.k < 4 ? 0 : 1;
    int16_t* out = bt.coefs + a.g * 64;
    if (a.m >= 0) {
        const int mx = a.m % im.mcus_x, my = a.m / im.mcus_x;
        int d[64];
        bool dummy = false;
        if (a.k < 4) {
            int bx, by;
            source_block(im, a.k, mx, my, bx, by);
            dummy = 2 * mx + (a.k & 1) >= im.wib || 2 * my + (a.k >> 1) >= im.hib;
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) d[8 * i + j] = luma_sample(im, bx, by, i, j) - 128;
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) d[8 * i + j] = chroma_sample(im, a.k, mx, my, i, j) - 128;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) fdct_1d<1, false>(d + 8 * i);
#pragma unroll
        for (int j = 0; j < 8; ++j) fdct_1d<8, true>(d + j);
        uint32_t w[32];
#pragma unroll
        for (int z = 0; z < 64; ++z) {
            const int v = (z == 0 || !dummy) ? quantize(d[zigzag(z)], q, t, zigzag(z)) : 0;
            if (z & 1) w[z >> 1] |= (uint32_t)(uint16_t)v << 16;
            else w[z >> 1] = (uint16_t)v;
        }
        uint4* o4 = reinterpret_cast<uint4*>(out);
#pragma unroll
        for (int i = 0; i < 8; ++i) o4[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
        dc[a.k][a.lane] = (int16_t)(w[0] & 0xFFFFu);
    }
    __syncthreads();
    int bits = 0;
    if (a.m >= 0) {
        // the DC predecessor: the previous luma block of the scan (Y11 of the previous MCU for Y00), the previous MCU's
        // block for chroma; 0 at the start of the image.  Lane 0 recomputes the previous tile's.
        int pred = 0;
        if (a.k >= 1 && a.k <= 3) pred = dc[a.k - 1][a.lane];
        else if (a.lane > 0) pred = dc[a.k == 0 ? 3 : a.k][a.lane - 1];
        else if (a.m > 0) pred = block_dc(im, a.k == 0 ? 3 : a.k, a.m - 1, q);
        walk(out, ac_mask(out), dc[a.k][a.lane] - pred, tab[2 * t], tab[2 * t + 1],
             [&](uint32_t, int len) { bits += len; });
    }
    int64_t total;
    bt.block_off[a.g] = (int32_t)tile_scan(bits, scan, &total);
    if (threadIdx.x == 0) bt.tile_bits[tile] = total;
}

// Where image i's stream lies: its first word in bt.raw and its length in bits (tile_bits holds offsets)
__device__ __forceinline__ void stream_of(const Batch& bt, int i, int64_t& word0, int64_t& nbits_) {
    const Image& im = bt.images[i];
    word0 = im.raw0;
    nbits_ = bt.tile_bits[im.tile0 + im.n_tiles] - bt.tile_bits[im.tile0];
}

// Appends codes MSB first to a 64-bit buffer and ORs each full 32-bit word into the stream
struct BitWriter {
    uint32_t* word;
    uint64_t buf;
    int n;
    __device__ __forceinline__ void put(uint32_t code, int len) {
        if (!len) return;
        buf |= (uint64_t)code << (64 - n - len);
        n += len;
        if (n >= 32) {
            atomicOr(word++, __byte_perm((uint32_t)(buf >> 32), 0, 0x0123));
            buf <<= 32;
            n -= 32;
        }
    }
    __device__ __forceinline__ void flush() {
        if (n > 0) atomicOr(word, __byte_perm((uint32_t)(buf >> 32), 0, 0x0123));
    }
};

__global__ void __launch_bounds__(kTileBlocks) jpeg_emit_kernel(Batch bt) {
    __shared__ uint32_t tab[4][256];
    load_tables(tab);
    __syncthreads();
    const int64_t tile = blockIdx.x;
    const BlockAt a = block_at(bt, tile);
    if (a.m < 0) return;
    const Image& im = bt.images[a.img];
    const int t = a.k < 4 ? 0 : 1;
    const int16_t* c = bt.coefs + a.g * 64;
    int pred = 0;
    if (a.k >= 1 && a.k <= 3) pred = bt.coefs[(a.g - 32) * 64];
    else if (a.lane > 0) pred = bt.coefs[(a.g - (a.k == 0 ? -3 * 32 : 0) - 1) * 64];
    else if (a.m > 0) pred = bt.coefs[((tile - 1) * kTileBlocks + (a.k == 0 ? 3 : a.k) * 32 + 31) * 64];
    int64_t word0, len;
    stream_of(bt, a.img, word0, len);
    const int64_t pos = bt.tile_bits[tile] - bt.tile_bits[im.tile0] + bt.block_off[a.g];
    BitWriter w{bt.raw + word0 + (pos >> 5), 0, (int)(pos & 31)};
    walk(c, ac_mask(c), c[0] - pred, tab[2 * t], tab[2 * t + 1], [&](uint32_t code, int n) { w.put(code, n); });
    if (a.m == im.n_mcu - 1 && a.k == 5) {  // the image's last block: 1-bits up to the byte (jchuff.c flush_bits)
        const int pad = (int)((8 - (len & 7)) & 7);
        w.put((1u << pad) - 1, pad);
    }
    w.flush();
}

// 0xFF bytes of each thread's 32 bytes of a chunk; chunks past the stream count nothing
__device__ __forceinline__ int chunk_ff_count(const Batch& bt, int i, int64_t chunk, int64_t& byte0, int64_t& nbytes,
                                              uint4 v[2]) {
    int64_t word0, len;
    stream_of(bt, i, word0, len);
    nbytes = (len + 7) >> 3;
    byte0 = (chunk - bt.images[i].chunk0) * kChunkBytes + 32 * (int64_t)threadIdx.x;
    int n = 0;
    if (byte0 < nbytes) {
        const uint4* p = reinterpret_cast<const uint4*>(bt.raw + word0) + (byte0 >> 4);
        v[0] = p[0];
        v[1] = p[1];
        const uint32_t w[8] = {v[0].x, v[0].y, v[0].z, v[0].w, v[1].x, v[1].y, v[1].z, v[1].w};
#pragma unroll
        for (int b = 0; b < 32; ++b)
            n += (byte0 + b < nbytes) && ((w[b >> 2] >> (8 * (b & 3))) & 255u) == 255u;
    }
    return n;
}

__device__ __forceinline__ int block_sum(int v, int* total) {
    __shared__ int ws[kChunkThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += y;
    }
    if (lane == 31) ws[w] = s;
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < kChunkThreads / 32; ++k) {
        before += k < w ? ws[k] : 0;
        all += ws[k];
    }
    *total = all;
    return before + s - v;
}

__global__ void __launch_bounds__(kChunkThreads) jpeg_ff_kernel(Batch bt) {
    const int64_t chunk = blockIdx.x;
    const int i = bt.chunk_image[chunk];
    int64_t byte0, nbytes;
    uint4 v[2];
    int total;
    block_sum(chunk_ff_count(bt, i, chunk, byte0, nbytes, v), &total);
    if (threadIdx.x == 0) bt.chunk_ff[chunk] = total;
}

// each file's size: header, stream, its stuffed zeros, EOI
__global__ void __launch_bounds__(128) jpeg_size_kernel(Batch bt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= bt.n_images) return;
    const Image& im = bt.images[i];
    int64_t word0, len;
    stream_of(bt, i, word0, len);
    const int64_t ff = bt.chunk_ff[im.chunk0 + im.n_chunks] - bt.chunk_ff[im.chunk0];
    bt.sizes[i] = kHeaderBytes + ((len + 7) >> 3) + ff + 2;
}

// the files of the sub-batch at out + image_bytes[first] + sizes[i]; image_bytes[first + i + 1] = its end.  A file
// that would end past out_cap is not written.
__global__ void __launch_bounds__(kChunkThreads) jpeg_copy_kernel(Batch bt, uint8_t* __restrict__ out, int64_t out_cap,
                                                                  int64_t* __restrict__ image_bytes) {
    const int64_t chunk = blockIdx.x;
    const int i = bt.chunk_image[chunk];
    const Image& im = bt.images[i];
    const int64_t start = image_bytes[0] + bt.sizes[i], end = image_bytes[0] + bt.sizes[i + 1];
    int64_t byte0, nbytes;
    uint4 v[2];
    int total;
    const int n = chunk_ff_count(bt, i, chunk, byte0, nbytes, v);
    const int before = block_sum(n, &total);
    if (chunk == im.chunk0 && threadIdx.x == 0) image_bytes[i + 1] = end;
    if (end > out_cap) return;
    uint8_t* f = out + start;
    if (chunk == im.chunk0) {
        for (int b = threadIdx.x; b < kHeaderBytes; b += blockDim.x) {
            uint8_t x = bt.header[b];
            if (b == kSofOffset + 5) x = (uint8_t)(im.height >> 8);
            if (b == kSofOffset + 6) x = (uint8_t)im.height;
            if (b == kSofOffset + 7) x = (uint8_t)(im.width >> 8);
            if (b == kSofOffset + 8) x = (uint8_t)im.width;
            f[b] = x;
        }
        if (threadIdx.x == 0) {
            f[end - start - 2] = 0xFF;
            f[end - start - 1] = 0xD9;
        }
    }
    if (byte0 >= nbytes) return;
    uint8_t* o = f + kHeaderBytes + byte0 + (bt.chunk_ff[chunk] - bt.chunk_ff[im.chunk0]) + before;
    const uint32_t w[8] = {v[0].x, v[0].y, v[0].z, v[0].w, v[1].x, v[1].y, v[1].z, v[1].w};
#pragma unroll
    for (int b = 0; b < 32; ++b) {
        if (byte0 + b >= nbytes) break;
        const uint8_t x = (uint8_t)(w[b >> 2] >> (8 * (b & 3)));
        *o++ = x;
        if (x == 0xFF) *o++ = 0;
    }
}

// jpeg_set_quality(quality, force_baseline = TRUE) after cv2's clamp to [0, 100] (jcparam.c), table t, natural order
int quant_value(int quality, int t, int i) {
    int q = quality < 1 ? 1 : quality > 100 ? 100 : quality;
    const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    const int v = (kStdQuant[t][i] * scale + 50) / 100;
    return v < 1 ? 1 : v > 255 ? 255 : v;
}

Quant make_quant(int quality) {
    Quant q{};
    for (int t = 0; t < 2; ++t)
        for (int i = 0; i < 64; ++i) {
            const uint32_t d = 8u * (uint32_t)quant_value(quality, t, i);  // islow output is scaled by 8
            int b = 31 - __builtin_clz(d), r = 16 + b;
            uint32_t fq = (1u << r) / d, fr = (1u << r) % d, c = d / 2;
            if (fr == 0) {  // a power of two: fq would need 17 bits
                fq >>= 1;
                --r;
            } else if (fr <= d / 2) {
                ++c;
            } else {
                ++fq;
            }
            q.recip[t][i] = (uint16_t)fq;
            q.corr[t][i] = (uint16_t)c;
            q.shift[t][i] = (uint8_t)r;
        }
    return q;
}

// SOI, APP0 (JFIF 1.01, no density, no thumbnail), DQT 0 and 1, SOF0 (8-bit, 3 components, 4:2:0), DHT DC0 AC0 DC1
// AC1, SOS: jcmarker.c's headers as cv2 writes them, with height and width 0 (the copy pass fills them in)
std::vector<uint8_t> make_header(int quality) {
    std::vector<uint8_t> h = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00,
                              0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
    for (int t = 0; t < 2; ++t) {
        h.insert(h.end(), {0xFF, 0xDB, 0x00, 0x43, (uint8_t)t});
        for (int z = 0; z < 64; ++z) h.push_back((uint8_t)quant_value(quality, t, kZigzag[z]));
    }
    h.insert(h.end(), {0xFF, 0xC0, 0x00, 0x11, 8, 0, 0, 0, 0, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
    const struct { uint8_t id; const uint8_t* bits; const uint8_t* vals; int n; } dht[4] = {
        {0x00, kDcLumaBits, kDcVals, 12}, {0x10, kAcLumaBits, kAcLumaVals, 162},
        {0x01, kDcChromaBits, kDcVals, 12}, {0x11, kAcChromaBits, kAcChromaVals, 162}};
    for (const auto& d : dht) {
        const int len = 2 + 1 + 16 + d.n;
        h.insert(h.end(), {0xFF, 0xC4, (uint8_t)(len >> 8), (uint8_t)len, d.id});
        h.insert(h.end(), d.bits, d.bits + 16);
        h.insert(h.end(), d.vals, d.vals + d.n);
    }
    h.insert(h.end(), {0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
    return h;
}

// the sub-batch arrays: device workspace of one sub-batch at a time
struct Sizes {
    int64_t tiles = 0, chunks = 0, raw_words = 0;
    int64_t images = 0;
    int64_t bytes() const {
        return tiles * kTileBlocks * (64 * 2 + 4) + raw_words * 4 + (tiles + 1) * (8 + 4) + (chunks + 1) * (8 + 4) +
               images * (sizeof(Image) + 8) + 8 + kHeaderBytes + 64 * 8;
    }
};


}  // namespace psd

using namespace psd;

extern "C" int psd_jpeg_encode(int device, const psd_jpeg_image* images, int32_t n, int32_t quality,
                               int64_t workspace_cap, uint8_t* out, int64_t out_cap, int64_t* image_bytes,
                               void* stream) {
    PSD_REQUIRE(n >= 0 && out_cap >= 0 && workspace_cap >= 0, "psd_jpeg_encode: bad image count, out_cap or "
                "workspace_cap");
    PSD_REQUIRE(image_bytes, "psd_jpeg_encode: no image_bytes");
    PSD_REQUIRE(n == 0 || images, "psd_jpeg_encode: no images");
    PSD_REQUIRE(out || out_cap == 0, "psd_jpeg_encode: no output buffer");
    PSD_CUDA(cudaSetDevice(device));
    cudaStream_t s = (cudaStream_t)stream;
    int rc = require_device_memory(image_bytes, device, "psd_jpeg_encode image_bytes");
    if (rc) return rc;
    if (out_cap > 0 && (rc = require_device_memory(out, device, "psd_jpeg_encode out"))) return rc;
    // every image: its descriptor (tile0 / chunk0 relative to its sub-batch, set below) and its workspace
    std::vector<Image> im((size_t)n);
    for (int32_t i = 0; i < n; ++i) {
        const psd_jpeg_image& x = images[i];
        PSD_REQUIRE(x.width >= 1 && x.height >= 1 && x.width <= 65535 && x.height <= 65535,
                    "psd_jpeg_encode: image %d is %d x %d (1 to 65535 pixels each way)", i, x.width, x.height);
        PSD_REQUIRE(x.base, "psd_jpeg_encode: image %d has no pixels", i);
        char what[64];
        snprintf(what, sizeof(what), "psd_jpeg_encode image %d", i);
        if ((rc = require_device_memory(x.base, device, what))) return rc;
        Image& m = im[i];
        m.base = (const uint8_t*)x.base;
        m.row_stride = x.layout.row_stride;
        m.pixel_stride = x.layout.pixel_stride;
        m.channel_stride = x.layout.channel_stride;
        m.width = x.width;
        m.height = x.height;
        m.mcus_x = (x.width + 15) / 16;
        m.n_mcu = m.mcus_x * ((x.height + 15) / 16);
        m.wib = (x.width + 7) / 8;
        m.hib = (x.height + 7) / 8;
        m.n_tiles = (m.n_mcu + kTileMcus - 1) / kTileMcus;
        m.n_chunks = (m.n_tiles * kTileBlocks * kBlockWords * 4 + kChunkBytes - 1) / kChunkBytes;
    }
    PSD_CUDA(cudaMemsetAsync(image_bytes, 0, sizeof(int64_t), s));
    if (n == 0) return PSD_OK;
    const int64_t cap = workspace_cap ? workspace_cap : (int64_t)512 << 20;
    // sub-batches: as many images as the workspace cap holds, at least one
    std::vector<int32_t> first = {0};
    Sizes big, cur;
    for (int32_t i = 0; i < n; ++i) {
        Sizes nx = cur;
        nx.tiles += im[i].n_tiles;
        nx.chunks += im[i].n_chunks;
        nx.raw_words += im[i].n_tiles * kTileBlocks * kBlockWords;
        nx.images += 1;
        if (cur.images > 0 && nx.bytes() > cap) {
            first.push_back(i);
            nx = Sizes{};
            nx.tiles = im[i].n_tiles;
            nx.chunks = im[i].n_chunks;
            nx.raw_words = im[i].n_tiles * kTileBlocks * kBlockWords;
            nx.images = 1;
        }
        cur = nx;
        big.tiles = std::max(big.tiles, cur.tiles);
        big.chunks = std::max(big.chunks, cur.chunks);
        big.raw_words = std::max(big.raw_words, cur.raw_words);
        big.images = std::max(big.images, cur.images);
    }
    first.push_back(n);
    // one workspace for the largest sub-batch
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
    bt.coefs = (int16_t*)take((size_t)big.tiles * kTileBlocks * 128);
    bt.raw = (uint32_t*)take((size_t)big.raw_words * 4);
    bt.block_off = (int32_t*)take((size_t)big.tiles * kTileBlocks * 4);
    bt.tile_bits = (int64_t*)take((size_t)(big.tiles + 1) * 8);
    bt.chunk_ff = (int64_t*)take((size_t)(big.chunks + 1) * 8);
    bt.sizes = (int64_t*)take((size_t)(big.images + 1) * 8);
    Image* d_images = (Image*)take((size_t)big.images * sizeof(Image));
    int32_t* d_tile_image = (int32_t*)take((size_t)big.tiles * 4);
    int32_t* d_chunk_image = (int32_t*)take((size_t)big.chunks * 4);
    uint8_t* d_header = take(kHeaderBytes);
    bt.images = d_images;
    bt.tile_image = d_tile_image;
    bt.chunk_image = d_chunk_image;
    bt.header = d_header;
    const std::vector<uint8_t> header = make_header(quality);
    PSD_CUDA(cudaMemcpyAsync(d_header, header.data(), kHeaderBytes, cudaMemcpyHostToDevice, s));  // pageable: staged
    const Quant q = make_quant(quality);
    std::vector<int32_t> tile_image, chunk_image;
    for (size_t b = 0; b + 1 < first.size(); ++b) {
        const int32_t i0 = first[b], nb = first[b + 1] - first[b];
        tile_image.clear();
        chunk_image.clear();
        int64_t raw_words = 0;
        for (int32_t j = 0; j < nb; ++j) {
            Image& m = im[i0 + j];
            m.tile0 = (int64_t)tile_image.size();
            m.chunk0 = (int64_t)chunk_image.size();
            m.raw0 = raw_words;
            tile_image.insert(tile_image.end(), (size_t)m.n_tiles, j);
            chunk_image.insert(chunk_image.end(), (size_t)m.n_chunks, j);
            raw_words += m.n_tiles * kTileBlocks * kBlockWords;
        }
        const int64_t n_tiles = (int64_t)tile_image.size(), n_chunks = (int64_t)chunk_image.size();
        PSD_CUDA(cudaMemcpyAsync(d_images, &im[i0], sizeof(Image) * nb, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_tile_image, tile_image.data(), 4 * n_tiles, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemcpyAsync(d_chunk_image, chunk_image.data(), 4 * n_chunks, cudaMemcpyHostToDevice, s));
        PSD_CUDA(cudaMemsetAsync(bt.raw, 0, (size_t)raw_words * 4, s));
        bt.n_images = nb;
        jpeg_block_kernel<<<(unsigned)n_tiles, kTileBlocks, 0, s>>>(bt, q);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(bt.tile_bits, n_tiles);
        PSD_CHECK_LAUNCH();
        jpeg_emit_kernel<<<(unsigned)n_tiles, kTileBlocks, 0, s>>>(bt);
        PSD_CHECK_LAUNCH();
        jpeg_ff_kernel<<<(unsigned)n_chunks, kChunkThreads, 0, s>>>(bt);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(bt.chunk_ff, n_chunks);
        PSD_CHECK_LAUNCH();
        jpeg_size_kernel<<<(unsigned)((nb + 127) / 128), 128, 0, s>>>(bt);
        PSD_CHECK_LAUNCH();
        psd_clip_scan_kernel<<<1, 1024, 0, s>>>(bt.sizes, nb);
        PSD_CHECK_LAUNCH();
        jpeg_copy_kernel<<<(unsigned)n_chunks, kChunkThreads, 0, s>>>(bt, out, out_cap, image_bytes + i0);
        PSD_CHECK_LAUNCH();
        count_launch(8);
    }
    return PSD_OK;
}
