"""numpy restatement of the baseline JPEG encoder cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, q]) runs
(libjpeg-turbo: jpeg_set_quality with force_baseline, 4:2:0, the ITU T.81 Annex K Huffman tables, no
optimisation, no restart interval).  Every step is integer arithmetic, so the twin and the device encoder
(jpeg_kernels.cu) produce the bytes cv2 does, and this module is what pins each step.  Test infrastructure only."""

from __future__ import annotations

import numpy as np

# ITU T.81 Annex K.1 / K.2, natural (row-major) order
STD_LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_Q = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
    24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99], np.int64)
# zigzag index k -> natural index
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

# Annex K.3: (bits[1..16], values) of DC luma, AC luma, DC chroma, AC chroma
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7,
    0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5,
    0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
    0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0,
    0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26,
    0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5,
    0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
    0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])


def huff_codes(spec):
    """T.81 Annex C: symbol -> (code, length) arrays of 256 entries"""
    bits, vals = spec
    code_of, len_of = np.zeros(256, np.int64), np.zeros(256, np.int64)
    code, k = 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            code_of[vals[k]], len_of[vals[k]] = code, length
            code, k = code + 1, k + 1
        code <<= 1
    return code_of, len_of


def quant_tables(quality: int):
    """jpeg_set_quality(q, force_baseline=TRUE) after cv2's clamp to [0, 100]: natural-order luma, chroma tables"""
    q = min(max(int(quality), 0), 100)
    q = max(q, 1)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((base * scale + 50) // 100, 1, 255) for base in (STD_LUMA_Q, STD_CHROMA_Q)]


def reciprocal(divisor):
    """jcdctmgr.c compute_reciprocal for 16-bit DCTELEM: (recip, correction, shift) with
    |x| -> ((|x| + correction) * recip) >> shift"""
    b = int(divisor).bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, int(divisor))
    c = int(divisor) // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= int(divisor) // 2:
        c += 1
    else:
        fq += 1
    return fq, c, r


def quantize(coefs, qtable):
    """coefs [..., 64] islow output (natural order) -> quantised, with libjpeg-turbo's reciprocal division by
    8 * qtable"""
    rec = np.array([reciprocal(8 * int(v)) for v in qtable], np.int64)
    a = np.abs(coefs)
    q = ((a + rec[:, 1]) * rec[:, 0]) >> rec[:, 2]
    return np.where(coefs < 0, -q, q)


def ycc(bgr):
    """jccolor.c rgb_ycc_convert, 16-bit fixed point (JCS_EXT_BGR input)"""
    b, g, r = (bgr[..., c].astype(np.int64) for c in range(3))
    half, off = 1 << 15, 128 << 16
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + off + half - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + off + half - 1) >> 16
    return y, cb, cr


def fdct_islow(blocks):
    """jfdctint.c jpeg_fdct_islow on [..., 8, 8] int64 samples already centred by -128; output scaled by 8"""
    d = blocks.astype(np.int64).copy()

    def pass_(d, axis, shift_even, descale_even):
        x = [np.take(d, i, axis=axis) for i in range(8)]
        tmp0, tmp7 = x[0] + x[7], x[0] - x[7]
        tmp1, tmp6 = x[1] + x[6], x[1] - x[6]
        tmp2, tmp5 = x[2] + x[5], x[2] - x[5]
        tmp3, tmp4 = x[3] + x[4], x[3] - x[4]
        tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
        tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
        n = 13 + shift_even if descale_even else 13 - shift_even

        def ds(v, s):
            return (v + (1 << (s - 1))) >> s
        out = [None] * 8
        if descale_even:
            out[0], out[4] = ds(tmp10 + tmp11, shift_even), ds(tmp10 - tmp11, shift_even)
        else:
            out[0], out[4] = (tmp10 + tmp11) << shift_even, (tmp10 - tmp11) << shift_even
        z1 = (tmp12 + tmp13) * 4433
        out[2] = ds(z1 + tmp13 * 6270, n)
        out[6] = ds(z1 - tmp12 * 15137, n)
        z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
        z5 = (z3 + z4) * 9633
        tmp4, tmp5, tmp6, tmp7 = tmp4 * 2446, tmp5 * 16819, tmp6 * 25172, tmp7 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069, z4 * -3196
        z3 += z5
        z4 += z5
        out[7] = ds(tmp4 + z1 + z3, n)
        out[5] = ds(tmp5 + z2 + z4, n)
        out[3] = ds(tmp6 + z2 + z3, n)
        out[1] = ds(tmp7 + z1 + z4, n)
        return np.stack(out, axis=axis)
    d = pass_(d, -1, 2, False)   # rows
    d = pass_(d, -2, 2, True)    # columns
    return d


def planes(bgr):
    """The Y, Cb, Cr sample planes the coefficient controller reads, edges replicated as jcprepct.c and
    jcsample.c do: Y (8*ceil(h/8)) x (8*ceil(w/8)), chroma (8*ceil(h/16)) x (8*ceil(w/16)), h2v2 with bias 1, 2"""
    h, w = bgr.shape[:2]
    y, cb, cr = ycc(bgr)
    yh, yw = 8 * -(-h // 8), 8 * -(-w // 8)
    ch, cw = 8 * -(-h // 16), 8 * -(-w // 16)
    rows, cols = np.minimum(np.arange(yh), h - 1), np.minimum(np.arange(yw), w - 1)
    yp = y[rows][:, cols]
    # chroma: full-resolution rows padded to an even count, downsampled, then the last downsampled row repeated;
    # columns expanded to 2 * cw by repetition before downsampling
    crow = np.minimum(np.arange(ch), (h + 1) // 2 - 1)
    r0, r1 = np.minimum(2 * crow, h - 1), np.minimum(2 * crow + 1, h - 1)
    c0, c1 = np.minimum(2 * np.arange(cw), w - 1), np.minimum(2 * np.arange(cw) + 1, w - 1)
    bias = np.tile([1, 2], cw)[:cw]
    out = []
    for p in (cb, cr):
        s = p[r0][:, c0] + p[r0][:, c1] + p[r1][:, c0] + p[r1][:, c1]
        out.append((s + bias) >> 2)
    return yp, out[0], out[1]


def to_blocks(plane):
    ph, pw = plane.shape
    return plane.reshape(ph // 8, 8, pw // 8, 8).transpose(0, 2, 1, 3)


def mcu_coefficients(bgr, quality):
    """Quantised zigzag coefficients of every block in scan order (MCU by MCU: Y00 Y01 Y10 Y11 Cb Cr), dummy
    blocks included ([n_mcu * 6, 64] int64), and each block's component (0 luma, 1 chroma)"""
    h, w = bgr.shape[:2]
    ql, qc = quant_tables(quality)
    yp, cb, cr = planes(bgr)
    yq = quantize(fdct_islow(to_blocks(yp) - 128).reshape(*to_blocks(yp).shape[:2], 64), ql)
    cq = [quantize(fdct_islow(to_blocks(p) - 128).reshape(*to_blocks(p).shape[:2], 64), qc) for p in (cb, cr)]
    hib, wib = yq.shape[:2]
    mh, mw = cq[0].shape[:2]
    out = np.zeros((mh, mw, 6, 64), np.int64)
    for k, (r, c) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        by, bx = 2 * np.arange(mh)[:, None] + r, 2 * np.arange(mw)[None, :] + c
        real = (by < hib) & (bx < wib)
        # jccoefct.c dummy blocks: a block right of the image takes the DC of its left neighbour, a block below it
        # the DC of the MCU's Y01 (itself a dummy of Y00 when the image ends at Y00)
        sy = np.where(by < hib, by, 2 * np.arange(mh)[:, None])
        sx = np.minimum(np.where(by < hib, bx, 2 * np.arange(mw)[None, :] + 1), wib - 1)
        blk = yq[np.broadcast_to(sy, real.shape), np.broadcast_to(sx, real.shape)]
        blk[..., 1:] *= real[..., None]
        out[:, :, k] = blk
    out[:, :, 4], out[:, :, 5] = cq
    return out.reshape(-1, 64)[:, ZIGZAG].copy()


def _bits_of(values, nbits):
    """(size category, the nbits low bits JPEG appends) of signed coefficients"""
    a = np.abs(values)
    size = np.zeros_like(a)
    nz = a > 0
    size[nz] = np.floor(np.log2(a[nz])).astype(np.int64) + 1
    extra = np.where(values < 0, values - 1, values) & ((1 << size) - 1)
    return size, extra


def entropy_codes(coefs):
    """Huffman codes of the scan in stream order: (code, length) int64 arrays"""
    n = coefs.shape[0]
    comp = np.tile([0, 0, 0, 0, 1, 2], n // 6)
    tables = [(huff_codes(DC_LUMA), huff_codes(AC_LUMA)), (huff_codes(DC_CHROMA), huff_codes(AC_CHROMA))]
    dc = coefs[:, 0]
    prev = np.zeros(n, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    diff = dc - prev
    dsize, dextra = _bits_of(diff, None)
    # every code as (block, order, code, length): order 0 the DC, then the ACs by zigzag index, EOB last
    chroma = comp > 0
    blocks, orders, codes, lens = [], [], [], []
    dcc = np.where(chroma, tables[1][0][0][dsize], tables[0][0][0][dsize])
    dcl = np.where(chroma, tables[1][0][1][dsize], tables[0][0][1][dsize])
    blocks.append(np.arange(n))
    orders.append(np.zeros(n, np.int64))
    codes.append((dcc << dsize) | dextra)
    lens.append(dcl + dsize)
    b, k = np.nonzero(coefs[:, 1:])
    k = k + 1
    v = coefs[b, k]
    first = np.ones(len(b), bool)
    first[1:] = b[1:] != b[:-1]
    prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prevk - 1
    size, extra = _bits_of(v, None)
    sym = ((run % 16) << 4) | size
    ch = chroma[b]
    acc = np.where(ch, tables[1][1][0][sym], tables[0][1][0][sym])
    acl = np.where(ch, tables[1][1][1][sym], tables[0][1][1][sym])
    zrl = run // 16
    zc = np.where(ch, tables[1][1][0][0xF0], tables[0][1][0][0xF0])
    zl = np.where(ch, tables[1][1][1][0xF0], tables[0][1][1][0xF0])
    # run // 16 ZRL codes ahead of each coefficient (all equal, so their relative order does not matter)
    zi = np.repeat(np.arange(len(b)), zrl)
    blocks.append(b[zi])
    orders.append(2 * k[zi] - 1)
    codes.append(zc[zi])
    lens.append(zl[zi])
    blocks.append(b)
    orders.append(2 * k)
    codes.append((acc << size) | extra)
    lens.append(acl + size)
    last = np.zeros(n, np.int64)
    np.maximum.at(last, b, k)
    eob = last < 63
    blocks.append(np.arange(n)[eob])
    orders.append(np.full(int(eob.sum()), 200, np.int64))
    codes.append(np.where(chroma, tables[1][1][0][0], tables[0][1][0][0])[eob])
    lens.append(np.where(chroma, tables[1][1][1][0], tables[0][1][1][0])[eob])
    blocks, orders = np.concatenate(blocks), np.concatenate(orders)
    o = np.lexsort((orders, blocks))
    return np.concatenate(codes)[o], np.concatenate(lens)[o]


def pack_bits(codes, lens):
    """MSB-first bit string of the codes, padded with 1-bits to a byte, every 0xFF followed by 0x00"""
    total = int(lens.sum())
    ends = np.cumsum(lens)
    # bit j of the stream: which code, and which bit of it
    owner = np.repeat(np.arange(len(lens)), lens)
    pos_in = np.arange(total) - (ends - lens)[owner]
    bits = (codes[owner] >> (lens[owner] - 1 - pos_in)) & 1
    pad = (-total) % 8
    bits = np.concatenate([bits, np.ones(pad, np.int64)]).astype(np.uint8)
    raw = np.packbits(bits)
    ff = np.nonzero(raw == 0xFF)[0]
    return np.insert(raw, ff + 1, 0).tobytes()


def header(width, height, quality):
    """SOI, APP0 (JFIF 1.01), DQT 0 and 1, SOF0 (4:2:0), DHT DC0 AC0 DC1 AC1, SOS: the 623 bytes ahead of the scan"""
    out = bytearray(b"\xff\xd8\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t, table in enumerate(quant_tables(quality)):
        out += bytes([0xFF, 0xDB, 0x00, 0x43, t]) + bytes(int(v) for v in table[ZIGZAG])
    out += bytes([0xFF, 0xC0, 0x00, 0x11, 8, height >> 8, height & 255, width >> 8, width & 255, 3,
                  1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for cls_id, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        n = 2 + 1 + 16 + len(vals)
        out += bytes([0xFF, 0xC4, n >> 8, n & 255, cls_id]) + bytes(bits) + bytes(vals)
    out += bytes([0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


def encode(bgr, quality=95):
    """The bytes of cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, quality])[1] for an (h, w, 3) uint8
    BGR image"""
    bgr = np.asarray(bgr)
    h, w = bgr.shape[:2]
    codes, lens = entropy_codes(mcu_coefficients(bgr, quality))
    return header(w, h, quality) + pack_bits(codes, lens) + b"\xff\xd9"
