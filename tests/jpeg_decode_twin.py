"""numpy restatement of the baseline JPEG decoder cv2.imread(path, IMREAD_COLOR) / cv2.imdecode run (libjpeg-turbo:
islow IDCT, fancy upsampling, ycc_rgb_convert, BGR output).  Every step is integer arithmetic, so the twin and the
device decoder (jpeg_decode_kernels.cu) give the bytes cv2 does; this module pins each step, and `probe` is the
Python parser psd_jpeg_probe is checked against.  Test infrastructure only."""

from __future__ import annotations

import struct

import numpy as np

from tests.jpeg_twin import ZIGZAG

# psd_jpeg_probe refusal codes (include/psd_b200.h PSD_JPEG_*)
OK, TRUNCATED, NOT_JPEG, PROCESS, PRECISION, COMPONENTS, SAMPLING, MULTI_SCAN, ORIENTATION, TABLES = range(10)


class Info:
    """What psd_jpeg_probe reports of one file, plus the tables the twin decodes with."""

    def __init__(self):
        self.width = self.height = self.ncomp = 0
        self.hs, self.vs, self.tq, self.td, self.ta = [], [], [], [], []
        self.restart = 0
        self.scan0 = self.scan1 = 0   # entropy-coded data: [scan0, scan1) bytes
        self.code = OK
        self.qt = {}
        self.dc, self.ac = {}, {}


def _exif_orientation(seg: bytes) -> int:
    if seg[:6] != b"Exif\0\0" or len(seg) < 14:
        return 1
    t = seg[6:]
    e = "<" if t[:2] == b"II" else ">" if t[:2] == b"MM" else None
    if e is None:
        return 1
    off = struct.unpack(e + "I", t[4:8])[0]
    if off + 2 > len(t):
        return 1
    n = struct.unpack(e + "H", t[off:off + 2])[0]
    for i in range(n):
        p = off + 2 + 12 * i
        if p + 12 > len(t):
            break
        tag, typ = struct.unpack(e + "HH", t[p:p + 4])
        if tag == 0x0112 and typ == 3:
            return struct.unpack(e + "H", t[p + 8:p + 10])[0]
    return 1


def probe(data: bytes) -> Info:
    """Parse the markers up to the scan; `code` says why the file is refused (OK: it is not)."""
    info = Info()
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        info.code = NOT_JPEG
        return info
    p, sof = 2, False
    while True:
        while p < n and data[p] != 0xFF:
            p += 1
        while p < n and data[p] == 0xFF:
            p += 1
        if p >= n:
            info.code = TRUNCATED
            return info
        m = data[p]
        p += 1
        if m == 0xD9 or (0xD0 <= m <= 0xD7) or m == 0x01:
            if m == 0xD9:
                info.code = TRUNCATED
                return info
            continue
        if p + 2 > n:
            info.code = TRUNCATED
            return info
        L = (data[p] << 8) | data[p + 1]
        if L < 2 or p + L > n:
            info.code = TRUNCATED
            return info
        seg = data[p + 2:p + L]
        if m in (0xC0, 0xC1):
            if sof or len(seg) < 6:
                info.code = MULTI_SCAN if sof else TRUNCATED
                return info
            sof = True
            if seg[0] != 8:
                info.code = PRECISION
                return info
            info.height, info.width, info.ncomp = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if info.ncomp not in (1, 3):
                info.code = COMPONENTS
                return info
            if len(seg) < 6 + 3 * info.ncomp or info.width == 0 or info.height == 0:
                info.code = TRUNCATED
                return info
            ids = []
            for c in range(info.ncomp):
                cid, hv, tq = seg[6 + 3 * c:9 + 3 * c]
                ids.append(cid)
                info.hs.append(hv >> 4)
                info.vs.append(hv & 15)
                info.tq.append(tq)
            info.ids = ids
            if info.ncomp == 1:
                info.hs, info.vs = [1], [1]
            elif (info.hs[1:], info.vs[1:]) != ([1, 1], [1, 1]) or (info.hs[0], info.vs[0]) not in ((1, 1), (2, 1),
                                                                                                        (2, 2)):
                info.code = SAMPLING
                return info
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            info.code = PROCESS
            return info
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    info.code = TRUNCATED
                    return info
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                cnt = sum(bits)
                if q + 17 + cnt > len(seg) or tc > 1 or th > 3 or cnt > 256:
                    info.code = TABLES
                    return info
                (info.ac if tc else info.dc)[th] = (bits, list(seg[q + 17:q + 17 + cnt]))
                q += 17 + cnt
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                size = 64 * (2 if pq else 1)
                if q + 1 + size > len(seg) or tq > 3:
                    info.code = TABLES
                    return info
                if pq:
                    vals = [(seg[q + 1 + 2 * i] << 8) | seg[q + 2 + 2 * i] for i in range(64)]
                else:
                    vals = list(seg[q + 1:q + 65])
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = vals
                info.qt[tq] = nat
                q += 1 + size
        elif m == 0xDD:
            if len(seg) < 2:
                info.code = TRUNCATED
                return info
            info.restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            if seg[:5] == b"JFIF\0" and len(seg) >= 14:
                info.jfif = True
        elif m == 0xEE:
            if seg[:5] == b"Adobe" and len(seg) >= 12:
                info.adobe = seg[11]
        elif m == 0xE1:
            if _exif_orientation(seg) not in (0, 1):
                info.code = ORIENTATION
                return info
        elif m == 0xDA:
            if not sof:
                info.code = TRUNCATED
                return info
            ns = seg[0] if seg else 0
            if ns != info.ncomp:
                info.code = MULTI_SCAN
                return info
            if len(seg) < 1 + 2 * ns + 3:
                info.code = TRUNCATED
                return info
            for c in range(ns):
                cid, t = seg[1 + 2 * c:3 + 2 * c]
                if cid != info.ids[c]:
                    info.code = MULTI_SCAN
                    return info
                info.td.append(t >> 4)
                info.ta.append(t & 15)
            adobe = getattr(info, "adobe", None)
            if info.ncomp == 3 and not getattr(info, "jfif", False) and (
                    adobe == 0 or (adobe is None and info.ids == [82, 71, 66])):
                # jdapimin.c default_decompress_parms: RGB, which libjpeg does not convert from YCbCr
                info.code = COMPONENTS
                return info
            for c in range(ns):
                if (info.td[c] not in info.dc or info.ta[c] not in info.ac or info.tq[c] not in info.qt):
                    info.code = TABLES
                    return info
            info.scan0 = p + L
            # the scan ends at the last EOI; anything else after it would be another scan
            end = data.rfind(b"\xff\xd9")
            if end < info.scan0:
                info.code = TRUNCATED
                return info
            info.scan1 = end
            return info
        p += L


def _lookup(spec):
    """(bits, values) -> {(length, code): symbol}"""
    bits, vals = spec
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            table[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return table


def destuff(data: bytes, info: Info):
    """The scan's bytes with stuffed zeros and restart markers removed, and the byte offsets where each restart
    interval after the first begins."""
    seg = data[info.scan0:info.scan1]
    out, rst = bytearray(), []
    i = 0
    while i < len(seg):
        b = seg[i]
        if b == 0xFF and i + 1 < len(seg):
            nx = seg[i + 1]
            if nx == 0:
                out.append(0xFF)
                i += 2
                continue
            if 0xD0 <= nx <= 0xD7:
                rst.append(len(out))
                i += 2
                continue
            if nx == 0xFF:
                i += 1
                continue
            raise ValueError("marker inside the entropy-coded data")
        out.append(b)
        i += 1
    return bytes(out), rst


def coefficients(data: bytes, info: Info | None = None):
    """Huffman decode (jdhuff.c decode_mcu): the quantised coefficients of every block in scan order, [n_blocks][64]
    natural order, absolute DCs."""
    info = info or probe(data)
    if info.code != OK:
        raise ValueError(f"refused: {info.code}")
    s, rst = destuff(data, info)
    nbits = 8 * len(s)
    bits = np.unpackbits(np.frombuffer(s, np.uint8)) if s else np.zeros(0, np.uint8)
    dct = [_lookup(info.dc[t]) for t in info.td]
    act = [_lookup(info.ac[t]) for t in info.ta]
    mcu_comps = [c for c in range(info.ncomp) for _ in range(info.hs[c] * info.vs[c])] if info.ncomp > 1 else [0]
    mx, my = mcu_dims(info)
    n_mcu = mx * my
    out = np.zeros((n_mcu * len(mcu_comps), 64), np.int64)
    pos = 0
    pred = [0] * info.ncomp
    rst_i = 0

    def read(n):
        nonlocal pos
        v = 0
        for _ in range(n):
            v = (v << 1) | (int(bits[pos]) if pos < nbits else 1)
            pos += 1
        return v

    def symbol(t):
        code = 0
        for length in range(1, 17):
            code = (code << 1) | read(1)
            if (length, code) in t:
                return t[(length, code)]
        raise ValueError("bad Huffman code")

    def extend(v, s):
        return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v

    b = 0
    for m in range(n_mcu):
        if info.restart and m and m % info.restart == 0:
            if rst_i >= len(rst):
                raise ValueError("missing restart marker")
            pos = 8 * rst[rst_i]
            rst_i += 1
            pred = [0] * info.ncomp
        for c in mcu_comps:
            sdc = symbol(dct[c])
            pred[c] += extend(read(sdc), sdc)
            out[b, 0] = np.int16(np.int64(pred[c]).astype(np.int16))
            k = 1
            while k < 64:
                rs = symbol(act[c])
                r, sz = rs >> 4, rs & 15
                if sz:
                    k += r
                    if k > 63:
                        raise ValueError("coefficient index past 63")
                    out[b, ZIGZAG[k]] = extend(read(sz), sz)
                    k += 1
                elif r == 15:
                    k += 16
                else:
                    break
            b += 1
    if pos > nbits:
        # libjpeg-turbo pads a short stream and warns; the device decoder refuses it
        raise ValueError("entropy-coded data ends inside a block")
    return out


def mcu_dims(info: Info):
    hmax, vmax = max(info.hs), max(info.vs)
    return -(-info.width // (8 * hmax)), -(-info.height // (8 * vmax))


def range_limit(x):
    """jdmaster.c prepare_range_limit_table behind IDCT_range_limit, indexed by x & RANGE_MASK: x is a sample minus
    128 taken modulo 1024 as a signed 10-bit value, then clamped to [0, 255]"""
    s = (x & 1023)
    s = np.where(s >= 512, s - 1024, s)
    return np.clip(s + 128, 0, 255)


def idct_islow(coef, q):
    """jidctint.c jpeg_idct_islow of blocks [n][64] (quantised, natural order) with quantisation table q[64]:
    [n][8][8] samples"""
    c = (coef.astype(np.int64) * q[None, :]).reshape(-1, 8, 8)

    def one_d(d0, d1, d2, d3, d4, d5, d6, d7):
        z2, z3 = d2, d6
        z1 = (z2 + z3) * 4433
        tmp2 = z1 + z3 * -15137
        tmp3 = z1 + z2 * 6270
        tmp0 = (d0 + d4) * 8192
        tmp1 = (d0 - d4) * 8192
        tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        t0, t1, t2, t3 = d7, d5, d3, d1
        z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
        z5 = (z3 + z4) * 9633
        t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069, z4 * -3196
        z3 += z5
        z4 += z5
        t0 += z1 + z3
        t1 += z2 + z4
        t2 += z2 + z3
        t3 += z1 + z4
        return (tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3)

    # pass 1: columns, DESCALE by CONST_BITS - PASS1_BITS = 11
    cols = one_d(*[c[:, i, :] for i in range(8)])
    ws = np.stack([(v + 1024) >> 11 for v in cols], axis=1)
    ac_zero = np.all(c[:, 1:, :] == 0, axis=1)     # [n][col]: the column's ACs are all zero
    ws = np.where(ac_zero[:, None, :], c[:, 0:1, :] * 4, ws)
    # pass 2: rows, DESCALE by CONST_BITS + PASS1_BITS + 3 = 18
    rows = one_d(*[ws[:, :, j] for j in range(8)])
    out = np.stack([(v + (1 << 17)) >> 18 for v in rows], axis=2)
    return range_limit(out).astype(np.uint8)


def planes(data: bytes, info: Info | None = None):
    """Every component's plane of IDCT samples, whole blocks: [ncomp] arrays of (8 * blocks_y, 8 * blocks_x)"""
    info = info or probe(data)
    coef = coefficients(data, info)
    mx, my = mcu_dims(info)
    per = [info.hs[c] * info.vs[c] for c in range(info.ncomp)]
    bpm = sum(per)
    out = []
    start = 0
    for c in range(info.ncomp):
        h, v = info.hs[c], info.vs[c]
        blocks = coef.reshape(my * mx, bpm, 64)[:, start:start + per[c]]
        start += per[c]
        s = idct_islow(blocks.reshape(-1, 64), info.qt[info.tq[c]]).reshape(my, mx, v, h, 8, 8)
        out.append(s.transpose(0, 2, 4, 1, 3, 5).reshape(my * v * 8, mx * h * 8))
    return out


def upsample(p, dw, dh, h2, v2, w, h):
    """jdsample.c fancy upsampling of one chroma plane p whose first dh rows and dw columns are real (the rows below
    replicate the last real one, jdmainct.c set_bottom_pointers; the column right of the last real one repeats it,
    as the SIMD kernels pad it): h2v1 / h2v2 triangle filters with their alternating biases"""
    x = p[:dh, :dw].astype(np.int64)
    if (h2 or v2) and dw <= 2:
        # jdsample.c jinit_upsampler: fancy upsampling only when downsampled_width > 2, else h2v1_upsample /
        # h2v2_upsample replicate each sample
        o = np.repeat(np.repeat(x, 2, axis=1), 2 if v2 else 1, axis=0)
    elif v2:
        above = np.vstack([x[:1], x[:-1]])
        below = np.vstack([x[1:], x[-1:]])
        rows = np.empty((2 * dh, dw), np.int64)
        rows[0::2] = 3 * x + above
        rows[1::2] = 3 * x + below
        left = np.hstack([rows[:, :1], rows[:, :-1]])
        right = np.hstack([rows[:, 1:], rows[:, -1:]])
        o = np.empty((2 * dh, 2 * dw), np.int64)
        o[:, 0::2] = (3 * rows + left + 8) >> 4
        o[:, 1::2] = (3 * rows + right + 7) >> 4
        o[:, 0] = (4 * rows[:, 0] + 8) >> 4
    elif h2:
        left = np.hstack([x[:, :1], x[:, :-1]])
        right = np.hstack([x[:, 1:], x[:, -1:]])
        o = np.empty((dh, 2 * dw), np.int64)
        o[:, 0::2] = (3 * x + left + 1) >> 2
        o[:, 1::2] = (3 * x + right + 2) >> 2
        o[:, 0] = x[:, 0]
    else:
        o = x
    return o[:h, :w]


def ycc_bgr(y, cb, cr):
    """jdcolor.c ycc_rgb_convert with build_ycc_rgb_table, written B, G, R"""
    def fix(v):
        return int(v * 65536 + 0.5)
    xb, xr = cb.astype(np.int64) - 128, cr.astype(np.int64) - 128
    r_off = (fix(1.40200) * xr + 32768) >> 16
    b_off = (fix(1.77200) * xb + 32768) >> 16
    g_off = (-fix(0.34414) * xb + 32768 - fix(0.71414) * xr) >> 16
    y = y.astype(np.int64)
    return np.stack([np.clip(y + b_off, 0, 255), np.clip(y + g_off, 0, 255), np.clip(y + r_off, 0, 255)],
                    axis=-1).astype(np.uint8)


def decode(data: bytes) -> np.ndarray:
    """cv2.imdecode(data, IMREAD_COLOR) of a file psd_jpeg_probe accepts: (H, W, 3) uint8 BGR"""
    info = probe(data)
    if info.code != OK:
        raise ValueError(f"refused: {info.code}")
    p = planes(data, info)
    w, h = info.width, info.height
    if info.ncomp == 1:
        y = p[0][:h, :w]
        return np.repeat(y[:, :, None], 3, axis=2)
    hmax, vmax = info.hs[0], info.vs[0]
    dw, dh = -(-w // hmax), -(-h // vmax)
    cb = upsample(p[1], dw, dh, hmax == 2, vmax == 2, w, h)
    cr = upsample(p[2], dw, dh, hmax == 2, vmax == 2, w, h)
    return ycc_bgr(p[0][:h, :w], cb, cr)
