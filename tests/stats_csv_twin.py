"""Python twin of csrc/stats_csv.cuh and of psd_clip_stats_csv (clip_kernels.cu): the three things a StatsManager
row prints, restated statement by statement with the device's integer widths, and the row layout of a pass.

* `format_f64(x)` is `str(float(x))` (and `str(numpy.float64(x))`): the shortest decimal that reads back as x,
  the nearest such when there are several (ties to an even last digit), found with Schubfach's rounding interval
  over a 126-bit power-of-ten table (`G`), then laid out as Python's repr lays it out.
* `timecode(frame, rate)` is `FrameTimecode(frame, rate).get_timecode()` (common.py:421-465) for `rate` =
  float(frame rate), with `round(secs, 3)` done exactly on the double's significand.
* `pass_csv` is what the counting, scan and writing passes leave for one pass: every clip's rows, back to back, and
  the clip byte offsets.

`python -m tests.stats_csv_twin` prints the table csrc/stats_csv.cuh holds."""

from __future__ import annotations

import struct

import numpy as np

M64 = (1 << 64) - 1
MASK_63 = (1 << 63) - 1
K_MIN, K_MAX = -324, 292      # flog10pow2 over the binary exponents of finite doubles
Q_MIN = -1074                 # exponent of the least subnormal's unit
C_MIN = 1 << 52               # implicit bit
C_TINY = 3                    # subnormal significands below this are special-cased
TEN_HIGH = 115292150460684698 << 4  # ceil(2^64 / 10): umulhi(s, TEN_HIGH) = s / 10 for the s that occur


def flog10pow2(e: int) -> int:
    """floor(e * log10(2)) for |e| <= 5456721"""
    return (e * 661971961083) >> 41


def flog10three_quarters_pow2(e: int) -> int:
    """floor(log10(3/4 * 2^e))"""
    return (e * 661971961083 - 274743187321) >> 41


def flog2pow10(e: int) -> int:
    """floor(e * log2(10))"""
    return (e * 913124641741) >> 38


def _g(k: int) -> int:
    """floor(10^-k * 2^(125 - flog2pow10(-k))) + 1: a 126-bit integer"""
    s = 125 - flog2pow10(-k)
    if -k >= 0:
        num, den = 10 ** -k, 1
    else:
        num, den = 1, 10 ** k
    num <<= max(s, 0)
    den <<= max(-s, 0)
    return num // den + 1


G = [(_g(k) >> 63, _g(k) & MASK_63) for k in range(K_MIN, K_MAX + 1)]  # (g1, g0)


def _umulhi(a: int, b: int) -> int:
    return ((a & M64) * (b & M64)) >> 64


def _rop(g1: int, g0: int, cp: int) -> int:
    """floor(g * cp / 2^127) with a sticky low bit (round to odd), as the device computes it in 64-bit words"""
    x1 = _umulhi(g0, cp)
    y0 = (g1 * cp) & M64
    y1 = _umulhi(g1, cp)
    z = ((y0 >> 1) + x1) & M64
    vbp = (y1 + (z >> 63)) & M64
    return vbp | ((((z & MASK_63) + MASK_63) & M64) >> 63)


def _schubfach(q: int, c: int) -> tuple[int, int]:
    """The decimal (f, e), f * 10^e, that prints c * 2^q"""
    out = c & 1
    cb = c << 2
    cbr = cb + 2
    if c != C_MIN or q == Q_MIN:
        cbl, k = cb - 2, flog10pow2(q)
    else:
        cbl, k = cb - 1, flog10three_quarters_pow2(q)
    h = q + flog2pow10(-k) + 2
    g1, g0 = G[k - K_MIN]
    vb = _rop(g1, g0, (cb << h) & M64)
    vbl = _rop(g1, g0, (cbl << h) & M64)
    vbr = _rop(g1, g0, (cbr << h) & M64)
    s = vb >> 2
    if s >= 10:  # one digit fewer (Python prints a single digit where one reads back; Java wants two)
        sp10 = 10 * _umulhi(s, TEN_HIGH)
        tp10 = sp10 + 10
        upin = vbl + out <= sp10 << 2
        wpin = (tp10 << 2) + out <= vbr
        if upin != wpin:
            return (sp10 if upin else tp10), k
    t = s + 1
    uin = vbl + out <= s << 2
    win = (t << 2) + out <= vbr
    if uin != win:
        return (s if uin else t), k
    cmp = vb - ((s + t) << 1)
    return (s if cmp < 0 or (cmp == 0 and (s & 1) == 0) else t), k


def decimal_of(x: float) -> tuple[int, int, int]:
    """(sign, f, e) of a finite nonzero double: f * 10^e is its shortest decimal, f without trailing zeros"""
    bits = struct.unpack("<Q", struct.pack("<d", x))[0]
    sign, bq, t = bits >> 63, (bits >> 52) & 0x7FF, bits & (C_MIN - 1)
    if bq:
        mq = -Q_MIN + 1 - bq
        c = C_MIN | t
        if 0 < mq < 53 and ((c >> mq) << mq) == c:  # an integer below 2^53: exact
            f, e = c >> mq, 0
        else:
            f, e = _schubfach(-mq, c)
    elif t < C_TINY:  # 2^-1074 and 2^-1073, whose rounding intervals are too narrow for the table: 5e-324, 1e-323
        f, e = (5, -324) if t == 1 else (1, -323)
    else:
        f, e = _schubfach(Q_MIN, t)
    while f % 10 == 0:
        f //= 10
        e += 1
    return sign, f, e


def format_f64(x) -> str:
    """str(float(x)): fixed notation for a decimal exponent -4 .. 15, else d.ddde+XX"""
    x = float(x)
    if x != x:
        return "nan"
    neg = "-" if struct.pack("<d", x)[7] & 0x80 else ""
    if x in (float("inf"), float("-inf")):
        return neg + "inf"
    if x == 0.0:
        return neg + "0.0"
    _, f, e = decimal_of(x)
    digits = str(f)
    n = len(digits)
    e10 = e + n - 1          # exponent of the first digit
    if -4 <= e10 <= 15:
        if e10 < 0:
            return neg + "0." + "0" * (-e10 - 1) + digits
        if e10 + 1 < n:
            return neg + digits[:e10 + 1] + "." + digits[e10 + 1:]
        return neg + digits + "0" * (e10 + 1 - n) + ".0"
    mant = digits[0] + ("." + digits[1:] if n > 1 else "")
    return f"{neg}{mant}e{'-' if e10 < 0 else '+'}{abs(e10):02d}"


def round_millis(secs: float) -> int:
    """round(secs * 1000) half to even on the exact value of a double 0 <= secs < 2^10 (what round(secs, 3) prints
    with 3 decimals)"""
    bits = struct.unpack("<Q", struct.pack("<d", secs))[0]
    bq, t = (bits >> 52) & 0x7FF, bits & (C_MIN - 1)
    if bq == 0 and t == 0:
        return 0
    m = (C_MIN | t) if bq else t
    sh = 1075 - bq if bq else 1074      # secs = m * 2^-sh
    n = m * 1000                        # < 2^63
    if sh <= 0:
        return n << -sh
    if sh >= 64:
        return 0                        # n / 2^sh < 1/2
    q, rem, half = n >> sh, n & ((1 << sh) - 1), 1 << (sh - 1)
    if rem > half or (rem == half and q & 1):
        q += 1
    return q


def timecode(frame: int, rate: float) -> str:
    """FrameTimecode(frame, rate).get_timecode(): HH:MM:SS.nnn"""
    secs = frame / rate
    hrs = int(secs / 3600.0)
    secs = secs - hrs * 3600.0
    mins = int(secs / 60.0)
    secs = max(0.0, secs - mins * 60.0)
    ms = round_millis(secs)
    if ms >= 60000:
        ms, mins = 0, mins + 1
        if mins >= 60:
            mins, hrs = 0, hrs + 1
    return f"{hrs:02d}:{mins:02d}:{ms // 1000:02d}.{ms % 1000:03d}"


def row_present(local: int, length: int, columns) -> bool:
    return any(head <= local < length - tail for _, _, head, tail in columns)


def pass_csv(columns, offsets, first_frames, rates) -> tuple[bytes, list[int]]:
    """What psd_clip_stats_csv writes for one pass: columns = [(values float64, stride, head, tail)] in CSV order (frame
    i's value at values[i * stride]) and the clip table.  -> (every clip's rows back to back, clip byte offsets)"""
    text, clip_bytes = b"", [0]
    for j in range(len(offsets) - 1):
        b, e = int(offsets[j]), int(offsets[j + 1])
        for i in range(b, e):
            local = i - b
            if not any(head <= local < (e - b) - tail for _, _, head, tail in columns):
                continue
            frame = int(first_frames[j]) + local
            cells = [str(frame + 1), timecode(frame, float(rates[j]))]
            for values, stride, head, tail in columns:
                cells.append(format_f64(values[i * stride]) if head <= local < (e - b) - tail else "None")
            text += (",".join(cells) + "\n").encode()
        clip_bytes.append(len(text))
    return text, clip_bytes


def cuh_table() -> str:
    """The g table of csrc/stats_csv.cuh: {g1, g0} for k = K_MIN .. K_MAX, two entries per line"""
    lines = []
    for i in range(0, len(G), 2):
        lines.append("    " + " ".join(f"{{0x{g1:016x}ull, 0x{g0:016x}ull}}," for g1, g0 in G[i:i + 2]))
    return "\n".join(lines)


def random_doubles(n: int, seed: int) -> np.ndarray:
    """n doubles from uniformly random bit patterns (NaNs and infinities included)"""
    return np.random.default_rng(seed).integers(0, 1 << 64, size=n, dtype=np.uint64).view(np.float64)


if __name__ == "__main__":
    print(cuh_table())
