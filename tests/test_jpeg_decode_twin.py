"""The numpy restatement of libjpeg-turbo's baseline decoder (tests/jpeg_decode_twin.py) gives what cv2.imdecode
gives on every sampling, size, quality, restart interval and table choice the device decoder takes; psd_jpeg_probe
agrees with the twin's parser and refuses what the decoder does not take; ImageSequenceStream resolves patterns as
cv2.VideoCapture does and reads, seeks and recycles its pool as documented."""

from __future__ import annotations

import os

import cv2
import numpy as np
import pytest

from tests import jpeg_decode_twin as D
from tests import jpeg_twin as J

SAMPLINGS = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "gray": None}


def frame(kind, w, h, seed=0):
    rng = np.random.default_rng(seed + 7919 * w + h)
    y, x = np.mgrid[:h, :w]
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "checker":
        v = ((x + y) % 2 * 255).astype(np.uint8)
        return np.stack([v, 255 - v, v], -1)
    return np.stack([(x * 7 + y) % 256, (y * 5) % 256, ((x + y) * 3) % 256], -1).astype(np.uint8)


def encode(img, sampling="420", q=95, restart=0, optimize=False):
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if sampling == "gray":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[sampling]]
    if restart:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    return cv2.imencode(".jpg", img, params)[1].tobytes()


def imdecode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def matrix():
    """(kind, w, h, sampling, q, restart, optimize): every width and height 1..40 (against a partner size), odd sizes
    up to 300x200, every sampling, qualities 1-100, restart intervals 1 and 4, optimised tables"""
    out = []
    samplings = list(SAMPLINGS)
    for n in range(1, 41):
        s = samplings[n % 4]
        out.append(("grad", n, 1 + (3 * n) % 40, s, (1, 50, 75, 95, 100)[n % 5], (0, 1, 4)[n % 3], n % 2 == 0))
        out.append(("noise", 1 + (7 * n) % 40, n, samplings[(n + 1) % 4], (100, 95, 75, 50, 1)[n % 5], 0, n % 3 == 0))
    for w, h in ((97, 61), (131, 77), (203, 149), (299, 199)):
        for s in samplings:
            out.append(("grad", w, h, s, 75, 4, False))
    for s in samplings:
        out.append(("noise", 64, 48, s, 100, 0, False))     # the largest coefficients
        out.append(("checker", 64, 48, s, 1, 1, True))      # the coarsest quantisation
    return out


CASES = matrix()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_twin_equals_imdecode(case):
    kind, w, h, s, q, rst, opt = case
    data = encode(frame(kind, w, h), s, q, rst, opt)
    assert np.array_equal(D.decode(data), imdecode(data)), case


def test_range_limit_equals_the_table():
    """D.range_limit (a signed 10-bit wrap, then a clamp) equals jdmaster.c prepare_range_limit_table indexed the way
    IDCT_range_limit and RANGE_MASK index it, over every value the mask can see"""
    table = np.zeros(5 * 256 + 128, np.int64)
    t0 = 256                                    # table += MAXJSAMPLE + 1: negative subscripts allowed
    table[t0:t0 + 256] = np.arange(256)
    table[t0 + 128 + 128:t0 + 128 + 512] = 255   # post-IDCT part: x in [128, 512) -> 255
    table[t0 + 128 + 512:t0 + 128 + 896] = 0
    table[t0 + 128 + 896:t0 + 128 + 1024] = np.arange(128)
    x = np.arange(-4096, 4096)
    assert np.array_equal(D.range_limit(x), table[t0 + 128 + (x & 1023)])


def test_own_encoder_round_trip():
    from tests import jpeg_cases as K
    for c, w, h, q in list(K.cases(large=False))[:40]:
        data = J.encode(K.frame(c, w, h), q)
        assert np.array_equal(D.decode(data), imdecode(data)), (c, w, h, q)


# ---- psd_jpeg_probe ----

def _lib_or_skip():
    from pyscenedetect_b200 import _capi
    try:
        _capi.load()
    except ImportError as e:
        pytest.skip(str(e))
    from pyscenedetect_b200 import image_sequence
    return image_sequence


@pytest.mark.parametrize("case", CASES[::3], ids=lambda c: "-".join(map(str, c)))
def test_probe_matches_parser(case):
    seq = _lib_or_skip()
    kind, w, h, s, q, rst, opt = case
    data = encode(frame(kind, w, h), s, q, rst, opt)
    got, want = seq.probe(data), D.probe(data)
    assert got.refusal == want.code == D.OK
    assert (got.width, got.height, got.components) == (want.width, want.height, want.ncomp)
    assert (got.h_samp, got.v_samp) == (want.hs[0], want.vs[0])
    assert got.restart_interval == want.restart
    assert (got.scan_begin, got.scan_end) == (want.scan0, want.scan1)


def _exif(orientation):
    tiff = b"II*\x00" + (8).to_bytes(4, "little") + (1).to_bytes(2, "little")
    tiff += (0x0112).to_bytes(2, "little") + (3).to_bytes(2, "little") + (1).to_bytes(4, "little")
    tiff += orientation.to_bytes(2, "little") + b"\x00\x00" + (0).to_bytes(4, "little")
    seg = b"Exif\x00\x00" + tiff
    return b"\xff\xe1" + (len(seg) + 2).to_bytes(2, "big") + seg


def refused_files():
    img = frame("grad", 48, 32)
    base = encode(img)
    sof = base.index(b"\xff\xc0")
    four = bytearray(base)
    four[sof + 9] = 4           # component count of the SOF
    return {
        "progressive": (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), D.PROCESS),
        "411": (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])[1].tobytes(), D.SAMPLING),
        "440": (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])[1].tobytes(), D.SAMPLING),
        "four_components": (bytes(four), D.COMPONENTS),
        "exif_orientation_6": (base[:2] + _exif(6) + base[2:], D.ORIENTATION),
        "truncated": (base[:len(base) // 2], D.TRUNCATED),
        "not_jpeg": (b"\x89PNG" + base[4:], D.NOT_JPEG),
    }


@pytest.mark.parametrize("name", list(refused_files()))
def test_probe_refuses(name):
    seq = _lib_or_skip()
    data, code = refused_files()[name]
    assert D.probe(data).code == code
    assert seq.probe(data).refusal == code
    with pytest.raises(ValueError, match="frame_x.jpg"):
        seq.check_file(data, "frame_x.jpg")


def test_exif_orientation_1_is_taken():
    seq = _lib_or_skip()
    base = encode(frame("grad", 24, 16))
    data = base[:2] + _exif(1) + base[2:]
    assert seq.probe(data).refusal == 0
    assert np.array_equal(D.decode(data), imdecode(data))


# ---- ImageSequenceStream host logic, the twin as its decoder ----

class TwinDecoder:
    def __init__(self):
        self.allocated = 0

    def dlpack_device(self):
        return (1, 0)

    def allocate(self, n, h, w):
        self.allocated += 1
        return np.zeros((n, h, w, 3), np.uint8)

    def decode(self, datas, names, out):
        for i, d in enumerate(datas):
            out[i] = D.decode(d)
        return out


def write_sequence(tmp, indexes, w=24, h=16):
    for i in indexes:
        with open(os.path.join(tmp, f"x_{i:04d}.jpg"), "wb") as f:
            f.write(encode(frame("noise", w, h, seed=i), "420", 90))
    return os.path.join(tmp, "x_%04d.jpg")


@pytest.mark.parametrize("start", [0, 1, 3, 4, 5])
def test_pattern_resolves_as_videocapture(tmp_path, start):
    seq = _lib_or_skip()
    pattern = write_sequence(str(tmp_path), list(range(start, start + 5)) + [start + 6, start + 7])
    cap = cv2.VideoCapture(pattern)
    n_cap = 0
    if cap.isOpened():
        while cap.read()[0]:
            n_cap += 1
    cap.release()
    if start >= seq.FIRST_INDEXES:
        assert n_cap == 0
        with pytest.raises(ValueError):
            seq.ImageSequenceStream(pattern, decoder=TwinDecoder())
        return
    s = seq.ImageSequenceStream(pattern, decoder=TwinDecoder())
    assert s.duration.frame_num == n_cap == 5
    assert s.paths[0].endswith(f"x_{start:04d}.jpg")
    assert s.name == "x_"
    assert float(s.frame_rate) == 25.0


def test_read_seek_and_batches(tmp_path):
    seq = _lib_or_skip()
    pattern = write_sequence(str(tmp_path), range(12))
    dec = TwinDecoder()
    s = seq.ImageSequenceStream(pattern, batch_size=4, decoder=dec)
    want = [cv2.imread(p) for p in s.paths]
    assert s.frame_size == (24, 16) and s.is_seekable
    f = s.read()
    assert np.array_equal(f, want[0]) and s.frame_number == 1 and s.position.frame_num == 0
    assert s.read(decode=False) is True and s.frame_number == 2
    b = s.read_batch(10)
    assert b.shape[0] == 4 and all(np.array_equal(b[i], want[2 + i]) for i in range(4))
    assert s.position.frame_num == 5
    s.seek(9)
    b = s.read_batch(10)
    assert b.shape[0] == 3 and np.array_equal(b[0], want[9]) and s.read_batch(1) is None and s.read() is False
    s.reset()
    assert s.frame_number == 0 and np.array_equal(s.read(), want[0])


def test_pool_reuse(tmp_path):
    """Batches rotate through three buffers: a batch is unchanged until two more have been read"""
    seq = _lib_or_skip()
    pattern = write_sequence(str(tmp_path), range(40))
    dec = TwinDecoder()
    s = seq.ImageSequenceStream(pattern, batch_size=2, decoder=dec)
    want = [cv2.imread(p) for p in s.paths]
    held = []
    while True:
        b = s.read_batch(2)
        if b is None:
            break
        held.append((s.frame_number - b.shape[0], b))
        if len(held) >= 3:
            first, old = held[-3]
            assert all(np.array_equal(old[i], want[first + i]) for i in range(old.shape[0]))
    assert dec.allocated == 3


def test_mixed_sizes_refused(tmp_path):
    seq = _lib_or_skip()
    a, b = str(tmp_path / "a.jpg"), str(tmp_path / "b.jpg")
    with open(a, "wb") as f:
        f.write(encode(frame("grad", 24, 16)))
    with open(b, "wb") as f:
        f.write(encode(frame("grad", 32, 16)))
    s = seq.ImageSequenceStream([a, b, a], decoder=TwinDecoder())
    assert s.name == "a"
    assert np.array_equal(s.read(), cv2.imread(a))
    with pytest.raises(ValueError, match=r"b\.jpg: 32x16"):
        s.read()
    s.seek(2)
    assert np.array_equal(s.read_batch(4)[0], cv2.imread(a))


def _without_jfif(data, ids=None, adobe=None):
    """data with its APP0 (JFIF) segment removed, optionally an APP14 Adobe segment with `adobe` as its transform,
    and the SOF / SOS component ids replaced by `ids`"""
    p = data.index(b"\xff\xe0")
    L = (data[p + 2] << 8) | data[p + 3]
    b = bytearray(data[:p] + data[p + 2 + L:])
    if ids is not None:
        sof = b.index(b"\xff\xc0")
        sos = b.index(b"\xff\xda")
        for c in range(3):
            b[sof + 10 + 3 * c] = ids[c]
            b[sos + 5 + 2 * c] = ids[c]
    if adobe is not None:
        seg = b"Adobe" + bytes([0, 100, 0, 0, 0, 0, adobe])
        b[2:2] = b"\xff\xee" + (len(seg) + 2).to_bytes(2, "big") + seg
    return bytes(b)


@pytest.mark.parametrize("case,refused", [("jfif_adobe0", False), ("adobe0", True), ("adobe1", False),
                                          ("adobe2", False), ("rgb_ids", True), ("rgb_ids_jfif", False),
                                          ("ycc_ids", False)])
def test_colour_space_of_three_components(case, refused):
    """jdapimin.c default_decompress_parms: a JFIF marker means YCbCr; without one an Adobe transform of 0, or
    (no Adobe marker) component ids 'R', 'G', 'B', mean RGB, which the decoder refuses; anything else is YCbCr"""
    seq = _lib_or_skip()
    base = encode(frame("grad", 40, 24), "444", 90)
    data = {
        "jfif_adobe0": base[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + base[2:],
        "adobe0": _without_jfif(base, adobe=0),
        "adobe1": _without_jfif(base, adobe=1),
        "adobe2": _without_jfif(base, adobe=2),
        "rgb_ids": _without_jfif(base, ids=b"RGB"),
        "rgb_ids_jfif": bytes(bytearray(base)),
        "ycc_ids": _without_jfif(base),
    }[case]
    if case == "rgb_ids_jfif":
        b = bytearray(base)
        sof, sos = b.index(b"\xff\xc0"), b.index(b"\xff\xda")
        for c in range(3):
            b[sof + 10 + 3 * c] = b"RGB"[c]
            b[sos + 5 + 2 * c] = b"RGB"[c]
        data = bytes(b)
    assert (seq.probe(data).refusal == D.COMPONENTS) == refused
    assert (D.probe(data).code == D.COMPONENTS) == refused
    if not refused:
        assert np.array_equal(D.decode(data), imdecode(data))
