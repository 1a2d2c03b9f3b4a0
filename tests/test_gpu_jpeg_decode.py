"""psd_jpeg_decode on the device gives cv2.imdecode's bytes on the twin's matrix and at 1080p, 4K and 8K, in mixed-size
batches, through packed, RGB and NCHW layouts and across sub-batches; corrupt or short data sets the file's error flag and the
stream's ValueError; SceneManager, detect_clips, ParameterSweep.run_clips and save_images take an ImageSequenceStream
and give what they give on the imread frames."""

from __future__ import annotations

import os
import subprocess

import cv2
import numpy as np
import pytest

from tests import test_jpeg_decode_twin as T

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _seq():
    from pyscenedetect_b200 import image_sequence
    return image_sequence


def big_frame(w, h, seed):
    """noise, a gradient and text: the synthetic frame the sequence benchmark encodes"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    f = np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y + seed * 40) % 256)], -1)
    f = (f + rng.integers(-20, 21, (h, w, 3))).clip(0, 255).astype(np.uint8)
    cv2.putText(f, f"frame {seed}", (w // 8, h // 2), cv2.FONT_HERSHEY_SIMPLEX, h / 300, (255, 255, 255), 3)
    return f


def decode_images(datas, layout="packed", workspace_cap=0):
    """psd_jpeg_decode of files of any sizes in one call, each into its own tensor in `layout`: BGR images"""
    import ctypes as C
    from pyscenedetect_b200 import _capi
    seq = _seq()
    n = len(datas)
    infos = [seq.probe(d) for d in datas]
    outs, imgs = [], (_capi.PsdJpegImage * n)()
    for i, info in enumerate(infos):
        w, h = info.width, info.height
        if layout == "nchw":
            t = torch.zeros((3, h, w), dtype=torch.uint8, device="cuda")
            base, lay = t[0].data_ptr(), _capi.PsdFrameLayout(0, w, 1, h * w)
        elif layout == "rgb":
            t = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
            base, lay = t[:, :, 2].data_ptr(), _capi.PsdFrameLayout(0, 3 * w, 3, -1)
        else:
            t = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
            base, lay = t.data_ptr(), _capi.PsdFrameLayout(0, 3 * w, 3, 1)
        outs.append(t)
        imgs[i].base, imgs[i].layout, imgs[i].width, imgs[i].height = base, lay, w, h
    host = [np.frombuffer(d, np.uint8) for d in datas]
    dev = [torch.from_numpy(h.copy()).cuda() for h in host]
    srcs = (_capi.PsdJpegSource * n)()
    for i in range(n):
        srcs[i].host, srcs[i].device, srcs[i].size = host[i].ctypes.data, dev[i].data_ptr(), host[i].size
    flags = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    rc = _capi.load().psd_jpeg_decode(0, srcs, n, imgs, workspace_cap, flags.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream)
    _capi.check(rc, "psd_jpeg_decode")
    torch.cuda.synchronize()
    res = []
    for t in outs:
        a = t.cpu().numpy()
        if layout == "nchw":
            a = a.transpose(1, 2, 0)
        elif layout == "rgb":
            a = a[..., ::-1]
        res.append(np.ascontiguousarray(a))
    return res, flags.cpu().numpy()


def test_matrix_equals_imdecode():
    datas = [T.encode(T.frame(k, w, h), s, q, r, o) for k, w, h, s, q, r, o in T.CASES]
    got, flags = decode_images(datas)
    assert not flags.any()
    bad = [T.CASES[i] for i, (g, d) in enumerate(zip(got, datas)) if not np.array_equal(g, T.imdecode(d))]
    assert not bad, bad[:5]


@pytest.mark.parametrize("layout", ["packed", "rgb", "nchw"])
def test_large_mixed_batches_layouts_and_sub_batches(layout):
    datas = []
    for i, (w, h) in enumerate([(1920, 1080), (3840, 2160), (7680, 4320), (1920, 1080), (333, 211)]):
        s = ["420", "422", "444", "gray", "420"][i]
        datas.append(T.encode(big_frame(w, h, i), s, 95, (0, 0, 0, 8, 1)[i], i == 3))
    for cap in (0, 8 << 20):   # one sub-batch; one file per sub-batch
        got, flags = decode_images(datas, layout, cap)
        assert not flags.any()
        for g, d in zip(got, datas):
            want = T.imdecode(d)
            assert np.array_equal(g, want), (layout, cap, g.shape, int((g != want).sum()))


def test_corrupt_data_is_an_error():
    seq = _seq()
    good = T.encode(big_frame(640, 360, 1), "420", 95)
    info = seq.probe(good)
    bad = bytearray(good)
    rng = np.random.default_rng(3)
    lo, hi = info.scan_begin + 100, info.scan_end - 100
    for p in rng.integers(lo, hi, 40):
        bad[p] = 0xFF if bad[p] != 0xFF else 0xFE   # markers inside the data
    got, flags = decode_images([good, bytes(bad)])
    assert flags[0] == 0 and flags[1] != 0
    short = bytearray(good[:info.scan_begin + (info.scan_end - info.scan_begin) // 2]) + b"\xff\xd9"
    _, flags = decode_images([bytes(short)])
    assert flags[0] != 0


def test_kernels_do_not_spill():
    so = os.path.join(os.path.dirname(__file__), "..", "pyscenedetect_b200", "libpsd_b200.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    fn, spills = None, {}
    for line in out.splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
        elif fn and "jd_" in fn and ("LDL" in line or "STL" in line):
            spills[fn] = spills.get(fn, 0) + 1
    assert not spills, spills


def write_seq(tmp, n=40, w=320, h=180, cut_every=9):
    """n frames of w x h with a cut every `cut_every`, written by cv2.imwrite: (pattern, paths)"""
    paths = []
    for i in range(n):
        f = big_frame(w, h, i // cut_every)
        f[(i * 3) % h] = 255 - f[(i * 3) % h]
        p = os.path.join(tmp, f"f_{i:04d}.jpg")
        cv2.imwrite(p, f, [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    return os.path.join(tmp, "f_%04d.jpg"), paths


def _detect(video, batch, crop=None, frame_skip=0):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    sm = SceneManager(StatsManager() if frame_skip == 0 else None, batch_size=batch)
    if crop is not None:
        sm.crop = crop
    sm.add_detector(ContentDetector())
    sm.detect_scenes(video, frame_skip=frame_skip)
    scenes = [(a.frame_num, b.frame_num) for a, b in sm.get_scene_list()]
    if sm.stats_manager is None:   # frame_skip: no StatsManager (the reference refuses the pair)
        return scenes, None
    import io
    buf = io.StringIO()
    sm.stats_manager.save_to_csv(buf)
    return scenes, buf.getvalue()


@pytest.mark.parametrize("batch,crop,frame_skip", [(7, None, 0), (64, None, 0), (64, (10, 20, 300, 170), 0),
                                                   (7, None, 2)])
def test_scene_manager_on_stream_equals_imread_frames(tmp_path, batch, crop, frame_skip):
    from pyscenedetect_b200.video import ArrayVideoStream
    seq = _seq()
    pattern, paths = write_seq(str(tmp_path))
    frames = np.stack([cv2.imread(p) for p in paths])
    got = _detect(seq.ImageSequenceStream(pattern, batch_size=batch), batch, crop, frame_skip)
    want = _detect(ArrayVideoStream(frames, fps=25.0), batch, crop, frame_skip)
    assert got == want


# ---- refusals through the stream ----

def test_stream_raises_for_corrupt_and_mixed_size_files(tmp_path):
    seq = _seq()
    pattern, paths = write_seq(str(tmp_path), n=6)
    good = open(paths[3], "rb").read()
    info = seq.probe(good)
    bad = bytearray(good)
    for p in range(info.scan_begin + 50, info.scan_end - 50, 97):
        bad[p] = 0xFF if bad[p] != 0xFF else 0xFE
    with open(paths[3], "wb") as f:
        f.write(bytes(bad))
    s = seq.ImageSequenceStream(pattern, batch_size=2)
    s.read_batch(2)
    with pytest.raises(ValueError, match="f_0003.jpg"):
        s.read_batch(2)
    cv2.imwrite(paths[3], big_frame(160, 90, 0))
    s.seek(2)
    with pytest.raises(ValueError, match="f_0003.jpg.*160x90"):
        s.read_batch(2)


def test_data_ending_inside_a_block_is_an_error():
    """A scan cut inside its last block's bits: libjpeg-turbo decodes it from zero bits with a warning; the device
    flags it instead of decoding 1-bits"""
    from tests import jpeg_decode_twin as D
    good = T.encode(T.frame("noise", 48, 32), "420", 95)
    info = D.probe(good)
    found = 0
    for cut in range(1, 24):
        data = good[:info.scan1 - cut] + good[info.scan1:]
        try:
            D.coefficients(data)
            continue
        except ValueError as e:
            if "ends inside a block" not in str(e):
                continue
        _, flags = decode_images([data])
        assert flags[0] != 0, cut
        found += 1
    assert found


def test_idct_outside_the_range_limit_band_equals_the_twin():
    """Quantisation tables inflated to 4 and 8 drive the islow IDCT far outside [-384, 384), where range_limit wraps
    (jidctint.c).  The device follows the C code, as the twin does; cv2's build decodes these blocks with its SIMD
    IDCT, which saturates instead, so cv2 gives other bytes for them (DESIGN.md §4.9)."""
    from tests import jpeg_decode_twin as D
    seen = []
    limit = D.range_limit

    def record(x):
        seen.append(int(np.abs(x).max()))
        return limit(x)

    datas = []
    for s in ("444", "420", "gray"):
        for v in (4, 8):
            b = bytearray(T.encode(T.frame("noise", 64, 48), s, 100))
            p = 0
            while (p := b.find(b"\xff\xdb", p)) >= 0:
                L = (b[p + 2] << 8) | b[p + 3]
                for q in range(p + 4, p + 2 + L, 65):
                    b[q + 1:q + 65] = bytes([v]) * 64
                p += 2 + L
            datas.append(bytes(b))
    got, flags = decode_images(datas)
    assert not flags.any()
    D.range_limit = record
    try:
        want = [D.decode(d) for d in datas]
    finally:
        D.range_limit = limit
    assert max(seen) >= 512   # past the clamp band, into the wrap
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


# ---- detect_clips, run_clips and save_images over streams ----

def scene_frame(w, h, scene, i):
    """a frame of scene `scene`: its own colours and stripes, with noise that changes every frame"""
    rng = np.random.default_rng(scene)
    base = rng.integers(0, 256, 3)
    y, x = np.mgrid[:h, :w]
    f = base[None, None, :] + ((x // (4 + scene % 5) + y // 6) % 2 * 90)[..., None]
    f = f + np.random.default_rng(1000 * scene + i).integers(-8, 9, (h, w, 3))
    return f.clip(0, 255).astype(np.uint8)


def _sequences(tmp, n, length, w=96, h=54):
    """n sequences of `length` frames (a new scene every 17 frames), as (paths, imread frames)"""
    out = []
    for k in range(n):
        d = os.path.join(tmp, f"s{k:02d}")
        os.makedirs(d)
        paths = []
        for i in range(length):
            f = scene_frame(w, h, 100 * k + (i + k) // 17, i)
            p = os.path.join(d, f"{i:04d}.jpg")
            cv2.imwrite(p, f, [cv2.IMWRITE_JPEG_QUALITY, 85])
            paths.append(p)
        out.append((paths, np.stack([cv2.imread(p) for p in paths])))
    return out


def test_detect_clips_over_50_sequences_equals_detect_scenes(tmp_path):
    from pyscenedetect_b200.clips import detect_clips
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.scene_manager import SceneManager
    seq = _seq()
    sets = _sequences(str(tmp_path), 50, 40)
    results = detect_clips([seq.ImageSequenceStream(p, batch_size=5) for p, _ in sets], [ContentDetector()],
                           batch_size=16)
    cuts = 0
    for (paths, _), r in zip(sets, results):
        sm = SceneManager(batch_size=16)
        sm.add_detector(ContentDetector())
        sm.detect_scenes(seq.ImageSequenceStream(paths, batch_size=5))
        want = [c.frame_num for c in sm.get_cut_list()]
        assert r.cut_frames == want and r.frames == len(paths)
        cuts += len(want)
    assert cuts > 0


def test_run_clips_counts_equal_imread_frames(tmp_path):
    """Stream batches of 16 under a sweep batch of 64, and frame_skip 3: more than the stream's three batches are read
    between two synchronisations of the engines unless the sweep honours `batches_kept`"""
    from pyscenedetect_b200.detectors import ContentDetector
    from pyscenedetect_b200.sweep import GroundTruth, ParameterSweep
    from pyscenedetect_b200.video import ArrayVideoStream
    seq = _seq()
    sets = _sequences(str(tmp_path), 3, 120)
    gts = [GroundTruth(list(range(17 - k % 17, 120, 17))) for k in range(3)]
    grid = [{"threshold": t} for t in (10.0, 20.0, 27.0, 40.0)]
    tols = (0, 2)
    settings = [{}, {"frame_skip": 3}]
    a = ParameterSweep(ContentDetector, grid, tolerances=tols, batch_size=64, settings=settings)
    ra = a.run_clips([seq.ImageSequenceStream(p, batch_size=16) for p, _ in sets], gts)
    b = ParameterSweep(ContentDetector, grid, tolerances=tols, batch_size=64, settings=settings)
    rb = b.run_clips([ArrayVideoStream(f, 25.0) for _, f in sets], gts)
    found = 0
    for k in range(len(grid) * len(settings)):
        for j in range(len(sets)):
            got = (ra.cuts(k, j), ra.raw_count(k, j), [ra.hard(k, j, t) for t in tols], ra.fades(k, j))
            want = (rb.cuts(k, j), rb.raw_count(k, j), [rb.hard(k, j, t) for t in tols], rb.fades(k, j))
            assert got == want, (k, j)
            found += ra.raw_count(k, j)
    assert found > 0


def test_save_images_from_stream_equals_imread_frames(tmp_path):
    from pyscenedetect_b200.images import save_images
    from pyscenedetect_b200.video import ArrayVideoStream
    seq = _seq()
    (paths, frames), = _sequences(str(tmp_path), 1, 30, 320, 180)
    scenes = [(a, b) for a, b in zip(range(0, 30, 7), list(range(7, 30, 7)) + [30])]
    from pyscenedetect_b200 import FrameTimecode
    scenes = [(FrameTimecode(a, 25.0), FrameTimecode(b, 25.0)) for a, b in scenes]
    tpl = "Scene-$SCENE_NUMBER-$IMAGE_NUMBER"
    got = save_images(scenes, seq.ImageSequenceStream(paths, batch_size=4), output_dir=str(tmp_path / "a"),
                      image_name_template=tpl)
    want = save_images(scenes, ArrayVideoStream(frames, 25.0), output_dir=str(tmp_path / "b"),
                       image_name_template=tpl)
    assert got == want and sum(len(v) for v in got.values()) == 3 * len(scenes)
    for files in got.values():
        for f in files:
            assert (tmp_path / "a" / f).read_bytes() == (tmp_path / "b" / f).read_bytes()
