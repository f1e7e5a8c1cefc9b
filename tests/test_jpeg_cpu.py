"""JPEG encoding and the MJPG AVI writer without a GPU (DESIGN.md section 8.9): oracle/jpeg_oracle.py equals cv2.imencode as a
whole file, the library's header bytes (whenet_debug_jpeg_header) equal cv2's for every quality, ``video.MJPGWriter``'s files
read back through cv2 and walk as RIFF, and the argument checks."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(__file__), "..")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
cv2 = pytest.importorskip("cv2")

import jpeg_oracle as J  # noqa: E402

EINVAL = -1         # WHENET_EINVAL
SIZES = [(1, 1), (1, 17), (17, 1), (7, 15), (8, 8), (15, 7), (16, 16), (17, 33), (37, 53), (120, 200), (224, 224)]
QUALITIES = [1, 10, 49, 50, 51, 75, 94, 95, 100]
KINDS = ["noise", "gradient", "constant", "extremes"]


def frame(kind, h, w, seed=0):
    """BGR test content: uniform noise (many 0xFF bytes to stuff), gradients (long zero runs, ZRL, EOB), a constant colour,
    and 0/255 channel extremes (large DC differences, saturated chroma)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(xx * 3 + yy + seed) % 256, (yy * 5) % 256, (xx + 2 * yy) % 256], -1).astype(np.uint8)
    if kind == "constant":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    return (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)


def cv2_jpeg(img, q):
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return buf.tobytes()


def _sos_end(jpeg):
    """Length of everything up to and including the SOS segment."""
    pos = 2
    while True:
        marker, length = jpeg[pos + 1], int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        pos += 2 + length
        if marker == 0xDA:
            return pos


@pytest.mark.parametrize("h,w", SIZES)
def test_oracle_equals_cv2(h, w):
    for q in QUALITIES:
        for k, kind in enumerate(KINDS):
            img = frame(kind, h, w, seed=q + k)
            assert J.encode(img, q) == cv2_jpeg(img, q), (h, w, q, kind)


def test_oracle_equals_cv2_on_sample_crops(sample_crops):
    for q in QUALITIES:
        for img in sample_crops:
            assert J.encode(np.ascontiguousarray(img), q) == cv2_jpeg(img, q), q


@pytest.mark.parametrize("kind,q", [("noise", 95), ("gradient", 1), ("extremes", 100)])
def test_oracle_equals_cv2_1081x1921(kind, q):
    img = frame(kind, 1081, 1921, seed=3)
    assert J.encode(img, q) == cv2_jpeg(img, q)


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def _header(L, h, w, q):
    buf = np.zeros(1024, np.uint8)
    n = C.c_int()
    rc = L.whenet_debug_jpeg_header(h, w, q, buf.ctypes.data, buf.size, C.byref(n))
    assert rc == 0, L.whenet_last_error()
    return buf[:n.value].tobytes()


@pytest.mark.parametrize("h,w", SIZES + [(1081, 1921), (16384, 24), (24, 16384), (16384, 16384)])
def test_library_header_equals_cv2(h, w):
    L = _lib()
    img = frame("gradient", min(h, 64), min(w, 64))
    for q in range(1, 101):
        got = _header(L, h, w, q)
        assert got == J.header(h, w, q), (h, w, q)
        if (h, w) == img.shape[:2]:
            ref = cv2_jpeg(img, q)
            assert got == ref[:_sos_end(ref)], (h, w, q)
        else:   # cv2 at full size only for a few qualities: the header depends on the size through SOF0 alone
            if q in (1, 50, 95, 100):
                big = np.zeros((h, w, 3), np.uint8)
                ref = cv2_jpeg(big, q)
                assert got == ref[:_sos_end(ref)], (h, w, q)


def test_library_argument_checks():
    """Every bad argument is refused with WHENET_EINVAL before the (here NULL) context is looked at."""
    L = _lib()
    buf = np.zeros(1024, np.uint8)
    n = C.c_int()
    for h, w, q, cap in [(0, 8, 95, 1024), (8, 16385, 95, 1024), (8, 8, 0, 1024), (8, 8, 101, 1024), (8, 8, 95, 622)]:
        assert L.whenet_debug_jpeg_header(h, w, q, buf.ctypes.data, cap, C.byref(n)) == EINVAL
    data = C.c_void_p()
    offs = np.zeros(66, np.int64)
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    for nn, h, w, q in [(0, 8, 8, 95), (65, 8, 8, 95), (1, 0, 8, 95), (1, 8, 16385, 95), (1, 8, 8, 0), (1, 8, 8, 101)]:
        rc = L.whenet_encode_jpeg_u8(None, frames.ctypes.data, nn, h, w, 0, q, C.byref(data), offs.ctypes.data)
        assert rc == EINVAL
        assert b"null context" not in L.whenet_last_error(), (nn, h, w, q)
    assert L.whenet_encode_jpeg_u8(None, frames.ctypes.data, 1, 8, 8, 0, 95, C.byref(data), offs.ctypes.data) == EINVAL
    assert b"null context" in L.whenet_last_error()
    hw = np.array([[8, 8], [16385, 8]], np.int32)
    ptrs = (C.c_void_p * 2)(frames.ctypes.data, frames.ctypes.data)
    assert L.whenet_encode_jpeg_ragged_u8(None, C.addressof(ptrs), hw.ctypes.data, 2, 0, 95, C.byref(data), offs.ctypes.data) == EINVAL
    assert b"frame 1" in L.whenet_last_error()
    ptrs = (C.c_void_p * 2)(frames.ctypes.data, None)
    hw[1] = 8
    assert L.whenet_encode_jpeg_ragged_u8(None, C.addressof(ptrs), hw.ctypes.data, 2, 0, 95, C.byref(data), offs.ctypes.data) == EINVAL
    assert b"frame 1 is NULL" in L.whenet_last_error()


# ----------------------------------------------------------------------------------------------------------------- AVI
def riff_walk(path):
    """Every chunk of an AVI file as (path of list types, fourcc, file offset of the data, size)."""
    out = []
    with open(path, "rb") as f:
        data = f.read()

    def walk(pos, end, where):
        while pos < end:
            cc, size = data[pos:pos + 4], struct.unpack("<I", data[pos + 4:pos + 8])[0]
            if cc in (b"RIFF", b"LIST"):
                kind = data[pos + 8:pos + 12]
                out.append((where, cc + kind, pos + 12, size - 4))
                walk(pos + 12, pos + 8 + size, where + (kind,))
            else:
                out.append((where, cc, pos + 8, size))
            pos += 8 + size + (size & 1)
        assert pos == end, (pos, end)

    walk(0, len(data), ())
    return out, data


def _jpegs(n, h, w, q=95):
    return [cv2_jpeg(frame("noise" if i % 2 else "gradient", h, w, seed=i), q) for i in range(n)]


def _check_file(path, jpegs, fps, h, w, segments):
    """The RIFF walk finds every frame unchanged in order, each segment's ix00 and the super index point at them, and
    idx1 covers the first segment."""
    chunks, data = riff_walk(path)
    riffs = [c for c in chunks if c[0] == ()]
    assert [c[1] for c in riffs] == [b"RIFFAVI "] + [b"RIFFAVIX"] * (segments - 1)
    frames = [c for c in chunks if c[1] == b"00dc"]
    assert len(frames) == len(jpegs)
    for (_, _, off, size), j in zip(frames, jpegs):
        assert data[off:off + size] == j
    avih = next(c for c in chunks if c[1] == b"avih")
    strh = next(c for c in chunks if c[1] == b"strh")
    dmlh = next(c for c in chunks if c[1] == b"dmlh")
    strf = next(c for c in chunks if c[1] == b"strf")
    assert struct.unpack("<I", data[dmlh[2]:dmlh[2] + 4])[0] == len(jpegs)
    assert struct.unpack("<I", data[strh[2] + 32:strh[2] + 36])[0] == len(jpegs)
    assert data[strh[2]:strh[2] + 8] == b"vidsMJPG" and data[strf[2] + 16:strf[2] + 20] == b"MJPG"
    assert struct.unpack("<II", data[avih[2] + 32:avih[2] + 40]) == (w, h)
    scale, rate = struct.unpack("<II", data[strh[2] + 20:strh[2] + 28])
    assert abs(rate / scale - fps) < 1e-6
    # standard indexes: one ix00 per segment, entries point at chunk data relative to the base offset
    ix = [c for c in chunks if c[1] == b"ix00"]
    assert len(ix) == segments
    seen = []
    for _, _, off, size in ix:
        longs, sub, typ, nent, cid, base = struct.unpack("<HBBI4sQ", data[off:off + 20])
        assert (longs, sub, typ, cid) == (2, 0, 1, b"00dc")
        for e in range(nent):
            rel, sz = struct.unpack("<II", data[off + 24 + 8 * e:off + 32 + 8 * e])
            seen.append((base + rel, sz))
    assert seen == [(c[2], c[3]) for c in frames]
    indx = next(c for c in chunks if c[1] == b"indx")
    nent = struct.unpack("<I", data[indx[2] + 4:indx[2] + 8])[0]
    entries = [struct.unpack("<QII", data[indx[2] + 24 + 16 * e:indx[2] + 40 + 16 * e]) for e in range(nent)]
    assert [(o, s) for o, s, _ in entries] == [(c[2] - 8, c[3] + 8) for c in ix]
    assert sum(d for _, _, d in entries) == len(jpegs)
    idx1 = next(c for c in chunks if c[1] == b"idx1")
    movi = next(c for c in chunks if c[1] == b"LISTmovi")
    first = [c for c in frames if c[0][0] == b"AVI "]
    assert idx1[3] == 16 * len(first)
    for e, c in enumerate(first):
        cid, flags, rel, sz = struct.unpack("<4sIII", data[idx1[2] + 16 * e:idx1[2] + 16 * e + 16])
        assert (cid, flags, sz) == (b"00dc", 0x10, c[3]) and movi[2] - 4 + rel == c[2] - 8


def _read_all(path, backend):
    cap = cv2.VideoCapture(path, backend)
    assert cap.isOpened()
    props = (cap.get(cv2.CAP_PROP_FRAME_COUNT), cap.get(cv2.CAP_PROP_FPS), cap.get(cv2.CAP_PROP_FRAME_WIDTH), cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    out = []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        out.append(img)
    cap.release()
    return props, out


@pytest.mark.parametrize("h,w,n,fps", [(37, 53, 7, 25), (120, 200, 3, 30), (1, 1, 2, 12.5), (17, 33, 4, 29.97)])
def test_writer_reads_back(tmp_path, h, w, n, fps):
    from whenet_b200 import video
    jpegs = _jpegs(n, h, w)
    path = str(tmp_path / "out.avi")
    with video.MJPGWriter(path, fps, (w, h)) as wr:
        wr.write(jpegs[:1])
        wr.write(jpegs[1])
        wr.write(jpegs[2:])
    _check_file(path, jpegs, fps, h, w, 1)
    (count, got_fps, gw, gh), frames = _read_all(path, cv2.CAP_OPENCV_MJPEG)
    assert (count, gw, gh) == (n, w, h) and abs(got_fps - fps) < 1e-3
    assert len(frames) == n
    for img, j in zip(frames, jpegs):
        assert np.array_equal(img, cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR))


def test_writer_opendml_segments(tmp_path, monkeypatch):
    """With the segment limit lowered to a few frames the file continues in RIFF AVIX segments.  cv2's built-in MJPEG reader
    follows only the first RIFF's idx1, so the whole file is read through the FFMPEG backend, whose every frame must equal
    its decode of the same JPEG on its own."""
    from whenet_b200 import video
    h, w, n = 37, 53, 11
    jpegs = _jpegs(n, h, w)
    monkeypatch.setattr(video, "SEGMENT_LIMIT", 3 * max(len(j) for j in jpegs))
    path = str(tmp_path / "seg.avi")
    with video.MJPGWriter(path, 25, (w, h)) as wr:
        wr.write(jpegs)
    chunks, _ = riff_walk(path)
    segments = sum(1 for c in chunks if c[0] == ())
    assert segments >= 4
    _check_file(path, jpegs, 25, h, w, segments)
    (count, fps, gw, gh), frames = _read_all(path, cv2.CAP_FFMPEG)
    assert (count, fps, gw, gh) == (n, 25, w, h) and len(frames) == n
    for i, (img, j) in enumerate(zip(frames, jpegs)):
        one = str(tmp_path / ("%d.jpg" % i))
        with open(one, "wb") as f:
            f.write(j)
        _, ref = _read_all(one, cv2.CAP_FFMPEG)
        assert np.array_equal(img, ref[0]), i
    # the first segment alone is a plain AVI: cv2's reader finds its frames exactly
    first = sum(1 for c in chunks if c[1] == b"00dc" and c[0][0] == b"AVI ")
    _, frames = _read_all(path, cv2.CAP_OPENCV_MJPEG)
    assert len(frames) == first
    for img, j in zip(frames, jpegs):
        assert np.array_equal(img, cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR))


def test_writer_argument_checks(tmp_path):
    from whenet_b200 import video
    path = str(tmp_path / "bad.avi")
    for fps, size in [(0, (8, 8)), (-1, (8, 8)), (float("nan"), (8, 8)), (25, (0, 8)), (25, (8,)), (25, (70000, 8))]:
        with pytest.raises(ValueError):
            video.MJPGWriter(path, fps, size)
    good = _jpegs(1, 8, 16)[0]
    with video.MJPGWriter(path, 25, (16, 8)) as wr:
        with pytest.raises(ValueError):
            wr.write([good, _jpegs(1, 16, 8)[0]])          # transposed size: nothing of the call is written
        with pytest.raises(ValueError):
            wr.write(good[2:])                              # no SOI
        with pytest.raises(ValueError):
            wr.write([good, "not bytes"])
        with pytest.raises(ValueError):
            wr.write(b"\xff\xd8\xff\xd9")                   # no SOF0
        wr.write(good)
    _check_file(path, [good], 25, 8, 16, 1)
    with pytest.raises(ValueError):
        wr.write(good)


def test_jpeg_size():
    from whenet_b200 import video
    assert video.jpeg_size(J.encode(frame("noise", 17, 33), 50)) == (33, 17)
    assert video.jpeg_size(b"") is None and video.jpeg_size(b"\xff\xd8") is None
