"""JPEG decoding without a GPU (DESIGN.md section 8.10): tools/jpeg_decode_dump.cu runs the GPU decoder's own parse, Huffman
state machine (with its subsequences and synchronisation rounds emulated), IDCT, upsampling and colour conversion on the
CPU under AddressSanitizer, and every frame equals cv2.imdecode.  Also: corrupt files end in a status, whenet_jpeg_info refuses
each unsupported kind with its reason, and ``video.MJPGReader`` reads back MJPG AVIs."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
cv2 = pytest.importorskip("cv2")
from test_jpeg_cpu import KINDS, SIZES, frame  # noqa: E402

ROOT = os.path.join(os.path.dirname(__file__), "..")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
QUALITIES = [1, 10, 50, 75, 95, 100]
SAMPLINGS = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "gray": None}
SAMPLES = ["mov_001_007585.jpeg", "mov_012_022606.jpeg"]


def encode(img, q, sampling="420", rst=0):
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if sampling == "gray":
        img = np.ascontiguousarray(img[:, :, 1])
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[sampling]]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def imdecode(buf):
    return cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)


def strip_dht(jpeg):
    out, pos = bytearray(jpeg[:2]), 2
    while True:
        marker, length = jpeg[pos + 1], int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        if marker != 0xC4:
            out += jpeg[pos:pos + 2 + length]
        pos += 2 + length
        if marker == 0xDA:
            return bytes(out + jpeg[pos:])


def with_exif(jpeg, orientation, big_endian=False, malformed=False):
    """``jpeg`` with an APP1 Exif block holding one IFD0 entry, the orientation tag, inserted after SOI."""
    e = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 0x2A, 8) + struct.pack(e + "H", 1)
    tiff += struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(e + "I", 0)
    if malformed:
        tiff = tiff[:8] + struct.pack(e + "H", 5) + tiff[10:14]      # five entries announced, the block ends inside the first
    app1 = b"Exif\0\0" + tiff
    return jpeg[:2] + b"\xff\xe1" + struct.pack(">H", len(app1) + 2) + app1 + jpeg[2:]


@pytest.fixture(scope="module")
def dump_tool(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    exe = str(tmp_path_factory.mktemp("dump") / "jpeg_decode_dump")
    src = os.path.join(ROOT, "tools", "jpeg_decode_dump.cu")
    base = [nvcc, "-std=c++17", "-arch=sm_90a", "-O2", "-g", "-o", exe, src]
    r = subprocess.run(base[:-3] + ["-Xcompiler", "-fsanitize=address", "-lasan"] + base[-3:], capture_output=True, text=True)
    if r.returncode != 0:       # a host compiler without AddressSanitizer
        r = subprocess.run(base, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def run_dump(exe, tmp_path, files, bits=2048):
    """One dump run over ``files``: per file ("ok", frame) or ("einval" / "status", text)."""
    args = []
    for i, f in enumerate(files):
        p = tmp_path / ("f%d.jpg" % i)
        p.write_bytes(f)
        args += [str(p), str(tmp_path / ("f%d.bgr" % i))]
    r = subprocess.run([exe, str(bits)] + args, capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stderr[-4000:]
    out = []
    for i, line in enumerate(r.stdout.splitlines()):
        kind, rest = line.split(" ", 1)
        if kind == "ok":
            h, w, _ = (int(v) for v in rest.split())
            out.append(("ok", np.fromfile(str(tmp_path / ("f%d.bgr" % i)), np.uint8).reshape(h, w, 3)))
        else:
            out.append((kind, rest))
    assert len(out) == len(files)
    return out


def assert_equal_cv2(exe, tmp_path, files, bits=2048):
    for i, (res, f) in enumerate(zip(run_dump(exe, tmp_path, files, bits), files)):
        assert res[0] == "ok", (i, res)
        ref = imdecode(f)
        assert res[1].shape == ref.shape and np.array_equal(res[1], ref), (i, ref.shape)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_dump_equals_cv2(dump_tool, tmp_path, sampling):
    files = []
    for h, w in SIZES:
        for q in QUALITIES:
            for k, kind in enumerate(KINDS):
                files.append(encode(frame(kind, h, w, seed=q + k), q, sampling))
    assert_equal_cv2(dump_tool, tmp_path, files)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_dump_equals_cv2_1081x1921(dump_tool, tmp_path, sampling):
    files = [encode(frame("noise", 1081, 1921, seed=3), 95, sampling)]
    assert_equal_cv2(dump_tool, tmp_path, files)


@pytest.mark.parametrize("rst", [1, 4, 7])
def test_dump_restart_intervals(dump_tool, tmp_path, rst):
    files = [encode(frame(kind, h, w, seed=rst), q, s, rst=rst)
             for (h, w) in [(17, 33), (37, 53), (120, 200)] for s in SAMPLINGS for q in [10, 95] for kind in ["noise", "gradient"]]
    assert_equal_cv2(dump_tool, tmp_path, files)


def test_dump_without_dht(dump_tool, tmp_path):
    files = []
    for s in SAMPLINGS:
        f = encode(frame("noise", 37, 53), 75, s)
        g = strip_dht(f)
        assert 0xC4 not in [g[i + 1] for i in range(len(g) - 1) if g[i] == 0xFF][:8]
        assert np.array_equal(imdecode(g), imdecode(f))
        files.append(g)
    assert_equal_cv2(dump_tool, tmp_path, files)


def test_dump_exif_orientation(dump_tool, tmp_path):
    base = encode(frame("gradient", 40, 64), 90)
    files = [with_exif(base, o, be) for o in range(1, 9) for be in (False, True)]
    files += [with_exif(base, 6, malformed=True), with_exif(base, 9), with_exif(base, 0)]
    assert imdecode(files[10]).shape == (64, 40, 3)          # orientation 6
    assert_equal_cv2(dump_tool, tmp_path, files)


def test_dump_reference_samples(dump_tool, tmp_path):
    files = [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    assert [imdecode(f).shape for f in files] == [(224, 528, 3), (226, 548, 3)]
    assert_equal_cv2(dump_tool, tmp_path, files)


@pytest.mark.parametrize("bits", [32, 1000])
def test_dump_short_subsequences(dump_tool, tmp_path, bits):
    files = [encode(frame(kind, 37, 53, seed=1), q, s, rst=r) for kind in ["noise", "gradient"] for q in [10, 95]
             for s in SAMPLINGS for r in [0, 3]]
    files += [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    assert_equal_cv2(dump_tool, tmp_path, files, bits)


def test_dump_corrupt_files_equal_cv2(dump_tool, tmp_path):
    """Seeded byte flips and truncations: each ends in a frame, a status or a refused header, never a sanitizer report, and
    every decoded frame equals cv2's.  Variant 91's flipped byte leaves luma DC values up to 1555 (12440 dequantised) in
    blocks without AC rows, which only the 16-bit IDCT steps of DESIGN.md section 8.10 decode as cv2 does."""
    rng = np.random.default_rng(7)
    bases = [encode(frame("noise", 37, 53), 75), encode(frame("gradient", 64, 80), 50, "422", rst=2),
             encode(frame("noise", 24, 24), 95, "gray"), open(os.path.join(GOLDEN, SAMPLES[0]), "rb").read()]
    files = []
    for k in range(300):
        b = bytearray(bases[k % len(bases)])
        if k % 3 == 2:
            b = b[:int(rng.integers(2, len(b)))]
        else:
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(2, len(b)))] = int(rng.integers(0, 256))
        files.append(bytes(b))
    kinds, ok, differ = set(), 0, []
    for k, (res, f) in enumerate(zip(run_dump(dump_tool, tmp_path, files, bits=64), files)):
        kinds.add(res[0])
        if res[0] == "ok":
            ref = imdecode(f)
            ok += 1
            if ref is None or not np.array_equal(res[1], ref):
                differ.append(k)
    assert {"status", "ok", "einval"} <= kinds
    assert ok == 66 and differ == [], (ok, differ)


def fill_and_trailing_segments(jpeg):
    """``jpeg`` (with restart markers) with 0xFF fill bytes before two RSTn and COM / APP3 segments between the data and EOI:
    all legal, and cv2 decodes the same pixels."""
    assert jpeg.endswith(b"\xff\xd9") and b"\xff\xd1" in jpeg
    f = jpeg.replace(b"\xff\xd0", b"\xff\xff\xff\xd0", 1).replace(b"\xff\xd1", b"\xff\xff\xd1", 1)
    return f[:-2] + b"\xff\xfe\x00\x05abc\xff\xe3\x00\x02\xff\xd9"


def test_dump_fill_bytes_and_trailing_segments(dump_tool, tmp_path):
    files = [fill_and_trailing_segments(encode(frame("noise", 64, 80), 75, s, rst=2)) for s in SAMPLINGS]
    assert_equal_cv2(dump_tool, tmp_path, files)


# ---------------------------------------------------------------------------------------------------- numpy oracle
def _oracle_equals_cv2(files):
    import jpeg_decode_oracle as O
    for i, f in enumerate(files):
        got, ref = O.decode(f), imdecode(f)
        assert got.shape == ref.shape and np.array_equal(got, ref), (i, ref.shape)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_oracle_equals_cv2(sampling):
    _oracle_equals_cv2([encode(frame(KINDS[(q + r) % 4], h, w, seed=q), q, sampling, rst=r)
                        for h, w in SIZES for q in (1, 50, 100) for r in (0, 3)])


def test_oracle_fixtures_exif_no_dht_fill():
    base = encode(frame("gradient", 40, 64), 90)
    files = [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    files += [with_exif(base, o, be) for o in range(1, 9) for be in (False, True)] + [with_exif(base, 6, malformed=True)]
    files += [strip_dht(encode(frame("noise", 37, 53), 75, s)) for s in SAMPLINGS]
    files += [encode(frame("noise", 37, 53), q, s, rst=r) for s in SAMPLINGS for q in (10, 95) for r in (1, 4, 7)]
    files += [fill_and_trailing_segments(encode(frame("noise", 64, 80), 75, s, rst=2)) for s in SAMPLINGS]
    _oracle_equals_cv2(files)


def test_oracle_refusals():
    import jpeg_decode_oracle as O
    img = frame("noise", 32, 48)
    for params, why in [([cv2.IMWRITE_JPEG_PROGRESSIVE, 1], "progressive"),
                        ([cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440], "sampling")]:
        with pytest.raises(ValueError, match=why):
            O.decode(cv2.imencode(".jpg", img, params)[1].tobytes())


# ---------------------------------------------------------------------------------------------------- header checks
def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def _info(data):
    from whenet_b200 import video
    return video.jpeg_info(data)


def _patch_sof(jpeg, fn):
    pos = 2
    while True:
        marker, length = jpeg[pos + 1], int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        if marker in (0xC0, 0xC1):
            b = bytearray(jpeg)
            fn(b, pos)
            return bytes(b)
        pos += 2 + length


def _strip_app0(jpeg):
    assert jpeg[2:4] == b"\xff\xe0"
    return jpeg[:2] + jpeg[4 + int.from_bytes(jpeg[4:6], "big"):]


def test_info_sizes():
    f = encode(frame("noise", 37, 53), 75)
    assert _info(f) == (37, 53)
    assert _info(with_exif(f, 6)) == (53, 37)
    assert _info(encode(frame("noise", 5, 9), 75, "gray")) == (5, 9)


def test_info_refusals():
    img = frame("noise", 32, 48)
    base = encode(img, 75)

    def sof_byte(off, v):
        return _patch_sof(base, lambda b, p: b.__setitem__(p + 4 + off, v))

    def rgb_ids(b, p):
        for c, ch in enumerate(b"RGB"):
            b[p + 10 + 3 * c] = ch
    rgb = _strip_app0(_patch_sof(base, rgb_ids))
    sos = rgb.index(b"\xff\xda")
    rgb = bytearray(rgb)
    for c, ch in enumerate(b"RGB"):
        rgb[sos + 5 + 2 * c] = ch
    cases = [
        (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), "progressive"),
        (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])[1].tobytes(), "sampling"),
        (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])[1].tobytes(), "sampling"),
        (_patch_sof(base, lambda b, p: b.__setitem__(p + 1, 0xC9)), "arithmetic"),
        (sof_byte(0, 12), "12-bit"),
        (sof_byte(5, 4), "components"),
        (sof_byte(5, 2), "components"),
        (bytes(rgb), "RGB"),
        (b"\x00\x01", "SOI"),
        (base[:40], "truncated"),
        (_patch_sof(base, lambda b, p: (b.__setitem__(p + 5, 0), b.__setitem__(p + 6, 0))), "DNL"),
    ]
    for data, why in cases:
        with pytest.raises(ValueError, match=why):
            _info(data)
        hw = (C.c_int32 * 2)()
        msg = C.create_string_buffer(128)
        assert _lib().whenet_jpeg_info(data, len(data), hw, msg, 128) == -1
        assert why.encode() in msg.value


def test_decode_argument_checks():
    """Refused with EINVAL before any device work, without a context."""
    from whenet_b200 import video
    L = _lib()
    f = encode(frame("noise", 8, 8), 75)
    buf = C.create_string_buffer(f, len(f))
    files = (C.c_void_p * 1)(C.addressof(buf))
    sizes = (C.c_int64 * 1)(len(f))
    outs = (C.c_void_p * 1)(1234)
    assert L.whenet_decode_jpeg_u8(None, files, sizes, 0, outs, None) == -1
    assert L.whenet_decode_jpeg_u8(None, files, sizes, 65, outs, None) == -1
    assert L.whenet_decode_jpeg_u8(None, None, sizes, 1, outs, None) == -1
    assert L.whenet_decode_jpeg_u8(None, files, sizes, 1, outs, None) == -1      # well-formed: the null context is refused
    assert b"null context" in L.whenet_last_error()
    bad = C.create_string_buffer(b"\xff\xd8\xff\xc2\x00\x02", 6)
    bad_files = (C.c_void_p * 1)(C.addressof(bad))
    assert L.whenet_decode_jpeg_u8(None, bad_files, (C.c_int64 * 1)(6), 1, outs, None) == -1
    assert b"file 0: progressive" in L.whenet_last_error()
    assert L.whenet_debug_jpeg_piece_bits(None, 16) == -1
    for arg in [b"abc", [f, 3], "x"]:
        with pytest.raises(ValueError):
            video.decode_jpeg(None, arg)
    with pytest.raises(ValueError, match="file 1: progressive"):
        video.decode_jpeg(None, [f, cv2.imencode(".jpg", frame("noise", 8, 8), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()])
    assert video.decode_jpeg(None, []) == []


# ---------------------------------------------------------------------------------------------------- MJPGReader
def _jpegs(n, h=24, w=40, q=80):
    return [encode(frame("noise", h, w, seed=i), q) for i in range(n)]


def _check_reader(path, jpegs, fps, size):
    from whenet_b200 import video
    with video.MJPGReader(path) as r:
        assert len(r) == len(jpegs)
        assert r.frame_size == size
        assert abs(r.fps - fps) < 1e-6 * fps
        got = []
        while (chunk := r.read(3)):
            got += chunk
        assert r.read(3) == []
    assert [g.rstrip(b"\0") for g in got] == [j.rstrip(b"\0") for j in jpegs]


def test_reader_writer_files(tmp_path):
    from whenet_b200 import video
    jpegs = _jpegs(7)
    p = str(tmp_path / "a.avi")
    with video.MJPGWriter(p, 29.97, (40, 24)) as w:
        w.write(jpegs)
    _check_reader(p, jpegs, 29.97, (40, 24))


def test_reader_opendml_segments(tmp_path, monkeypatch):
    from whenet_b200 import video
    jpegs = _jpegs(11)
    monkeypatch.setattr(video, "SEGMENT_LIMIT", 3 * max(len(j) for j in jpegs))
    p = str(tmp_path / "s.avi")
    with video.MJPGWriter(p, 25, (40, 24)) as w:
        w.write(jpegs)
    assert open(p, "rb").read().count(b"AVIX") >= 3
    _check_reader(p, jpegs, 25, (40, 24))


@pytest.mark.parametrize("backend", ["CAP_FFMPEG", "CAP_OPENCV_MJPEG"])
def test_reader_cv2_files(tmp_path, backend):
    from whenet_b200 import video
    p = str(tmp_path / "c.avi")
    frames = [frame("gradient", 48, 64, seed=i) for i in range(5)]
    w = cv2.VideoWriter(p, getattr(cv2, backend), cv2.VideoWriter_fourcc(*"MJPG"), 15, (64, 48))
    if not w.isOpened():
        pytest.skip("cv2 backend %s cannot write" % backend)
    for f in frames:
        w.write(f)
    w.release()
    with video.MJPGReader(p) as r:
        assert len(r) == 5 and r.frame_size == (64, 48) and abs(r.fps - 15) < 1e-6
        files = r.read(10)
    # cv2's readers decode through FFmpeg, not libjpeg: check the chunks are the stream's baseline JPEG frames
    assert len(files) == 5
    for f in files:
        assert video.jpeg_size(f) == (64, 48) and imdecode(f).shape == (48, 64, 3)


def test_reader_without_index_and_truncated(tmp_path):
    from whenet_b200 import video
    jpegs = _jpegs(5)
    p = str(tmp_path / "a.avi")
    with video.MJPGWriter(p, 10, (40, 24)) as w:
        w.write(jpegs)
    data = bytearray(open(p, "rb").read())
    for tag in (b"idx1", b"indx", b"ix00"):           # rename every index so that only the movi walk remains
        i = data.find(tag)
        while i >= 0:
            data[i:i + 4] = b"JUNK"
            i = data.find(tag, i + 4)
    q = tmp_path / "noindex.avi"
    q.write_bytes(bytes(data))
    _check_reader(str(q), jpegs, 10, (40, 24))
    # cut inside the last frame: that frame is not returned
    movi = data.find(b"movi")
    last = data.rfind(b"00dc", 0, data.find(b"JUNK", movi))       # the last frame chunk, before the renamed ix00
    t = tmp_path / "trunc.avi"
    t.write_bytes(bytes(data[:last + 8 + 10]))
    _check_reader(str(t), jpegs[:-1], 10, (40, 24))
    with pytest.raises(ValueError, match="not a RIFF AVI"):
        video.MJPGReader(__file__)
