"""JPEG encoding options without a GPU (DESIGN.md section 8.11): the oracle equals cv2.imencode with the sampling, restart,
optimise and luma/chroma-quality parameters and on gray images; the library's headers equal cv2's up to SOS; the host and
oracle optimal-table builders agree on synthetic histograms; MJPG files of every kind pass through the writer and reader; and
the argument checks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
cv2 = pytest.importorskip("cv2")
from test_jpeg_cpu import EINVAL, KINDS, _sos_end, frame  # noqa: E402

import jpeg_options_oracle as J  # noqa: E402

SIZES = [(1, 1), (1, 17), (17, 1), (7, 15), (15, 7), (17, 33), (37, 53), (120, 200)]
SAMPLINGS = ["420", "422", "444", "gray"]
# (quality, restart interval, optimize): a covering subset of qualities 1, 50, 95, 100 x restarts 0, 1, 3, more than the MCUs
OPTION_SETS = [(95, 0, False), (1, 1, True), (50, 3, False), (100, 65535, True), (95, 1, False), (50, 0, True), (100, 3, True),
               (1, 0, False)]


def cv2_params(quality=95, sampling="420", restart_interval=0, optimize=False, chroma_quality=None):
    """The cv2.imencode parameters that ``video.encode_jpeg(..., quality, sampling=, restart_interval=, optimize=,
    chroma_quality=)`` equals."""
    if chroma_quality is not None and chroma_quality != quality:
        p = [cv2.IMWRITE_JPEG_LUMA_QUALITY, quality, cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma_quality]
    else:
        p = [cv2.IMWRITE_JPEG_QUALITY, quality]
    p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)]
    if restart_interval:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart_interval]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    return p


def cv2_file(img, **opts):
    """cv2's file of a BGR (H, W, 3) or gray (H, W, 1) image."""
    if img.ndim == 3 and img.shape[2] == 1:
        img = img[..., 0]
    ok, buf = cv2.imencode(".jpg", img, cv2_params(**opts))
    assert ok
    return buf.tobytes()


def option_image(kind, h, w, sampling, seed=0):
    """A BGR test frame, or its G channel as an (h, w, 1) gray frame for sampling "gray"."""
    img = frame(kind, h, w, seed=seed)
    return np.ascontiguousarray(img[..., 1:2]) if sampling == "gray" else img


def oracle_file(img, **opts):
    opts = dict(opts)
    q = opts.pop("quality", 95)
    s = opts.pop("sampling", "420")
    return J.encode_ex(img[..., 0] if img.shape[2] == 1 else img, q, s, opts.get("restart_interval", 0),
                       opts.get("optimize", False), opts.get("chroma_quality"))


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_oracle_equals_cv2(h, w, sampling):
    for k, kind in enumerate(KINDS):
        for q, r, o in OPTION_SETS:
            img = option_image(kind, h, w, sampling, seed=q + k)
            s = "420" if sampling == "gray" else sampling
            opts = dict(quality=q, sampling=s, restart_interval=r, optimize=o)
            assert oracle_file(img, **opts) == cv2_file(img, **opts), (kind, opts)


@pytest.mark.parametrize("q,cq", [(90, 40), (40, 90), (1, 100), (100, 1)])
def test_oracle_equals_cv2_two_qualities(q, cq):
    for h, w in [(7, 15), (37, 53), (120, 200)]:
        for o in (False, True):
            img = frame("noise", h, w, seed=q)
            opts = dict(quality=q, sampling="444", optimize=o, chroma_quality=cq)
            assert oracle_file(img, **opts) == cv2_file(img, **opts), (h, w, opts)


def test_cv2_parameter_semantics():
    """What the option mapping relies on: LUMA_QUALITY alone is QUALITY, CHROMA_QUALITY alone is ignored, two different
    qualities force 4:4:4, a gray image ignores SAMPLING_FACTOR, RST_INTERVAL 0 is no parameter."""
    img = frame("noise", 37, 53)
    base = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 70])[1].tobytes()
    assert cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 20, cv2.IMWRITE_JPEG_LUMA_QUALITY, 70])[1].tobytes() == base
    assert cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 70, cv2.IMWRITE_JPEG_CHROMA_QUALITY, 20])[1].tobytes() == base
    assert cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 70, cv2.IMWRITE_JPEG_RST_INTERVAL, 0])[1].tobytes() == base
    two = [cv2.IMWRITE_JPEG_LUMA_QUALITY, 70, cv2.IMWRITE_JPEG_CHROMA_QUALITY, 20]
    assert cv2.imencode(".jpg", img, two)[1].tobytes() == J.encode_ex(img, 70, "444", chroma_quality=20)
    g = np.ascontiguousarray(img[..., 0])
    assert (cv2.imencode(".jpg", g, [cv2.IMWRITE_JPEG_QUALITY, 70, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                     cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444])[1].tobytes() == J.encode_ex(g, 70))


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("kind,q,r,o", [("noise", 95, 0, False), ("gradient", 1, 1, True), ("extremes", 100, 3, True)])
def test_oracle_equals_cv2_1081x1921(sampling, kind, q, r, o):
    img = option_image(kind, 1081, 1921, sampling, seed=3)
    opts = dict(quality=q, sampling="420" if sampling == "gray" else sampling, restart_interval=r, optimize=o)
    assert oracle_file(img, **opts) == cv2_file(img, **opts)


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def _opts(quality=95, sampling="420", restart_interval=0, optimize=False, chroma_quality=None):
    from whenet_b200._lib import JpegOptions
    return JpegOptions(quality, quality if chroma_quality is None else chroma_quality, int(sampling), restart_interval, int(optimize))


def _header_ex(L, h, w, channels, **opts):
    buf = np.zeros(1024, np.uint8)
    n = C.c_int()
    o = _opts(**opts)
    rc = L.whenet_debug_jpeg_header_ex(h, w, channels, C.byref(o), buf.ctypes.data, buf.size, C.byref(n))
    assert rc == 0, L.whenet_last_error()
    return buf[:n.value].tobytes()


@pytest.mark.parametrize("h,w", SIZES + [(1081, 1921), (16384, 24), (24, 16384), (16384, 16384)])
def test_library_header_equals_cv2(h, w):
    L = _lib()
    small = (h, w) == (min(h, 64), min(w, 64))
    cases = [(s, q, r, None) for s in SAMPLINGS for q in (1, 50, 95, 100) for r in (0, 1, 3, 65535)]
    cases += [("444", 90, 0, 40), ("444", 40, 90, 90), ("444", 1, 7, 100)]
    for s, q, r, cq in cases:
        channels = 1 if s == "gray" else 3
        ss = "420" if s == "gray" else s
        opts = dict(quality=q, sampling=ss, restart_interval=r, chroma_quality=cq)
        got = _header_ex(L, h, w, channels, **opts)
        assert got == J.header_ex(h, w, q, cq, ss, channels, r), (s, opts)
        if small or (q in (1, 95) and r in (0, 3)):
            img = np.zeros((h, w, channels), np.uint8)
            ref = cv2_file(img, **opts)
            assert got == ref[:_sos_end(ref)], (s, opts)


def fib_counts():
    c = np.zeros(256, np.int64)
    a, b = 1, 1
    for i in range(40):
        c[i] = a
        a, b = b, a + b
    return c


HISTOGRAMS = {
    "one symbol": np.eye(1, 256, 7, dtype=np.int64)[0] * 1000,
    "all equal": np.full(256, 5, np.int64),
    "ties": np.array([3, 3, 1, 1, 2, 2, 0, 7] * 32, np.int64),
    "two symbols": np.eye(1, 256, 0, dtype=np.int64)[0] + np.eye(1, 256, 255, dtype=np.int64)[0],
    "fibonacci, codes past 16 bits": fib_counts(),
    "eob-heavy": np.r_[[10 ** 6], np.arange(1, 256) % 17].astype(np.int64),
}


def optimal_table(L, counts, gpu_ctx=None):
    bits = np.zeros(16, np.uint8)
    vals = np.zeros(256, np.uint8)
    nv = C.c_int()
    c32 = np.ascontiguousarray(counts, np.int32)
    if gpu_ctx is None:
        rc = L.whenet_debug_jpeg_optimal_table(c32.ctypes.data, bits.ctypes.data, vals.ctypes.data, C.byref(nv))
    else:
        rc = L.whenet_debug_jpeg_optimal_table_gpu(gpu_ctx, c32.ctypes.data, bits.ctypes.data, vals.ctypes.data, C.byref(nv))
    assert rc == 0, L.whenet_last_error()
    return bits.tolist(), vals[:nv.value].tolist()


@pytest.mark.parametrize("name", sorted(HISTOGRAMS))
def test_optimal_table_equals_oracle(name):
    counts = HISTOGRAMS[name]
    bits, vals = J.gen_optimal_table(counts)
    assert optimal_table(_lib(), counts) == (bits, vals)
    assert sum(bits) == len(vals) == int(np.count_nonzero(counts))
    if name.startswith("fibonacci"):
        # the raw Huffman tree is deeper than 16: only the length-limiting adjustment brings it to 16 bits
        assert bits[15] > 0


def test_optimal_table_argument_checks():
    L = _lib()
    c = np.zeros(256, np.int32)
    out = np.zeros(256, np.uint8)
    nv = C.c_int()
    assert L.whenet_debug_jpeg_optimal_table(None, out.ctypes.data, out.ctypes.data, C.byref(nv)) == EINVAL
    c[3] = -1
    assert L.whenet_debug_jpeg_optimal_table(c.ctypes.data, out.ctypes.data, out.ctypes.data, C.byref(nv)) == EINVAL
    c[3] = 1
    assert L.whenet_debug_jpeg_optimal_table_gpu(None, c.ctypes.data, out.ctypes.data, out.ctypes.data, C.byref(nv)) == EINVAL
    assert b"null context" in L.whenet_last_error()


def test_library_argument_checks():
    """Every bad option is refused with WHENET_EINVAL before the (here NULL) context is looked at."""
    L = _lib()
    data = C.c_void_p()
    offs = np.zeros(66, np.int64)
    frames = np.zeros((8, 8, 3), np.uint8)
    ptrs = (C.c_void_p * 1)(frames.ctypes.data)
    hw = np.array([[8, 8]], np.int32)
    bad = [(3, dict(quality=0)), (3, dict(quality=101)), (3, dict(chroma_quality=0)), (3, dict(chroma_quality=101)),
           (3, dict(sampling="411")), (3, dict(restart_interval=-1)), (3, dict(restart_interval=65536)),
           (3, dict(optimize=2)), (3, dict(chroma_quality=40)), (3, dict(sampling="422", chroma_quality=40)),
           (1, dict(sampling="444")), (1, dict(chroma_quality=40)), (2, {}), (4, {})]
    for channels, kw in bad:
        o = _opts(**{k: v for k, v in kw.items() if k != "optimize"})
        if "optimize" in kw:
            o.optimize = kw["optimize"]
        rc = L.whenet_encode_jpeg_ex_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, channels, 0, C.byref(o), C.byref(data), offs.ctypes.data)
        assert rc == EINVAL, (channels, kw)
        assert b"null context" not in L.whenet_last_error(), (channels, kw)
        buf = np.zeros(1024, np.uint8)
        n = C.c_int()
        assert L.whenet_debug_jpeg_header_ex(8, 8, channels, C.byref(o), buf.ctypes.data, buf.size, C.byref(n)) == EINVAL
    o = _opts()
    assert L.whenet_encode_jpeg_ex_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, 3, 0, None, C.byref(data), offs.ctypes.data) == EINVAL
    assert L.whenet_encode_jpeg_ex_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, 3, 0, C.byref(o), C.byref(data), offs.ctypes.data) == EINVAL
    assert b"null context" in L.whenet_last_error()
    buf = np.zeros(1024, np.uint8)
    n = C.c_int()
    o.optimize = 1
    assert L.whenet_debug_jpeg_header_ex(8, 8, 3, C.byref(o), buf.ctypes.data, buf.size, C.byref(n)) == EINVAL
    o.optimize = 0
    assert L.whenet_debug_jpeg_header_ex(8, 8, 3, C.byref(o), buf.ctypes.data, 100, C.byref(n)) == EINVAL


def test_python_argument_checks():
    """encode_jpeg refuses bad options before it looks at the context (None here) or runs anything."""
    from whenet_b200 import video
    f = np.zeros((1, 8, 8, 3), np.uint8)
    g = np.zeros((1, 8, 8, 1), np.uint8)
    for kw in [dict(sampling="411"), dict(sampling=444), dict(restart_interval=-1), dict(restart_interval=65536),
               dict(restart_interval=1.0), dict(restart_interval=True), dict(optimize=1), dict(optimize="yes"),
               dict(chroma_quality=0), dict(chroma_quality=101), dict(chroma_quality=40.0), dict(chroma_quality=40),
               dict(sampling="422", chroma_quality=40)]:
        with pytest.raises(ValueError):
            video.encode_jpeg(None, f, 95, **kw)
    for kw in [dict(sampling="444"), dict(sampling="444", chroma_quality=40)]:
        with pytest.raises(ValueError):
            video.encode_jpeg(None, g, 95, **kw)
    with pytest.raises(ValueError):
        video.encode_jpeg(None, [f[0], g[0]], 95)
    with pytest.raises(ValueError):
        video.encode_jpeg(None, np.zeros((1, 8, 8, 2), np.uint8), 95)
    assert video.encode_jpeg(None, [], 95, sampling="444", optimize=True) == []


def test_mjpg_writer_reader_take_every_kind(tmp_path):
    """Gray, 4:4:4, 4:2:2, restart and optimised files go through MJPGWriter and MJPGReader unchanged, and cv2 decodes them."""
    from whenet_b200 import video
    img = frame("gradient", 37, 53)
    files = [J.encode_ex(img[..., 1], 90), J.encode_ex(img, 90, "444"), J.encode_ex(img, 90, "422", restart=2),
             J.encode_ex(img, 90, "420", restart=1, optimize=True), J.encode_ex(img, 90, "444", optimize=True, chroma_quality=30)]
    path = str(tmp_path / "k.avi")
    with video.MJPGWriter(path, 25, (53, 37)) as w:
        w.write(files)
    with video.MJPGReader(path) as r:
        assert r.frame_size == (53, 37)
        assert r.read(len(files)) == files
    for f in files:
        assert cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_UNCHANGED) is not None
