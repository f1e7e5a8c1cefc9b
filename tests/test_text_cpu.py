"""Text on frames without a GPU (DESIGN.md section 8.8): oracle/text_oracle.py equals cv2.putText bit for bit, the committed
glyph table equals what tools/extract_hershey.py reads from the installed cv2, the C host geometry
(whenet_debug_text_segments) equals the oracle's, the label numbers equal numpy's, and the argument checks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(__file__), "..")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
cv2 = pytest.importorskip("cv2")

import text_oracle as T  # noqa: E402

EINVAL = -1         # WHENET_EINVAL
PRINTABLE = "".join(chr(c) for c in range(32, 127))


def _random_text(rng, lo=1, hi=40):
    return "".join(chr(int(c)) for c in rng.integers(32, 127, int(rng.integers(lo, hi + 1))))


def _cmp(img, text, org, scale, color):
    a = img.copy()
    b = img.copy()
    cv2.putText(a, text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, color, 1)
    T.put_text(b, text, org, scale, color)
    assert np.array_equal(a, b), (img.shape, text, org, scale, color, np.argwhere((a != b).any(-1))[:5].tolist())
    return a


@pytest.mark.parametrize("scale", [0.1, 0.4, 0.5, 1.0, 2.5, 8.0])
def test_every_character_alone(scale):
    h, w = int(45 * scale) + 8, int(40 * scale) + 8
    org = (int(10 * scale) + 3, int(32 * scale) + 3)
    for ch in PRINTABLE:
        _cmp(np.zeros((h, w, 3), np.uint8), ch, org, scale, (255, 255, 255))


def test_random_strings_scales_origins_and_overlap():
    """Random strings on one canvas per size, each over the earlier ones, at random scales, colours and origins inside,
    straddling and outside the frame."""
    rng = np.random.default_rng(0)
    sizes = [(1, 1, 150), (2, 3, 150), (17, 40, 200), (240, 320, 200), (1080, 1920, 60), (2160, 3840, 20), (16384, 24, 20),
             (24, 16384, 20)]
    for H, W, k in sizes:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        for _ in range(k):
            scale = float(rng.choice([0.4, float(rng.uniform(0.1, 8.0))]))
            span = int(30 * scale * 40)
            x = int(rng.integers(-span - 50, W + 50))
            y = int(rng.integers(-int(40 * scale) - 50, H + int(40 * scale) + 50))
            c = tuple(int(v) for v in rng.integers(0, 256, 3))
            img = _cmp(img, _random_text(rng), (x, y), scale, c)


def test_far_outside_and_negative_origins():
    img = np.full((50, 60, 3), 9, np.uint8)
    for org in [(-100000, 20), (100000, 20), (10, -100000), (10, 100000), (-70, -5), (59, 49), (-3, 60)]:
        _cmp(img, "yaw: -179.0", org, 0.4, (100, 255, 0))


def test_committed_table_equals_extraction():
    import extract_hershey as E
    import hershey_simplex as HS
    ver, base_line, table = E.extract()
    assert base_line == HS.BASE_LINE == -9
    assert tuple(table) == HS.GLYPHS
    inc, py = E.render(ver, base_line, table)
    for path, text in ((E.INC, inc), (E.PY, py)):
        with open(path) as f:
            committed = f.read()
        strip = lambda s: s.split("\n", 2)[2]          # noqa: E731 - the first two lines name the cv2 version
        assert strip(committed) == strip(text), path


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def _c_segments(text, org, scale):
    L = _lib()
    n = C.c_int32()
    assert L.whenet_debug_text_segments(text.encode(), org[0], org[1], scale, 1, None, 0, C.byref(n)) == 0
    out = np.zeros((max(n.value, 1), 4), np.int64)
    assert L.whenet_debug_text_segments(text.encode(), org[0], org[1], scale, 1, out.ctypes.data, n.value, C.byref(n)) == 0
    return [tuple(int(v) for v in s) for s in out[:n.value]]


def test_host_geometry_equals_oracle():
    rng = np.random.default_rng(1)
    cases = [(PRINTABLE, (0, 0), 0.4), (PRINTABLE, (-5, 7), 1.0), ("yaw: -12.0", (100, 30), 0.4)]
    for _ in range(2000):
        cases.append((_random_text(rng), (int(rng.integers(-(1 << 24), 1 << 24)), int(rng.integers(-(1 << 24), 1 << 24))),
                      float(rng.choice([0.4, 0.5, float(rng.uniform(0.01, 256))]))))
    for text, org, scale in cases:
        assert _c_segments(text, org, scale) == T.text_segments(text, org, scale), (text, org, scale)


def _c_labels(a):
    L = _lib()
    a = np.ascontiguousarray(a, np.float32)
    out = C.create_string_buffer(32 * len(a))
    assert L.whenet_debug_label_text(a.ctypes.data, len(a), out, 32) == 0
    raw = out.raw
    return [raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode() for i in range(len(a))]


def test_label_numbers_equal_the_reference_format():
    grid = np.arange(-180.0, 180.0 + 1e-9, 1 / 256, dtype=np.float64).astype(np.float32)
    ties = np.arange(-180, 181, dtype=np.float32) + np.float32(0.5)
    near = np.concatenate([np.nextafter(ties, np.float32(np.inf)), np.nextafter(ties, np.float32(-np.inf))])
    rng = np.random.default_rng(2)
    big = np.concatenate([np.float32(10.0) ** np.arange(-3, 39, dtype=np.float32), rng.uniform(-1e38, 1e38, 500),
                          rng.uniform(-1e17, 1e17, 500), rng.uniform(-1e7, 1e7, 500), [1e16, 9.999999e15, 16777217.0, 1e6, 999999.0, 999999.5, 1e6 + 1]])
    special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 0.4999999, -0.4999999, 0.5, -0.5, 1.5, 2.5, -2.5,
                        np.finfo(np.float32).max, -np.finfo(np.float32).max], np.float32)
    a = np.concatenate([grid, ties, near, big.astype(np.float32), special]).astype(np.float32)
    got = _c_labels(a)
    for v, g in zip(a, got):
        assert g == T.label_text(v) == "{}".format(np.round(np.float32(v))), (repr(v), g)
        if abs(v) <= 180 or not np.isfinite(v):
            assert g == str(np.round(np.float32(v))), (repr(v), g)
    assert _c_labels([-0.0, -0.4, 12.5, 13.5, np.nan, 1e6]) == ["-0.0", "-0.0", "12.0", "14.0", "nan", "1000000.0"]


def test_argument_checks():
    L = _lib()
    n = C.c_int32()
    assert L.whenet_debug_text_segments(b"ok", 0, 0, 0.4, 1, None, 0, C.byref(n)) == 0 and n.value > 0
    assert L.whenet_debug_text_segments(b"tab\there", 0, 0, 0.4, 1, None, 0, None) == EINVAL
    assert L.whenet_debug_text_segments(b"\xc3\xa9", 0, 0, 0.4, 1, None, 0, None) == EINVAL
    assert L.whenet_debug_text_segments(None, 0, 0, 0.4, 1, None, 0, None) == EINVAL
    for t in (0, 2, -1):
        assert L.whenet_debug_text_segments(b"ok", 0, 0, 0.4, t, None, 0, None) == EINVAL
    assert b"thickness" in L.whenet_last_error()
    for s in (0.0, -1.0, 257.0, float("nan"), float("inf")):
        assert L.whenet_debug_text_segments(b"ok", 0, 0, s, 1, None, 0, None) == EINVAL
    assert L.whenet_debug_text_segments(b"ok", 1 << 25, 0, 0.4, 1, None, 0, None) == EINVAL
    assert L.whenet_debug_text_segments(b"x" * 4097, 0, 0, 0.4, 1, None, 0, None) == EINVAL
    assert L.whenet_debug_label_text(None, 1, None, 32) == EINVAL

    b = np.zeros((1, 4), np.float32)
    a = np.zeros((1, 3), np.float32)
    fo = np.zeros(1, np.int32)
    buf = (C.c_uint8 * 3)()
    d = C.addressof(buf)
    for disp in (-1, 2, 7):
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert b"display" in L.whenet_last_error()
    for disp in (0, 1):
        assert L.whenet_draw_heads_ex_u8(None, None, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 0, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 65, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 16385, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, None, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        bad_fo = np.array([1], np.int32)
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, bad_fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, -1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, disp, None) == EINVAL
        assert b"context" in L.whenet_last_error()
        assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, None, None, None, 0, disp, None) == 0
        hw = np.array([[1, 0]], np.int32)
        ptrs = (C.c_void_p * 1)(d)
        assert L.whenet_draw_heads_ex_ragged_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, b.ctypes.data, a.ctypes.data,
                                                fo.ctypes.data, 1, disp, None) == EINVAL
        assert L.whenet_draw_heads_ex_ragged_u8(None, None, hw.ctypes.data, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1,
                                                disp, None) == EINVAL

    def put(texts, org=(0, 0), scale=0.4, thick=1, fo_=0, n_=1, H=1, W=1, frames=d):
        m = len(texts)
        tp = (C.c_char_p * max(m, 1))(*texts)
        o = np.array([org] * m, np.int32).reshape(-1, 2)
        s = np.full(m, scale, np.float64)
        c = np.zeros((m, 3), np.uint8)
        t = np.full(m, thick, np.int32)
        f = np.full(m, fo_, np.int32)
        return L.whenet_put_text_u8(None, frames, n_, H, W, f.ctypes.data, C.addressof(tp), o.ctypes.data, s.ctypes.data,
                                    c.ctypes.data, t.ctypes.data, m)

    assert put([b"ok"], thick=2) == EINVAL and b"thickness" in L.whenet_last_error()
    assert put([b"ok\x01"]) == EINVAL and b"printable" in L.whenet_last_error()
    assert put([b"ok\x7f"]) == EINVAL
    assert put([b"ok"], scale=0.0) == EINVAL
    assert put([b"ok"], fo_=1) == EINVAL and b"frame_of" in L.whenet_last_error()
    assert put([b"ok"], n_=0) == EINVAL
    assert put([b"ok"], n_=65) == EINVAL
    assert put([b"ok"], H=16385) == EINVAL
    assert put([b"ok"], frames=None) == EINVAL
    assert put([b"ok"]) == EINVAL and b"context" in L.whenet_last_error()
    assert put([]) == 0
    big = b"x" * 4096
    assert put([big] * 1025) == EINVAL and b"characters" in L.whenet_last_error()        # 2^22 + 4096 characters
    m = (1 << 16) + 1
    bm = np.zeros((m, 4), np.float32)
    am = np.zeros((m, 3), np.float32)
    fm = np.zeros(m, np.int32)
    assert L.whenet_draw_heads_ex_u8(None, d, 1, 1, 1, bm.ctypes.data, am.ctypes.data, fm.ctypes.data, m, 1, None) == EINVAL
    assert b"65536" in L.whenet_last_error()


def test_python_entries_refuse_bad_input():
    from whenet_b200 import overlay

    class FakeWhenet:
        device = 0

    res = [(np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros((0, 3), np.float32))]
    with pytest.raises(ValueError):
        overlay.draw_heads(FakeWhenet(), np.zeros((1, 4, 4, 3), np.uint8), res, display="full")
    with pytest.raises(ValueError):
        overlay.draw_heads(FakeWhenet(), np.zeros((1, 4, 4, 3), np.uint8), res, display="labels")
    with pytest.raises(ValueError):
        overlay.put_text(FakeWhenet(), np.zeros((1, 4, 4, 3), np.uint8), [(0, "x", (0, 0), 0.4, (0, 0, 0))])
