"""Progressive JPEG (DESIGN.md section 8.12) without a GPU: ``oracle/jpeg_progressive_oracle.py`` equals cv2.imencode with
IMWRITE_JPEG_PROGRESSIVE 1 on the options matrix of section 8.11; the facts about cv2's files that the encoder relies on (scan
script, DHT placement, OPTIMIZE ignored, the same coefficients as the optimised baseline file); both EOB run caps, shown
firing by the oracle's counters and agreeing with cv2; and the ABI and Python argument checks without a context."""
import ctypes as C
import os
import sys

import cv2
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_jpeg_cpu import EINVAL, KINDS  # noqa: E402
from test_jpeg_options_cpu import SAMPLINGS, SIZES, cv2_params, option_image  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import jpeg_progressive_oracle as P  # noqa: E402
from jpeg_options_oracle import blocks_ex  # noqa: E402

# (quality, restart interval): qualities 1, 50, 95, 100 and restarts 0, 1, 3, more than the MCUs, each at least once
PROG_SETS = [(95, 0), (1, 1), (50, 3), (100, 65535), (95, 1), (50, 0), (100, 3), (1, 0), (95, 3)]


def cv2_prog(img, quality=95, sampling="420", restart_interval=0, chroma_quality=None, optimize=False):
    """cv2's progressive file of a BGR (H, W, 3) or gray (H, W, 1) image."""
    if img.ndim == 3 and img.shape[2] == 1:
        img = img[..., 0]
    params = cv2_params(quality, sampling, restart_interval, optimize, chroma_quality) + [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def oracle_prog(img, quality=95, sampling="420", restart_interval=0, chroma_quality=None):
    return P.encode_progressive(img[..., 0] if img.shape[2] == 1 else img, quality, sampling, restart_interval, chroma_quality)


def be_cap_frame(h=64, w=256, seed=2):
    """A gray frame whose every block has, at quality 100, about 57 AC coefficients with |c| >= 4 and none with |c| in {2, 3}:
    in the Ah 2 Al 1 refinement scan each block sends correction bits and no symbol, so the run's buffer passes 937 bits
    every ~17 blocks.  Built by the inverse of the orthonormal 8x8 DCT (the scale of libjpeg's quantised coefficients at
    quantiser 1); rounding the pixels moves a coefficient by at most 1, so +-6..8 stays >= 4 and 0 stays in {-1, 0, 1}."""
    from scipy.fft import idctn
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w), np.float64)
    for by in range(h // 8):
        for bx in range(w // 8):
            c = rng.choice([-8, -7, -6, 6, 7, 8], size=(8, 8)) * (rng.random((8, 8)) < 0.9)
            c[0, 0] = 0
            img[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8] = idctn(c, norm="ortho") + 128
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)[..., None]


def _segments(data):
    """(marker, payload) of every marker segment, skipping entropy-coded data"""
    out, i = [], 2
    while i < len(data):
        m = data[i + 1]
        if m == 0xD9:
            break
        n = int.from_bytes(data[i + 2:i + 4], "big")
        out.append((m, data[i + 4:i + 2 + n]))
        i += 2 + n
        if m == 0xDA:
            while not (data[i] == 0xFF and data[i + 1] != 0 and not 0xD0 <= data[i + 1] <= 0xD7):
                i += 1
    return out


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("h,w", SIZES)
def test_oracle_equals_cv2(h, w, sampling):
    for q, r in PROG_SETS:
        for k, kind in enumerate(KINDS):
            img = option_image(kind, h, w, sampling, seed=q + k)
            opts = dict(quality=q, sampling="420" if sampling == "gray" else sampling, restart_interval=r)
            assert oracle_prog(img, **opts) == cv2_prog(img, **opts), (kind, opts)


@pytest.mark.parametrize("q,cq", [(90, 40), (40, 90)])
def test_oracle_two_qualities(q, cq):
    for kind in KINDS:
        img = option_image(kind, 37, 53, "444", seed=cq)
        for r in (0, 3):
            opts = dict(quality=q, sampling="444", restart_interval=r, chroma_quality=cq)
            assert oracle_prog(img, **opts) == cv2_prog(img, **opts)


def test_oracle_equals_cv2_1081p():
    for sampling in SAMPLINGS:
        img = option_image("noise", 1081, 1921, sampling, seed=7)
        opts = dict(quality=95, sampling="420" if sampling == "gray" else sampling, restart_interval=0 if sampling != "444" else 120)
        assert oracle_prog(img, **opts) == cv2_prog(img, **opts), sampling


@pytest.mark.parametrize("channels", [1, 3])
def test_scan_script_and_dht_placement(channels):
    """SOF2; per scan the DHTs of its own tables just before its SOS (two DC tables in the first colour scan, one AC table
    per AC scan, none for DC refinement); DRI once, before the first SOS; SOS components, table selectors, Ss, Se, Ah, Al."""
    sampling = "gray" if channels == 1 else "420"
    img = option_image("noise", 37, 53, sampling, seed=1)
    segs = _segments(cv2_prog(img, restart_interval=3))
    markers = [m for m, _ in segs]
    sof = 0xC2
    assert markers[:4] == [0xE0, 0xDB] + ([0xDB] if channels == 3 else []) + [sof] or markers[:3] == [0xE0, 0xDB, sof]
    assert 0xC0 not in markers and markers.count(0xDD) == 1
    scans, dhts = [], []
    for m, p in segs[markers.index(sof) + 1:]:
        if m == 0xC4:
            dhts.append(p[0])
        elif m == 0xDD:
            assert not scans, "DRI comes before the first SOS"
        elif m == 0xDA:
            ns = p[0]
            comps = tuple(p[1 + 2 * i] - 1 for i in range(ns))
            sel = tuple(p[2 + 2 * i] for i in range(ns))
            Ss, Se, AhAl = p[1 + 2 * ns:4 + 2 * ns]
            scans.append((comps, Ss, Se, AhAl >> 4, AhAl & 15, sel, tuple(dhts)))
            dhts = []
    script = P.scan_script(channels)
    assert [s[:5] for s in scans] == [s for s in script]
    for comps, Ss, Se, Ah, Al, sel, tabs in scans:
        if Ss == 0 and Ah:
            assert tabs == () and set(sel) == {0}
        elif Ss == 0:
            assert tabs == ((0x00, 0x01) if channels == 3 else (0x00,))
            assert sel == tuple(0x00 if c == 0 else 0x10 for c in comps)
        else:
            assert tabs == (0x10 | (comps[0] != 0),) and sel == (int(comps[0] != 0),)


def test_optimize_has_no_effect_and_coefficients_match():
    """OPTIMIZE 1 changes no byte of a progressive file, and the progressive file decodes to the optimised baseline file's
    pixels: the coefficients are the baseline transform's."""
    for sampling in SAMPLINGS:
        for h, w in [(17, 33), (37, 53), (120, 200)]:
            for q, r in [(95, 0), (50, 3), (100, 0), (1, 1)]:
                img = option_image("noise" if q != 50 else "gradient", h, w, sampling, seed=h + q)
                opts = dict(quality=q, sampling="420" if sampling == "gray" else sampling, restart_interval=r)
                prog = cv2_prog(img, **opts)
                assert cv2_prog(img, optimize=True, **opts) == prog
                src = img[..., 0] if sampling == "gray" else img
                base = cv2.imencode(".jpg", src, cv2_params(optimize=True, **opts))[1]
                assert np.array_equal(cv2.imdecode(np.frombuffer(prog, np.uint8), cv2.IMREAD_UNCHANGED),
                                      cv2.imdecode(base, cv2.IMREAD_UNCHANGED)), opts


def test_units_per_scan():
    """A one-component scan walks the component's own block grid, not the MCU-padded one."""
    img = option_image("noise", 17, 33, "420", seed=3)
    P.encode_progressive(img, 95, "420")
    mcus, luma = 2 * 3, 3 * 5          # 4:2:0 MCUs of 16x16 over 33x17; 8x8 luma blocks
    assert P.STATS["units"] == [mcus, luma, mcus, mcus, luma, luma, mcus, mcus, mcus, luma]


def test_eobrun_cap():
    """A flat 2048x2048 gray frame: 65,536 empty luma blocks per AC scan, so each run is flushed at 0x7FFF.  A flat 4:2:0
    frame of 2912x2912 does the same for the chroma scans (182 x 182 blocks per plane)."""
    gray = np.full((2048, 2048, 1), 77, np.uint8)
    assert oracle_prog(gray) == cv2_prog(gray)
    assert P.STATS["eobrun_cap"] == 2 * 4 and P.STATS["be_cap"] == 0
    col = np.empty((2912, 2912, 3), np.uint8)
    col[:] = (40, 160, 90)
    assert oracle_prog(col) == cv2_prog(col)
    assert P.STATS["eobrun_cap"] == 4 * (364 * 364 // 0x7FFF) + 4 * (182 * 182 // 0x7FFF)


def test_be_cap():
    """Correction bits alone fill the run's buffer: the Ah 2 Al 1 scan flushes at 937 buffered bits, and cv2 agrees."""
    img = be_cap_frame()
    c = np.abs(blocks_ex(img[..., 0], 100)[:, 1:])
    assert not ((c == 2) | (c == 3)).any() and (c >= 4).sum(1).min() > 40
    assert oracle_prog(img, 100) == cv2_prog(img, 100)
    assert P.STATS["be_cap"] >= 10


def test_abi_argument_checks():
    """progressive outside {0, 1} and a progressive header request are refused before any device call (no context)."""
    from whenet_b200 import _lib
    L = _lib.load()
    buf = np.zeros(4096, np.uint8)
    n = C.c_int()
    frame = np.zeros((8, 8, 3), np.uint8)
    ptrs = (C.c_void_p * 1)(frame.ctypes.data)
    hw = np.array([[8, 8]], np.int32)
    data = C.c_void_p()
    offs = np.zeros(2, np.int64)
    for prog in (2, -1):
        o = _lib.JpegOptions(95, 95, 420, 0, 0, prog)
        assert L.whenet_encode_jpeg_ex_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, 3, 0, C.byref(o), C.byref(data),
                                          offs.ctypes.data) == EINVAL
        assert b"progressive" in L.whenet_last_error()
    o = _lib.JpegOptions(95, 95, 420, 0, 0, 1)
    assert L.whenet_debug_jpeg_header_ex(8, 8, 3, C.byref(o), buf.ctypes.data, buf.size, C.byref(n)) == EINVAL
    assert b"progressive" in L.whenet_last_error()
    # without the field, ctypes zero-fills it: the baseline header
    o5 = _lib.JpegOptions(95, 95, 420, 0, 0)
    assert o5.progressive == 0
    assert L.whenet_debug_jpeg_header_ex(8, 8, 3, C.byref(o5), buf.ctypes.data, buf.size, C.byref(n)) == 0


def test_python_argument_checks():
    from whenet_b200 import video
    f = np.zeros((1, 8, 8, 3), np.uint8)
    for bad in (1, 0, None, "yes", 1.0):
        with pytest.raises(ValueError, match="progressive"):
            video.encode_jpeg(None, f, 95, progressive=bad)
