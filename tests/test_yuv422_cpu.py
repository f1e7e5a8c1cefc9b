"""Packed YUV 4:2:2 frames (YUYV, UYVY) and the YUV -> BGR conversion entries without a GPU: the integer oracle against
cv2.cvtColor bit for bit, the argument validation of the six new C entries (every bad argument is refused, naming it, before
anything touches a device), the pixel_format and to_bgr checks of the Python wrappers, and the new kernel instances as ptxas
builds them."""
import ctypes as C
import os
import re
import subprocess
import tempfile
import types

import numpy as np
import pytest

import yuv422_oracle as Y
import yuv_oracle

NV12, I420, YUYV, UYVY = 1, 2, 3, 4
CODES = {"yuyv": "COLOR_YUV2BGR_YUYV", "uyvy": "COLOR_YUV2BGR_UYVY"}
SIZES = [(1, 2), (3, 6), (7, 34), (5, 1002), (2, 2), (33, 64), (480, 640), (1081, 1920), (1080, 1920), (2160, 3840)]
LAYOUT_MSG = b"yuv422_layout=%d: WHENET_YUV_YUYV (3) or WHENET_YUV_UYVY (4)"
CONVERT_MSG = b"layout=%d: WHENET_YUV_NV12 (1), WHENET_YUV_I420 (2), WHENET_YUV_YUYV (3) or WHENET_YUV_UYVY (4)"


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def P(a):
    return None if a is None else a.ctypes.data


# ----------------------------------------------------------------------------------------------- the conversion
@pytest.mark.parametrize("layout", Y.LAYOUTS_422)
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_oracle_equals_cv2_on_random_frames(layout, size):
    cv2 = pytest.importorskip("cv2")
    H, W = size
    buf = np.random.default_rng(H * 7919 + W).integers(0, 256, (H, W, 2), dtype=np.uint8)
    assert np.array_equal(Y.yuv422_to_bgr(buf, layout), cv2.cvtColor(buf, getattr(cv2, CODES[layout])))


@pytest.mark.parametrize("layout", Y.LAYOUTS_422)
def test_oracle_equals_cv2_on_the_extremes(layout):
    """Every Y in {0, 16, 235, 255} against every (U, V) in {0, 128, 255}^2, each on its own pixel pair."""
    cv2 = pytest.importorskip("cv2")
    combos = [(y, u, v) for y in (0, 16, 235, 255) for u in (0, 128, 255) for v in (0, 128, 255)]
    quads = [(y, u, y, v) if layout == "yuyv" else (u, y, v, y) for y, u, v in combos]
    buf = np.array(quads, np.uint8).reshape(1, 2 * len(combos), 2)
    got = Y.yuv422_to_bgr(buf, layout)
    assert np.array_equal(got, cv2.cvtColor(buf, getattr(cv2, CODES[layout])))
    assert got.min() == 0 and got.max() == 255                 # both clips are reached


def test_oracle_planes_and_refusals():
    buf = np.arange(2 * 4 * 2, dtype=np.uint8).reshape(2, 4, 2)  # two rows of two pixel pairs
    y, u, v = Y.planes422(buf, "yuyv")
    assert np.array_equal(y, [[0, 2, 4, 6], [8, 10, 12, 14]]) and np.array_equal(u, [[1, 5], [9, 13]]) and np.array_equal(v, [[3, 7], [11, 15]])
    y, u, v = Y.planes422(buf, "uyvy")
    assert np.array_equal(y, [[1, 3, 5, 7], [9, 11, 13, 15]]) and np.array_equal(u, [[0, 4], [8, 12]]) and np.array_equal(v, [[2, 6], [10, 14]])
    for bad in (np.zeros((2, 3, 2), np.uint8), np.zeros((2, 4, 3), np.uint8), np.zeros((2, 4), np.uint8), np.zeros((0, 4, 2), np.uint8),
                np.zeros((2, 4, 2), np.int16)):
        with pytest.raises(ValueError):
            Y.planes422(bad, "yuyv")
    for layout in ("nv12", "yuy2", "YUYV"):
        with pytest.raises(ValueError):
            Y.planes422(buf, layout)
    with pytest.raises(ValueError):
        yuv_oracle.planes(np.zeros((6, 4), np.uint8), "nv21")    # the 4:2:0 oracle is as it was


def test_scene_maker_round_trips():
    bgr = np.random.default_rng(3).integers(0, 256, (5, 8, 3), dtype=np.uint8)
    bgr[:, 1::2] = bgr[:, ::2]                                   # pairs of equal pixels keep their chroma
    for layout in Y.LAYOUTS_422:
        f = Y.bgr_to_yuv422(bgr, layout)
        assert f.shape == (5, 8, 2) and f.dtype == np.uint8
        assert np.abs(Y.yuv422_to_bgr(f, layout).astype(int) - bgr).max() <= 3


# ----------------------------------------------------------------------------------------------- C entries
def _det_outputs(n):
    return np.zeros((n, 20, 4), np.float32), np.zeros((n, 20), np.float32), np.zeros((n, 20), np.int32), np.zeros(n, np.int32)


def test_detect_yuv422_argument_validation():
    L = _lib()
    frames = np.zeros((2, 7, 8, 2), np.uint8)                  # two 8 x 7 frames
    boxes, scores, classes, counts = _det_outputs(2)

    def call(fr=frames, n=2, H=7, W=8, layout=YUYV, out=counts):
        rc = L.whenet_det_detect_yuv422_u8(None, P(fr), n, H, W, 0, layout, 0.3, 0.45, 20, P(boxes), P(scores), P(classes), P(out))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null detector")                     # every other argument is fine, the odd height too
    assert call(layout=UYVY) == (-1, b"null detector")
    for bad in (0, 1, 2, 5, -1):
        assert call(layout=bad) == (-1, LAYOUT_MSG % bad)
    assert call(fr=None) == (-1, b"null frames")
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d outside [1, 64]" % n)
    for H, W in ((7, 7), (8, 1), (0, 8), (8, 0), (16385, 8), (8, 16386), (-1, 8)):
        rc, msg = call(H=H, W=W)
        assert rc == -1 and msg == b"frame size %dx%d: a 4:2:2 frame has an even width in [2, 16384] and a height in [1, 16384]" % (W, H), msg
    for H, W in ((1, 2), (16384, 2), (1, 16384), (16384, 16384)):
        assert call(H=H, W=W) == (-1, b"null detector")
    assert call(out=None) == (-1, b"null output pointer")


def test_detect_ragged_yuv422_argument_validation():
    L = _lib()
    keep = [np.zeros((8, 8, 2), np.uint8), np.zeros((5, 10, 2), np.uint8)]
    ptrs = (C.c_void_p * 2)(*(f.ctypes.data for f in keep))
    hw = np.array([8, 8, 5, 10], np.int32)
    boxes, scores, classes, counts = _det_outputs(2)

    def call(fr=ptrs, hw=hw, n=2, layout=UYVY, out=counts):
        rc = L.whenet_det_detect_ragged_yuv422_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, layout, 0.3, 0.45, 20,
                                                  P(boxes), P(scores), P(classes), P(out))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null detector")
    for bad in (0, 1, 2, 5):
        assert call(layout=bad) == (-1, LAYOUT_MSG % bad)
    assert call(fr=None) == (-1, b"null frames or hw")
    assert call(hw=None) == (-1, b"null frames or hw")
    for n in (0, 65):
        assert call(n=n) == (-1, b"n=%d outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(ptrs[0], None)) == (-1, b"frame 1 is NULL")
    rc, msg = call(hw=np.array([8, 8, 5, 9], np.int32))
    assert rc == -1 and msg == b"frame 1: frame size 9x5: a 4:2:2 frame has an even width", msg
    assert call(hw=np.array([8, 8, 1, 2], np.int32)) == (-1, b"null detector")
    assert call(hw=np.array([8, 8, 16386, 8], np.int32)) == (-1, b"frame 1: bad frame size 8x16386")
    assert call(hw=np.array([8, 0, 5, 10], np.int32)) == (-1, b"frame 0: bad frame size 0x8")
    assert call(out=None) == (-1, b"null output pointer")


def test_crop_boxes_yuv422_argument_validation():
    L = _lib()
    frames = np.zeros((2, 7, 8, 2), np.uint8)
    boxes = np.array([[1, 1, 6, 6], [0, 0, 7, 8]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)

    def call(fr=frames, n=2, H=7, W=8, bx=boxes, f=fo, m=2, layout=YUYV, crops=out):
        rc = L.whenet_crop_boxes_yuv422_u8(None, P(fr), n, H, W, 0, P(bx), P(f), m, layout, P(crops), None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")
    for bad in (0, 1, 2, 5):
        assert call(layout=bad) == (-1, LAYOUT_MSG % bad)
    null_msg = b"null frames, boxes, frame_of or crops_out"
    for kw in ({"fr": None}, {"bx": None}, {"f": None}, {"crops": None}):
        assert call(**kw) == (-1, null_msg), kw
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    for H, W in ((7, 7), (7, 1), (16385, 8), (8, 16386)):
        rc, msg = call(H=H, W=W)
        assert rc == -1 and msg == b"frame size %dx%d: a 4:2:2 frame has an even width in [2, 16384] and a height of at most 16384" % (H, W), msg
    assert call(H=0, W=8) == (-1, b"bad frame size 0x8")
    assert call(H=1, W=2) == (-1, b"null context")
    assert call(m=0) == (-1, b"m=0 boxes")
    assert call(f=np.array([0, 2], np.int32)) == (-1, b"box 1: frame_of=2 outside [0, 2)")


def test_crop_boxes_ragged_yuv422_argument_validation():
    L = _lib()
    keep = [np.zeros((7, 8, 2), np.uint8), np.zeros((5, 10, 2), np.uint8)]
    ptrs = (C.c_void_p * 2)(*(f.ctypes.data for f in keep))
    hw = np.array([7, 8, 5, 10], np.int32)
    boxes = np.array([[1, 1, 6, 6], [0, 0, 5, 10]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)

    def call(fr=ptrs, hw=hw, n=2, bx=boxes, f=fo, m=2, layout=UYVY, crops=out):
        rc = L.whenet_crop_boxes_ragged_yuv422_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, P(bx), P(f), m, layout,
                                                  P(crops), None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")
    for bad in (0, 1, 2, 5):
        assert call(layout=bad) == (-1, LAYOUT_MSG % bad)
    null_msg = b"null frames, hw, boxes, frame_of or crops_out"
    for kw in ({"fr": None}, {"hw": None}, {"bx": None}, {"f": None}, {"crops": None}):
        assert call(**kw) == (-1, null_msg), kw
    for n in (0, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(None, ptrs[1])) == (-1, b"frame 0 is NULL")
    rc, msg = call(hw=np.array([7, 8, 5, 11], np.int32))
    assert rc == -1 and msg == b"frame 1: frame size 11x5: a 4:2:2 frame has an even width", msg
    assert call(hw=np.array([7, 8, 16385, 10], np.int32)) == (-1, b"frame 1: bad frame size 10x16385")
    assert call(m=0) == (-1, b"m=0 boxes")


def test_yuv_to_bgr_argument_validation():
    L = _lib()
    frames = np.zeros((2, 8, 8, 2), np.uint8)
    out = np.zeros((2, 8, 8, 3), np.uint8)

    def call(fr=frames, n=2, H=8, W=8, layout=YUYV, o=out):
        rc = L.whenet_yuv_to_bgr_u8(None, P(fr), n, H, W, 0, layout, P(o))
        return rc, L.whenet_last_error()

    for layout in (NV12, I420, YUYV, UYVY):
        assert call(layout=layout) == (-1, b"null context")
    for bad in (0, 5, -1):
        assert call(layout=bad) == (-1, CONVERT_MSG % bad)
    assert call(fr=None) == (-1, b"null frames or out_frames")
    assert call(o=None) == (-1, b"null frames or out_frames")
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    for H, W in ((0, 8), (8, 0), (16385, 8), (8, 16386)):
        for layout in (NV12, YUYV):
            assert call(H=H, W=W, layout=layout) == (-1, b"frame size %dx%d: sides must be in [1, 16384]" % (W, H))
    for layout in (YUYV, UYVY):
        assert call(H=8, W=7, layout=layout) == (-1, b"frame size 7x8: a 4:2:2 frame has an even width")
        assert call(H=1, W=2, layout=layout) == (-1, b"null context")
        assert call(H=16384, W=16384, layout=layout) == (-1, b"null context")
    for layout in (NV12, I420):
        for H, W in ((7, 8), (8, 7), (1, 2)):
            assert call(H=H, W=W, layout=layout) == (-1, b"frame size %dx%d: a 4:2:0 frame has even sides" % (W, H))
        assert call(H=2, W=2, layout=layout) == (-1, b"null context")


def test_yuv_to_bgr_ragged_argument_validation():
    L = _lib()
    keep = [np.zeros((7, 8, 2), np.uint8), np.zeros((5, 10, 2), np.uint8)]
    outs = [np.zeros((7, 8, 3), np.uint8), np.zeros((5, 10, 3), np.uint8)]
    ptrs = (C.c_void_p * 2)(*(f.ctypes.data for f in keep))
    dst = (C.c_void_p * 2)(*(f.ctypes.data for f in outs))
    hw = np.array([7, 8, 5, 10], np.int32)

    def call(fr=ptrs, hw=hw, n=2, layout=UYVY, o=dst):
        rc = L.whenet_yuv_to_bgr_ragged_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, layout,
                                           None if o is None else C.addressof(o))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")
    for bad in (0, 5):
        assert call(layout=bad) == (-1, CONVERT_MSG % bad)
    for kw in ({"fr": None}, {"hw": None}, {"o": None}):
        assert call(**kw) == (-1, b"null frames, hw or out_frames"), kw
    for n in (0, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(ptrs[0], None)) == (-1, b"frame 1: null frame or output")
    assert call(o=(C.c_void_p * 2)(None, dst[1])) == (-1, b"frame 0: null frame or output")
    assert call(hw=np.array([7, 8, 5, 9], np.int32)) == (-1, b"frame 1: frame size 9x5: a 4:2:2 frame has an even width")
    assert call(hw=np.array([7, 8, 16385, 10], np.int32)) == (-1, b"frame 1: frame size 10x16385: sides must be in [1, 16384]")
    assert call(layout=NV12) == (-1, b"frame 0: frame size 8x7: a 4:2:0 frame has even sides")
    assert call(hw=np.array([8, 8, 6, 10], np.int32), layout=I420) == (-1, b"null context")


# ----------------------------------------------------------------------------------------------- Python wrappers
def _fake_yolo():
    import whenet_b200
    y = whenet_b200.YOLO.__new__(whenet_b200.YOLO)
    y.device, y.max_frames = 0, 8
    return y


def test_wrappers_refuse_bad_yuv422_frames():
    from whenet_b200 import pipeline
    y = _fake_yolo()
    y0, w0 = types.SimpleNamespace(device=0), types.SimpleNamespace(device=0)
    bgr = np.zeros((2, 8, 8, 3), np.uint8)
    good = np.zeros((2, 7, 8, 2), np.uint8)
    nv12 = np.zeros((2, 12, 8), np.uint8)
    for fmt in ("yuyv", "uyvy"):
        for bad in (bgr, nv12, np.zeros((2, 7, 7, 2), np.uint8), np.zeros((7, 8, 2), np.uint8), np.zeros((2, 0, 8, 2), np.uint8)):
            with pytest.raises(ValueError):
                y.detect_frames(bad, pixel_format=fmt)
            with pytest.raises(ValueError):
                pipeline.detect_and_estimate_frames(y0, w0, bad, pixel_format=fmt)
        with pytest.raises(ValueError, match="frame 1"):
            y.detect_frames([good[0], np.zeros((8, 8, 3), np.uint8)], pixel_format=fmt)       # a 3-channel frame in the list
        with pytest.raises(ValueError, match="frame 1"):
            y.detect_frames([good[0], nv12[0]], pixel_format=fmt)                              # a 4:2:0 frame in the list
        with pytest.raises(ValueError, match="frame 0"):
            pipeline.detect_and_estimate_frames(y0, w0, [np.zeros((7, 9, 2), np.uint8)], pixel_format=fmt)
        with pytest.raises(ValueError, match="4:2:2"):
            pipeline.detect_and_estimate(y0, w0, np.zeros((7, 8, 3), np.uint8), pixel_format=fmt)
        with pytest.raises(ValueError, match="even width"):
            pipeline.detect_and_estimate(y0, w0, np.zeros((7, 9, 2), np.uint8), pixel_format=fmt)
        assert pipeline.detect_and_estimate_frames(y0, w0, np.zeros((0, 7, 8, 2), np.uint8), pixel_format=fmt) == []
        assert y.detect_frames([], pixel_format=fmt) == []
    for fmt in ("YUYV", "yuy2", "2vuy", "yvyu"):
        with pytest.raises(ValueError, match="pixel_format"):
            y.detect_frames(good, pixel_format=fmt)
        with pytest.raises(ValueError, match="pixel_format"):
            pipeline.detect_and_estimate_frames(y0, w0, good, pixel_format=fmt)


def test_to_bgr_refuses_bad_input():
    from whenet_b200 import video
    w0 = types.SimpleNamespace(device=0)
    for fmt in ("bgr", "nv21", "YUYV", None, 3):
        with pytest.raises(ValueError, match="pixel_format"):
            video.to_bgr(w0, np.zeros((1, 2, 2, 2), np.uint8), fmt)
    bad = {
        "yuyv": [np.zeros((1, 2, 3, 2), np.uint8), np.zeros((1, 2, 2, 3), np.uint8), np.zeros((2, 2, 2), np.uint8),
                 np.zeros((1, 2, 2, 2), np.int16), np.zeros((1, 2, 16386, 2), np.uint8), [np.zeros((2, 2, 2), np.uint8), np.zeros((3, 2), np.uint8)]],
        "nv12": [np.zeros((1, 4, 2), np.uint8), np.zeros((1, 3, 3), np.uint8), np.zeros((1, 3, 2, 2), np.uint8),
                 [np.zeros((3, 2), np.uint8), np.zeros((2, 2, 2), np.uint8)], [np.zeros((3, 2), np.uint8), np.zeros((24579, 2), np.uint8)]],
    }
    bad["uyvy"], bad["i420"] = bad["yuyv"], bad["nv12"]
    for fmt, cases in bad.items():
        for b in cases:
            with pytest.raises(ValueError):
                video.to_bgr(w0, b, fmt)


def test_frame_table_gives_422_image_sizes():
    from whenet_b200.yolo import _frame_table
    frames = [np.zeros((7, 8, 2), np.uint8), np.zeros((1081, 1920, 2), np.uint8)]
    _ptrs, hw = _frame_table(frames, YUYV)
    assert hw.tolist() == [7, 8, 1081, 1920]


# ----------------------------------------------------------------------------------------------- ptxas
_INST = """
#include "kernels_crop.cuh"
#include "kernels_yolo.cuh"
using namespace whenet;
void* yuv422_instances[] = {
    (void*)crop_resize_yuv_kernel<OneSizeFrames, kYuvYUYV>, (void*)crop_resize_yuv_kernel<OneSizeFrames, kYuvUYVY>,
    (void*)crop_resize_yuv_kernel<PerFrameSources, kYuvYUYV>, (void*)crop_resize_yuv_kernel<PerFrameSources, kYuvUYVY>,
    (void*)yolo::letterbox_h_yuv_kernel<kYuvYUYV>, (void*)yolo::letterbox_h_yuv_kernel<kYuvUYVY>,
    (void*)yolo::letterbox_h_ragged_yuv_kernel<kYuvYUYV>, (void*)yolo::letterbox_h_ragged_yuv_kernel<kYuvUYVY>,
    (void*)yuv_to_bgr_kernel<kYuvNV12>, (void*)yuv_to_bgr_kernel<kYuvI420>,
    (void*)yuv_to_bgr_kernel<kYuvYUYV>, (void*)yuv_to_bgr_kernel<kYuvUYVY>,
};
"""


def test_yuv422_and_convert_kernels_do_not_spill():
    from whenet_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "yuv422_inst.cu")
        with open(src, "w") as f:
            f.write(_INST)
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas=-v", "-I", build.CSRC, "-c", "-o", os.path.join(tmp, "y.o"), src],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.split(r"Compiling entry function '", r.stdout + r.stderr)[1:]
    seen = []
    for e in entries:
        name = e.split("'", 1)[0]
        if "yuv" not in name or not (re.search(r"Li[34]E", name) or "yuv_to_bgr" in name):
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.group(1) == "0" and m.group(2) == "0", "%s spills" % name
        if "yuv_to_bgr" in name:
            assert re.search(r"\b0 bytes stack frame", e), "%s has a stack frame" % name
            assert "bytes smem" not in e or re.search(r"\b0 bytes smem", e), "%s uses shared memory" % name
        seen.append(name)
    assert len(seen) == 12, seen
