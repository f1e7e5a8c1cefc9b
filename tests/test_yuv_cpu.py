"""YUV 4:2:0 frames without a GPU: the integer oracle of the conversion against cv2.cvtColor bit for bit, the argument
validation of the four *_yuv_u8 entries (every bad argument is refused, naming it, before anything touches a device), the
pixel_format checks of the Python wrappers, and the new kernel instances as ptxas builds them."""
import ctypes as C
import os
import re
import subprocess
import tempfile
import types

import numpy as np
import pytest

import yuv_oracle as Y

NV12, I420 = 1, 2
CODES = {"nv12": "COLOR_YUV2BGR_NV12", "i420": "COLOR_YUV2BGR_I420"}
SIZES = [(2, 2), (4, 6), (34, 1002), (480, 640), (720, 1280), (1080, 1920), (1920, 1080), (2160, 3840)]


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def P(a):
    return None if a is None else a.ctypes.data


# ----------------------------------------------------------------------------------------------- the conversion
@pytest.mark.parametrize("layout", Y.LAYOUTS)
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_oracle_equals_cv2_on_random_frames(layout, size):
    cv2 = pytest.importorskip("cv2")
    H, W = size
    buf = np.random.default_rng(H * 7919 + W).integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
    assert np.array_equal(Y.yuv420_to_bgr(buf, layout), cv2.cvtColor(buf, getattr(cv2, CODES[layout])))


@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_oracle_equals_cv2_on_the_extremes(layout):
    """Every Y in {0, 16, 235, 255} against every (U, V) in {0, 128, 255}^2, each on its own 2 x 2 block (one chroma sample)."""
    cv2 = pytest.importorskip("cv2")
    combos = [(y, u, v) for y in (0, 16, 235, 255) for u in (0, 128, 255) for v in (0, 128, 255)]
    H, W = 2, 2 * len(combos)
    ys = np.repeat(np.array([c[0] for c in combos], np.uint8), 2)[None].repeat(2, axis=0)
    us = np.array([c[1] for c in combos], np.uint8)[None]
    vs = np.array([c[2] for c in combos], np.uint8)[None]
    chroma = np.stack([us, vs], axis=-1).reshape(1, W) if layout == "nv12" else np.concatenate([us, vs], axis=1)
    buf = np.ascontiguousarray(np.concatenate([ys, chroma]))
    got = Y.yuv420_to_bgr(buf, layout)
    assert np.array_equal(got, cv2.cvtColor(buf, getattr(cv2, CODES[layout])))
    assert got.min() == 0 and got.max() == 255                 # both clips are reached


def test_oracle_planes_and_refusals():
    buf = np.arange(6 * 4, dtype=np.uint8).reshape(6, 4)        # a 4 x 4 frame
    y, u, v = Y.planes(buf, "nv12")
    assert y.shape == (4, 4) and np.array_equal(u, [[16, 18], [20, 22]]) and np.array_equal(v, [[17, 19], [21, 23]])
    y, u, v = Y.planes(buf, "i420")
    assert np.array_equal(u, [[16, 17], [18, 19]]) and np.array_equal(v, [[20, 21], [22, 23]])
    for bad in (np.zeros((5, 4), np.uint8), np.zeros((6, 3), np.uint8), np.zeros((6, 4), np.int16), np.zeros((6, 4, 1), np.uint8)):
        with pytest.raises(ValueError):
            Y.planes(bad, "nv12")
    with pytest.raises(ValueError):
        Y.planes(buf, "nv21")


# ----------------------------------------------------------------------------------------------- C entries
def _det_outputs(n):
    return np.zeros((n, 20, 4), np.float32), np.zeros((n, 20), np.float32), np.zeros((n, 20), np.int32), np.zeros(n, np.int32)


def test_detect_yuv_argument_validation():
    L = _lib()
    frames = np.zeros((2, 12, 8), np.uint8)                     # two 8 x 8 frames
    boxes, scores, classes, counts = _det_outputs(2)

    def call(fr=frames, n=2, H=8, W=8, layout=NV12, out=counts):
        rc = L.whenet_det_detect_yuv_u8(None, P(fr), n, H, W, 0, layout, 0.3, 0.45, 20, P(boxes), P(scores), P(classes), P(out))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null detector")                     # every other argument is fine
    assert call(layout=I420) == (-1, b"null detector")
    for bad in (0, 3, -1):
        assert call(layout=bad) == (-1, b"yuv_layout=%d: WHENET_YUV_NV12 (1) or WHENET_YUV_I420 (2)" % bad)
    assert call(fr=None) == (-1, b"null frames")
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d outside [1, 64]" % n)
    for H, W in ((7, 8), (8, 7), (0, 8), (8, 0), (16386, 8), (8, 16386)):
        rc, msg = call(H=H, W=W)
        assert rc == -1 and msg == b"frame size %dx%d: a 4:2:0 frame has even sides in [2, 16384]" % (W, H), msg
    assert call(H=16384, W=2) == (-1, b"null detector")
    assert call(out=None) == (-1, b"null output pointer")


def test_detect_ragged_yuv_argument_validation():
    L = _lib()
    keep = [np.zeros((12, 8), np.uint8), np.zeros((9, 10), np.uint8)]
    ptrs = (C.c_void_p * 2)(*(f.ctypes.data for f in keep))
    hw = np.array([8, 8, 6, 10], np.int32)
    boxes, scores, classes, counts = _det_outputs(2)

    def call(fr=ptrs, hw=hw, n=2, layout=I420, out=counts):
        rc = L.whenet_det_detect_ragged_yuv_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, layout, 0.3, 0.45, 20,
                                               P(boxes), P(scores), P(classes), P(out))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null detector")
    for bad in (0, 3):
        assert call(layout=bad) == (-1, b"yuv_layout=%d: WHENET_YUV_NV12 (1) or WHENET_YUV_I420 (2)" % bad)
    assert call(fr=None) == (-1, b"null frames or hw")
    assert call(hw=None) == (-1, b"null frames or hw")
    for n in (0, 65):
        assert call(n=n) == (-1, b"n=%d outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(ptrs[0], None)) == (-1, b"frame 1 is NULL")
    for bad in ((7, 8), (8, 9)):
        rc, msg = call(hw=np.array([8, 8] + list(bad), np.int32))
        assert rc == -1 and msg == b"frame 1: frame size %dx%d: a 4:2:0 frame has even sides" % (bad[1], bad[0]), msg
    assert call(hw=np.array([8, 8, 16386, 8], np.int32)) == (-1, b"frame 1: bad frame size 8x16386")
    assert call(out=None) == (-1, b"null output pointer")


def test_crop_boxes_yuv_argument_validation():
    L = _lib()
    frames = np.zeros((2, 12, 8), np.uint8)
    boxes = np.array([[1, 1, 6, 6], [0, 0, 8, 8]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)

    def call(fr=frames, n=2, H=8, W=8, bx=boxes, f=fo, m=2, layout=NV12, crops=out):
        rc = L.whenet_crop_boxes_yuv_u8(None, P(fr), n, H, W, 0, P(bx), P(f), m, layout, P(crops), None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")
    for bad in (0, 3):
        assert call(layout=bad) == (-1, b"yuv_layout=%d: WHENET_YUV_NV12 (1) or WHENET_YUV_I420 (2)" % bad)
    null_msg = b"null frames, boxes, frame_of or crops_out"
    for kw in ({"fr": None}, {"bx": None}, {"f": None}, {"crops": None}):
        assert call(**kw) == (-1, null_msg), kw
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    for H, W in ((7, 8), (8, 7), (16386, 8), (8, 16386)):
        rc, msg = call(H=H, W=W)
        assert rc == -1 and msg == b"frame size %dx%d: a 4:2:0 frame has even sides of at most 16384" % (H, W), msg
    assert call(H=0, W=8) == (-1, b"bad frame size 0x8")
    assert call(m=0) == (-1, b"m=0 boxes")
    assert call(f=np.array([0, 2], np.int32)) == (-1, b"box 1: frame_of=2 outside [0, 2)")


def test_crop_boxes_ragged_yuv_argument_validation():
    L = _lib()
    keep = [np.zeros((12, 8), np.uint8), np.zeros((9, 10), np.uint8)]
    ptrs = (C.c_void_p * 2)(*(f.ctypes.data for f in keep))
    hw = np.array([8, 8, 6, 10], np.int32)
    boxes = np.array([[1, 1, 6, 6], [0, 0, 6, 10]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)

    def call(fr=ptrs, hw=hw, n=2, bx=boxes, f=fo, m=2, layout=I420, crops=out):
        rc = L.whenet_crop_boxes_ragged_yuv_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, P(bx), P(f), m, layout, P(crops),
                                               None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")
    assert call(layout=5) == (-1, b"yuv_layout=5: WHENET_YUV_NV12 (1) or WHENET_YUV_I420 (2)")
    null_msg = b"null frames, hw, boxes, frame_of or crops_out"
    for kw in ({"fr": None}, {"hw": None}, {"bx": None}, {"f": None}, {"crops": None}):
        assert call(**kw) == (-1, null_msg), kw
    for n in (0, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(None, ptrs[1])) == (-1, b"frame 0 is NULL")
    rc, msg = call(hw=np.array([8, 8, 6, 11], np.int32))
    assert rc == -1 and msg == b"frame 1: frame size 11x6: a 4:2:0 frame has even sides", msg
    assert call(m=0) == (-1, b"m=0 boxes")


# ----------------------------------------------------------------------------------------------- Python wrappers
def _fake_yolo():
    import whenet_b200
    y = whenet_b200.YOLO.__new__(whenet_b200.YOLO)
    y.device, y.max_frames = 0, 8
    return y


def test_wrappers_refuse_bad_yuv_frames_and_formats():
    from whenet_b200 import pipeline
    y = _fake_yolo()
    y0, w0 = types.SimpleNamespace(device=0), types.SimpleNamespace(device=0)
    bgr = np.zeros((2, 8, 8, 3), np.uint8)
    good = np.zeros((2, 12, 8), np.uint8)
    for fmt in ("nv12", "i420"):
        for bad in (bgr, np.zeros((2, 13, 8), np.uint8), np.zeros((2, 12, 7), np.uint8), np.zeros((12, 8), np.uint8)):
            with pytest.raises(ValueError):
                y.detect_frames(bad, pixel_format=fmt)
            with pytest.raises(ValueError):
                pipeline.detect_and_estimate_frames(y0, w0, bad, pixel_format=fmt)
        with pytest.raises(ValueError, match="frame 1"):
            y.detect_frames([good[0], np.zeros((8, 8, 3), np.uint8)], pixel_format=fmt)
        with pytest.raises(ValueError, match="frame 0"):
            pipeline.detect_and_estimate_frames(y0, w0, [np.zeros((14, 8), np.uint8)], pixel_format=fmt)
        with pytest.raises(ValueError, match="rows"):
            pipeline.detect_and_estimate(y0, w0, np.zeros((13, 8), np.uint8), pixel_format=fmt)
        with pytest.raises(ValueError, match="even width"):
            pipeline.detect_and_estimate(y0, w0, np.zeros((12, 9), np.uint8), pixel_format=fmt)
        assert pipeline.detect_and_estimate_frames(y0, w0, np.zeros((0, 12, 8), np.uint8), pixel_format=fmt) == []
        assert y.detect_frames([], pixel_format=fmt) == []
    for fmt in ("rgb", "NV12", "nv21", None, 1):
        with pytest.raises(ValueError, match="pixel_format"):
            y.detect_frames(good, pixel_format=fmt)
        with pytest.raises(ValueError, match="pixel_format"):
            pipeline.detect_and_estimate_frames(y0, w0, good, pixel_format=fmt)
        with pytest.raises(ValueError, match="pixel_format"):
            pipeline.detect_and_estimate(y0, w0, good[0], pixel_format=fmt)


def test_frame_table_gives_image_sizes():
    from whenet_b200.yolo import _frame_table
    frames = [np.zeros((12, 8), np.uint8), np.zeros((1620, 1920), np.uint8)]
    _ptrs, hw = _frame_table(frames, NV12)
    assert hw.tolist() == [8, 8, 1080, 1920]


# ----------------------------------------------------------------------------------------------- ptxas
_INST = """
#include "kernels_crop.cuh"
#include "kernels_yolo.cuh"
using namespace whenet;
void* yuv_instances[] = {
    (void*)crop_resize_yuv_kernel<OneSizeFrames, kYuvNV12>, (void*)crop_resize_yuv_kernel<OneSizeFrames, kYuvI420>,
    (void*)crop_resize_yuv_kernel<PerFrameSources, kYuvNV12>, (void*)crop_resize_yuv_kernel<PerFrameSources, kYuvI420>,
    (void*)yolo::letterbox_h_yuv_kernel<kYuvNV12>, (void*)yolo::letterbox_h_yuv_kernel<kYuvI420>,
    (void*)yolo::letterbox_h_ragged_yuv_kernel<kYuvNV12>, (void*)yolo::letterbox_h_ragged_yuv_kernel<kYuvI420>,
};
"""


def test_yuv_kernels_do_not_spill():
    from whenet_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "yuv_inst.cu")
        with open(src, "w") as f:
            f.write(_INST)
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas=-v", "-I", build.CSRC, "-c", "-o", os.path.join(tmp, "y.o"), src],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.split(r"Compiling entry function '", r.stdout + r.stderr)[1:]
    seen = []
    for e in entries:
        name = e.split("'", 1)[0]
        if "yuv" not in name:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.group(1) == "0" and m.group(2) == "0", "%s spills" % name
        seen.append(name)
    assert len(seen) == 8, seen
