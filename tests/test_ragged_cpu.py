"""Frames of several sizes without a GPU: the argument validation of whenet_det_detect_ragged_u8 and
whenet_crop_boxes_ragged_u8 (every bad argument is refused, naming it, before anything touches a device), and the frame-list
checks of YOLO.detect_frames and pipeline.detect_and_estimate_frames."""
import ctypes as C
import types

import numpy as np
import pytest

from test_pipeline_cpu import _FakeCudaFrames


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def P(a):
    return None if a is None else a.ctypes.data


def _frames(sizes):
    frames = [np.zeros((h, w, 3), np.uint8) for h, w in sizes]
    ptrs = (C.c_void_p * len(frames))(*(f.ctypes.data for f in frames))
    return frames, ptrs, np.array(sizes, np.int32).reshape(-1)


def test_detect_ragged_argument_validation():
    L = _lib()
    keep, ptrs, hw = _frames([(8, 8), (6, 10)])
    boxes = np.zeros((2, 20, 4), np.float32)
    scores = np.zeros((2, 20), np.float32)
    classes = np.zeros((2, 20), np.int32)
    counts = np.zeros(2, np.int32)

    def call(fr=ptrs, hw=hw, n=2, out=counts):
        rc = L.whenet_det_detect_ragged_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, 1, 0.3, 0.45, 20, P(boxes), P(scores),
                                           P(classes), P(out))
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null detector")                     # every other argument is fine
    assert call(fr=None) == (-1, b"null frames or hw")
    assert call(hw=None) == (-1, b"null frames or hw")
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d outside [1, 64]" % n)
    null_one = (C.c_void_p * 2)(ptrs[0], None)
    assert call(fr=null_one) == (-1, b"frame 1 is NULL")
    for bad in ((0, 8), (8, 0), (-3, 8), (16385, 8), (8, 16385)):
        rc, msg = call(hw=np.array([8, 8] + list(bad), np.int32))
        assert rc == -1 and msg == b"frame 1: bad frame size %dx%d" % (bad[1], bad[0]), msg
    assert call(hw=np.array([16384, 1, 1, 16384], np.int32)) == (-1, b"null detector")
    assert call(out=None) == (-1, b"null output pointer")


def test_crop_boxes_ragged_argument_validation():
    L = _lib()
    keep, ptrs, hw = _frames([(8, 8), (6, 10)])
    boxes = np.array([[1, 1, 6, 6], [0, 0, 6, 10]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)

    def call(fr=ptrs, hw=hw, n=2, bx=boxes, f=fo, m=2, crops=out):
        rc = L.whenet_crop_boxes_ragged_u8(None, None if fr is None else C.addressof(fr), P(hw), n, 0, P(bx), P(f), m, 1, P(crops), None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")                      # every other argument is fine
    null_msg = b"null frames, hw, boxes, frame_of or crops_out"
    for kw in ({"fr": None}, {"hw": None}, {"bx": None}, {"f": None}, {"crops": None}):
        assert call(**kw) == (-1, null_msg), kw
    for n in (0, -1, 65):
        assert call(n=n) == (-1, b"n=%d frames outside [1, 64]" % n)
    assert call(fr=(C.c_void_p * 2)(None, ptrs[1])) == (-1, b"frame 0 is NULL")
    for bad in ((0, 8), (8, 0), (-3, 8), (16385, 8), (8, 16385)):
        rc, msg = call(hw=np.array(list(bad) + [6, 10], np.int32))
        assert rc == -1 and msg == b"frame 0: bad frame size %dx%d" % (bad[1], bad[0]), msg
    assert call(m=0) == (-1, b"m=0 boxes")
    for bad in (2, -1):
        assert call(f=np.array([0, bad], np.int32)) == (-1, b"box 1: frame_of=%d outside [0, 2)" % bad)


class _FakeFrame(_FakeCudaFrames):
    def __init__(self, index, shape=(8, 8, 3), **kw):
        super().__init__(index, shape=shape, **kw)


def _fake_yolo(device=0):
    """A YOLO with nothing behind it: detect_frames must refuse a bad list before it reaches the library."""
    import whenet_b200
    y = whenet_b200.YOLO.__new__(whenet_b200.YOLO)
    y.device, y.max_frames = device, 8
    return y


def test_detect_frames_list_checks():
    import torch
    y = _fake_yolo()
    host = np.zeros((8, 8, 3), np.uint8)
    assert y.detect_frames([]) == [] and y.detect_frames(()) == []
    with pytest.raises(ValueError, match="mix"):
        y.detect_frames([host, _FakeFrame(0)])
    for bad in (np.zeros((8, 8), np.uint8), np.zeros((8, 8, 4), np.uint8), np.zeros((1, 8, 8, 3), np.uint8), np.zeros((8, 8, 3), np.float32),
                np.zeros((0, 8, 3), np.uint8)):
        with pytest.raises(ValueError, match="frame 1"):
            y.detect_frames([host, bad])
    with pytest.raises(ValueError, match="cuda:1"):
        y.detect_frames([_FakeFrame(0), _FakeFrame(1)])
    for bad in (_FakeFrame(0, dtype=torch.float32), _FakeFrame(0, contiguous=False), _FakeFrame(0, shape=(8, 8))):
        with pytest.raises(ValueError, match="frame 0"):
            y.detect_frames([bad])
    with pytest.raises(ValueError):                             # an ndarray keeps its own checks
        y.detect_frames(np.zeros((8, 8, 3), np.uint8))


def test_detect_and_estimate_frames_list_checks():
    import torch
    from whenet_b200 import pipeline
    y0, w0, w1 = (types.SimpleNamespace(device=d) for d in (0, 0, 1))
    host = np.zeros((8, 8, 3), np.uint8)
    assert pipeline.detect_and_estimate_frames(y0, w0, []) == []
    assert pipeline.detect_and_estimate_frames(y0, w0, ()) == []
    with pytest.raises(ValueError, match="device"):
        pipeline.detect_and_estimate_frames(y0, w1, [host])
    with pytest.raises(ValueError, match="mix"):
        pipeline.detect_and_estimate_frames(y0, w0, [_FakeFrame(0), host])
    for bad in (np.zeros((8, 8), np.uint8), np.zeros((8, 8, 3), np.int64), _FakeFrame(0, dtype=torch.float32)):
        with pytest.raises(ValueError, match="frame 0"):
            pipeline.detect_and_estimate_frames(y0, w0, [bad])
    with pytest.raises(ValueError, match="cuda:1"):
        pipeline.detect_and_estimate_frames(y0, w0, [_FakeFrame(1), _FakeFrame(1, shape=(4, 8, 3))])
