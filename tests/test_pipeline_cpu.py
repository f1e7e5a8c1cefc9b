"""Multi-frame pipeline without a GPU: the C++ margin arithmetic of whenet_crop_boxes_u8 against crops.enlarge_box (the numpy
restatement of reference demo_video.py:13-21) on 100,000 boxes including non-finite and out-of-range coordinates, and the
argument validation of whenet_crop_boxes_u8 and pipeline.detect_and_estimate_frames."""
import types

import numpy as np
import pytest

NAN, INF = float("nan"), float("inf")

# (box, H, W) -> enlarge_box as numpy 2 computes it (see the comments of crops.enlarge_bounds)
EXAMPLES = [
    ((NAN, 10, 100, 200), 1080, 1920, (0, 110, 0, 240)),
    ((10, 10, -INF, 200), 1080, 1920, (0, 1080, 0, 240)),     # -inf + inf = NaN, and min(H, NaN) is H
    ((10, 10, INF, 200), 1080, 1920, (0, 1080, 0, 240)),
    ((500.5, 10, 500.9, 200), 1080, 1920, (500, 500, 0, 240)),  # truncates to an empty slice
]


def _lib():
    from whenet_b200 import _lib
    return _lib.load()


def _hook(boxes, H, W):
    boxes = np.ascontiguousarray(boxes, np.float32).reshape(-1, 4)
    rects = np.full((len(boxes), 4), -7, np.int32)
    valid = np.full(len(boxes), -7, np.int32)
    assert _lib().whenet_debug_enlarge_boxes(boxes.ctypes.data, len(boxes), H, W, rects.ctypes.data, valid.ctypes.data) == 0
    return rects, valid


def _reference(box, H, W):
    """crops.enlarge_box and the slice predicate of whenet_crop_resize_u8 on its integers."""
    from whenet_b200 import crops
    with np.errstate(all="ignore"):             # inf - inf and overflow are part of the cases
        r = crops.enlarge_box(box, H, W)
    return r, (0 <= r[0] < r[1] <= H and 0 <= r[2] < r[3] <= W)


def _boxes(rng, H, W, k):
    """k boxes of an H x W frame: inside, straddling, outside, zero-area, sub-pixel, on integer and .5 corners, with +-0,
    NaN, +-inf and values >= 2^31 dropped into single coordinates."""
    kind = rng.integers(0, 6, k)
    span = np.array([H, W, H, W], np.float64)
    lo = rng.uniform(0, 1, (k, 2)) * span[:2]
    ext = rng.uniform(0, 1, (k, 2)) * span[:2]
    b = np.concatenate([lo, lo + ext], 1)                               # inside (or up to the far border)
    s = kind == 1                                                      # straddling a border
    b[s] = rng.uniform(-0.5, 1.5, (s.sum(), 4)) * span
    s = kind == 2                                                      # fully outside
    b[s] = rng.uniform(1.01, 3, (s.sum(), 4)) * span * rng.choice([-1, 1], (s.sum(), 1))
    s = kind == 3                                                      # zero area
    b[s, 2] = b[s, 0]
    s = kind == 4                                                      # sub-pixel: truncates to an empty slice
    b[s, 2] = b[s, 0] + rng.uniform(0, 0.6, s.sum())
    b[s, 3] = b[s, 1] + rng.uniform(0, 0.6, s.sum())
    s = kind == 5                                                      # integer and .5 corners
    b[s] = np.round(b[s] * 2) / 2
    special = np.array([0.0, -0.0, NAN, INF, -INF, 2.0 ** 31, 2.0 ** 31 + 2 ** 8, -(2.0 ** 31), 1e30, -1e30, 3.4e38, -3.4e38, 2e9])
    hit = rng.random((k, 4)) < 0.04
    b[hit] = rng.choice(special, hit.sum())
    return b.astype(np.float32)


def test_examples():
    from whenet_b200 import crops
    for box, H, W, want in EXAMPLES:
        assert _reference(box, H, W)[0] == want
        rects, valid = _hook(box, H, W)
        ok = want[0] < want[1]
        assert valid[0] == ok and (not ok or tuple(rects[0]) == want), (box, rects, valid)
    big = crops.enlarge_box((1e30, 10, 2e30, 200), 1080, 1920)        # far beyond int32: invalid, and nothing is cast
    assert big[0] > 2 ** 31
    assert _hook((1e30, 10, 2e30, 200), 1080, 1920)[1][0] == 0


def test_enlarge_hook_equals_enlarge_box_on_100k_boxes():
    rng = np.random.default_rng(7)
    sizes = [(1, 1), (1, 3840), (2160, 1), (2, 2), (1080, 1920), (2160, 3840), (720, 1280), (300, 1200)]
    sizes += [(int(rng.integers(1, 2161)), int(rng.integers(1, 3841))) for _ in range(192)]
    total = n_valid = 0
    for H, W in sizes:
        boxes = _boxes(rng, H, W, 500)
        rects, valid = _hook(boxes, H, W)
        for i, b in enumerate(boxes):
            r, ok = _reference(b, H, W)
            assert bool(valid[i]) == ok, (b, H, W, r)
            if ok:
                assert tuple(rects[i]) == r, (b, H, W, r, rects[i])
        total += len(boxes)
        n_valid += int(valid.sum())
    assert total == 100_000
    assert 0.2 < n_valid / total < 0.9          # both outcomes are well represented


def test_crop_boxes_argument_validation():
    L = _lib()
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    boxes = np.array([[1, 1, 6, 6], [0, 0, 8, 8]], np.float32)
    fo = np.array([0, 1], np.int32)
    out = np.zeros((2, 224, 224, 3), np.uint8)
    P = lambda a: None if a is None else a.ctypes.data   # noqa: E731

    def call(ctx=None, fr=frames, n=2, H=8, W=8, bx=boxes, f=fo, m=2):
        rc = L.whenet_crop_boxes_u8(ctx, P(fr), n, H, W, 0, P(bx), P(f), m, 1, P(out), None, None)
        return rc, L.whenet_last_error()

    assert call() == (-1, b"null context")                    # every other argument is fine
    assert call(fr=None)[0] == -1 and b"null frames" in call(fr=None)[1]
    assert call(bx=None)[0] == -1 and b"null frames" in call(bx=None)[1]
    for n in (0, -1, 65):
        rc, msg = call(n=n)
        assert rc == -1 and msg.startswith(b"n=%d" % n), msg
    for H, W in ((0, 8), (8, 0), (-3, 8)):
        rc, msg = call(H=H, W=W)
        assert rc == -1 and b"frame size" in msg, msg
    assert call(m=0) == (-1, b"m=0 boxes")
    for bad in (2, -1):
        rc, msg = call(f=np.array([0, bad], np.int32))
        assert rc == -1 and msg == b"box 1: frame_of=%d outside [0, 2)" % bad, msg
    assert L.whenet_debug_enlarge_boxes(None, 1, 8, 8, None, None) == -1
    assert L.whenet_debug_enlarge_boxes(P(boxes), 0, 8, 8, None, None) == -1
    assert L.whenet_debug_enlarge_boxes(P(boxes), 1, 0, 8, None, None) == -1


class _FakeCudaFrames:
    """Just enough of a CUDA uint8 tensor for the argument checks (no GPU is touched)."""

    def __init__(self, index, dtype=None, contiguous=True, shape=(2, 8, 8, 3)):
        import torch
        self.is_cuda = True
        self.device = torch.device("cuda", index)
        self.dtype = torch.uint8 if dtype is None else dtype
        self.shape = shape
        self._contiguous = contiguous

    def is_contiguous(self):
        return self._contiguous


def test_detect_and_estimate_frames_argument_validation():
    import torch
    from whenet_b200 import pipeline
    y0, w0, w1 = (types.SimpleNamespace(device=d) for d in (0, 0, 1))
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="device"):
        pipeline.detect_and_estimate_frames(y0, w1, frames)
    for bad in (np.zeros((8, 8, 3), np.uint8), np.zeros((2, 8, 8, 4), np.uint8), np.zeros((2, 8, 8), np.uint8),
                np.zeros((2, 8, 8, 3), np.float32), np.zeros((2, 8, 8, 3), np.int64)):
        with pytest.raises(ValueError):
            pipeline.detect_and_estimate_frames(y0, w0, bad)
    with pytest.raises(ValueError, match="cuda:1"):
        pipeline.detect_and_estimate_frames(y0, w0, _FakeCudaFrames(1))
    for bad in (_FakeCudaFrames(0, dtype=torch.float32), _FakeCudaFrames(0, contiguous=False), _FakeCudaFrames(0, shape=(2, 8, 8))):
        with pytest.raises(ValueError):
            pipeline.detect_and_estimate_frames(y0, w0, bad)
    assert pipeline.detect_and_estimate_frames(y0, w0, np.zeros((0, 8, 8, 3), np.uint8)) == []
    assert pipeline.detect_and_estimate_frames(y0, w0, _FakeCudaFrames(0, shape=(0, 8, 8, 3))) == []
    with pytest.raises(ValueError, match="H x W x 3"):
        pipeline.detect_and_estimate(y0, w0, np.zeros((8, 8), np.uint8))
