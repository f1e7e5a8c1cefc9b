"""GPU JPEG encoding (``video.encode_jpeg``, DESIGN.md section 8.9): every file equals cv2.imencode's bytes, at any batch size,
for ragged lists, host or device frames, on a context whose buffers grow and shrink, and after the detect, estimate and draw
chain."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_jpeg_cpu import KINDS, SIZES, cv2_jpeg, frame  # noqa: E402

pytestmark = pytest.mark.gpu
QS = [1, 50, 95, 100]


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _dev(frames):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.stack(frames))).cuda()


def _check(got, frames, q):
    assert len(got) == len(frames)
    for i, (g, f) in enumerate(zip(got, frames)):
        assert g == cv2_jpeg(f, q), (i, f.shape, q)


@pytest.mark.parametrize("h,w", SIZES + [(1081, 1921), (720, 1280), (1080, 1920)])
def test_equals_cv2(wn, h, w):
    from whenet_b200 import video
    frames = [frame(kind, h, w, seed=k) for k, kind in enumerate(KINDS)]
    dev = _dev(frames)
    for q in QS:
        _check(video.encode_jpeg(wn, dev, q), frames, q)


def test_equals_cv2_on_sample_crops(wn, sample_crops):
    from whenet_b200 import video
    frames = [np.ascontiguousarray(c) for c in sample_crops]
    for q in [1, 10, 49, 50, 51, 75, 94, 95, 100]:
        _check(video.encode_jpeg(wn, _dev(frames), q), frames, q)


@pytest.mark.parametrize("h,w,kinds", [(2160, 3840, ["noise", "gradient"]), (4096, 4096, ["noise"]), (16384, 24, KINDS),
                                       (24, 16384, KINDS)])
def test_equals_cv2_large(wn, h, w, kinds):
    from whenet_b200 import video
    frames = [frame(kind, h, w, seed=k) for k, kind in enumerate(kinds)]
    dev = _dev(frames)
    for q in QS:
        _check(video.encode_jpeg(wn, dev, q), frames, q)


@pytest.mark.parametrize("n", [1, 8, 64, 65])
def test_batches(wn, n):
    """n frames in one call (65: two groups); each frame's bytes are its own, alone or in the batch."""
    from whenet_b200 import video
    frames = [frame(KINDS[i % 4], 48, 64, seed=i) for i in range(n)]
    got = video.encode_jpeg(wn, _dev(frames), 95)
    _check(got, frames, 95)
    for i in {0, n // 2, n - 1}:
        assert video.encode_jpeg(wn, _dev(frames[i:i + 1]), 95)[0] == got[i]


def test_ragged_host_and_device(wn):
    """A list of frames of mixed sizes, as device tensors and as host arrays: the same bytes, equal to cv2's, and equal to
    each frame encoded alone."""
    import torch
    from whenet_b200 import video
    rng = np.random.default_rng(5)
    shapes = [(1, 1), (17, 33), (480, 640), (8, 8), (1081, 1921), (37, 53), (224, 224), (1, 300), (301, 1)]
    frames = [frame(KINDS[i % 4], h, w, seed=i) for i, (h, w) in enumerate(shapes)]
    order = rng.permutation(len(frames))
    frames = [frames[i] for i in order]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    for q in (1, 95):
        got = video.encode_jpeg(wn, dev, q)
        _check(got, frames, q)
        assert video.encode_jpeg(wn, frames, q) == got
        assert video.encode_jpeg(wn, np.stack([frames[1]] * 3), q) == [got[1]] * 3
        for i in range(len(frames)):
            assert video.encode_jpeg(wn, [dev[i]], q)[0] == got[i]


@pytest.mark.parametrize("order", ["grow_then_shrink", "shrink_then_grow"])
def test_buffers_grow_and_shrink(order):
    """A fresh context per order: the scratch buffers grow with the call and later, smaller calls reuse them."""
    import whenet_b200
    from whenet_b200 import video
    sizes = [(16, 16, 1), (120, 200, 8), (1080, 1920, 4), (2160, 3840, 2), (64, 48, 64), (8, 8, 1)]
    if order == "shrink_then_grow":
        sizes = sizes[::-1]
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    try:
        for k, (h, w, n) in enumerate(sizes):
            frames = [frame(KINDS[(i + k) % 4], h, w, seed=i + k) for i in range(n)]
            _check(video.encode_jpeg(m, _dev(frames), 95), frames, 95)
    finally:
        m.close()


def test_chain_detect_draw_encode(wn):
    """detect_and_estimate_frames -> draw_heads(display="full") -> encode_jpeg equals cv2.imencode of the annotated frames."""
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    from test_gpu_yolo import _frame
    yolo = whenet_b200.YOLO(None, max_frames=4, score=0.0)
    frames = np.stack([_frame(480, 640, seed=s) for s in range(3)])
    dev = torch.from_numpy(frames).cuda()
    res = pipeline.detect_and_estimate_frames(yolo, wn, dev)
    assert sum(len(r[0]) for r in res) > 0
    overlay.draw_heads(wn, dev, res, display="full")
    got = video.encode_jpeg(wn, dev)
    _check(got, list(dev.cpu().numpy()), 95)


def test_argument_checks(wn):
    """Each bad argument raises ValueError before any device work; n = 0 gives []."""
    import torch
    from whenet_b200 import video
    good = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device="cuda")
    bad = [
        lambda: video.encode_jpeg(wn, good, 0),
        lambda: video.encode_jpeg(wn, good, 101),
        lambda: video.encode_jpeg(wn, good, 95.0),
        lambda: video.encode_jpeg(wn, good.float()),
        lambda: video.encode_jpeg(wn, torch.zeros((2, 8, 16, 3), dtype=torch.uint8, device="cuda")[:, :, ::2]),
        lambda: video.encode_jpeg(wn, good.cpu()),
        lambda: video.encode_jpeg(wn, torch.zeros((1, 16385, 1, 3), dtype=torch.uint8, device="cuda")),
        lambda: video.encode_jpeg(wn, [good[0], torch.zeros((1, 16385, 3), dtype=torch.uint8, device="cuda")]),
        lambda: video.encode_jpeg(wn, [good[0], np.zeros((8, 8, 3), np.uint8)]),
        lambda: video.encode_jpeg(wn, good[..., :2].contiguous()),
        lambda: video.encode_jpeg(wn, np.zeros((8, 8, 3), np.uint8)),
        lambda: video.encode_jpeg(wn, np.zeros((1, 8, 8, 3), np.int16)),
    ]
    if torch.cuda.device_count() > 1:
        bad.append(lambda: video.encode_jpeg(wn, good.to("cuda:1")))
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    assert video.encode_jpeg(wn, good[:0]) == []
    assert video.encode_jpeg(wn, []) == []
