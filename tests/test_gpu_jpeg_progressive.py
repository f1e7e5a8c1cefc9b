"""GPU progressive JPEG encoding (``video.encode_jpeg(..., progressive=True)``, DESIGN.md section 8.12): every file equals
cv2.imencode's bytes with IMWRITE_JPEG_PROGRESSIVE 1 and the same options, from 1x1 to 4096x4096 and 16384-long strips, with
restart intervals down to one block, at both EOB run caps, at any batch size, for ragged lists and host frames, independently
of the rest of its batch, and at the end of the detect -> draw -> encode chain."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_jpeg_cpu import KINDS, frame  # noqa: E402
from test_jpeg_options_cpu import SAMPLINGS, SIZES, option_image  # noqa: E402
from test_jpeg_progressive_cpu import PROG_SETS, be_cap_frame, cv2_prog  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _dev(frames):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.stack(frames))).cuda()


def _opts(sampling, q, r, **kw):
    return dict(quality=q, sampling="420" if sampling == "gray" else sampling, restart_interval=r, **kw)


def _check(wn, frames, opts, device=True):
    from whenet_b200 import video
    kw = dict(opts)
    q = kw.pop("quality")
    got = video.encode_jpeg(wn, _dev(frames) if device else frames, q, progressive=True, **kw)
    assert len(got) == len(frames)
    for i, (g, f) in enumerate(zip(got, frames)):
        assert g == cv2_prog(f, **opts), (i, f.shape, opts)
    return got


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("h,w", SIZES)
def test_equals_cv2(wn, h, w, sampling):
    for q, r in PROG_SETS:
        frames = [option_image(kind, h, w, sampling, seed=q + k) for k, kind in enumerate(KINDS)]
        _check(wn, frames, _opts(sampling, q, r))


@pytest.mark.parametrize("q,cq", [(90, 40), (40, 90)])
def test_two_qualities(wn, q, cq):
    for h, w in [(37, 53), (1080, 1920)]:
        frames = [frame(kind, h, w, seed=k) for k, kind in enumerate(KINDS)]
        for r in (0, 3):
            _check(wn, frames, dict(quality=q, sampling="444", restart_interval=r, chroma_quality=cq))


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("h,w", [(720, 1280), (1080, 1920), (1081, 1921), (2160, 3840)])
def test_equals_cv2_video_sizes(wn, h, w, sampling):
    frames = [option_image(kind, h, w, sampling, seed=k) for k, kind in enumerate(["noise", "gradient"])]
    for r in (0, 120):
        _check(wn, frames, _opts(sampling, 95, r))


@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_restart_every_mcu_1080p(wn, sampling):
    """restart_interval=1: every block of a one-component scan is its own segment (32,400 per AC scan at 4:4:4)"""
    frames = [option_image("noise", 1080, 1920, sampling, seed=1), option_image("gradient", 1080, 1920, sampling, seed=2)]
    _check(wn, frames, _opts(sampling, 95, 1))


@pytest.mark.parametrize("h,w,sampling", [(4096, 4096, "420"), (4096, 4096, "444"), (4096, 4096, "gray"), (16384, 24, "422"),
                                          (24, 16384, "444"), (16384, 24, "gray"), (24, 16384, "420")])
def test_equals_cv2_large(wn, h, w, sampling):
    frames = [option_image("noise", h, w, sampling, seed=5)]
    _check(wn, frames, _opts(sampling, 95, 0))
    if h != w:
        _check(wn, frames, _opts(sampling, 50, 3))


def test_eobrun_cap(wn):
    """Flat frames whose AC scans have runs past 0x7FFF empty blocks: 2048x2048 gray (luma) and 2912x2912 4:2:0 (chroma)."""
    gray = np.full((2048, 2048, 1), 77, np.uint8)
    _check(wn, [gray], _opts("gray", 95, 0))
    col = np.empty((2912, 2912, 3), np.uint8)
    col[:] = (40, 160, 90)
    _check(wn, [col], _opts("420", 95, 0))
    _check(wn, [col], _opts("444", 95, 0))


def test_be_cap(wn):
    """Runs of blocks that send only correction bits, flushed at 937 buffered bits, also across restart intervals."""
    img = be_cap_frame()
    for r in (0, 7, 40):
        _check(wn, [img], _opts("gray", 100, r))
    big = np.ascontiguousarray(np.tile(img, (4, 4, 1)))
    _check(wn, [big, img], _opts("gray", 100, 0), device=False)


@pytest.mark.parametrize("n", [1, 8, 64, 65])
def test_batches(wn, n):
    rng = np.random.default_rng(n)
    for sampling in ("420", "444", "gray"):
        frames = [option_image(KINDS[i % 4], 24, 40, sampling, seed=int(rng.integers(1 << 30))) for i in range(n)]
        _check(wn, frames, _opts(sampling, 90, 2))


def test_ragged_host_and_device_and_independence(wn):
    """A ragged list on the device, the same as host arrays, and each frame alone: all equal cv2.  Each frame's scans have
    their own tables, so a frame alone against inside the batch catches one scan's histogram or runs leaking into another."""
    import torch
    from whenet_b200 import video
    sizes = [(1, 1), (17, 33), (120, 200), (7, 15), (1081, 1921), (37, 53), (16, 16)]
    for sampling in SAMPLINGS:
        for q, r in [(95, 0), (50, 1), (75, 5)]:
            opts = _opts(sampling, q, r)
            kw = dict(opts)
            kw.pop("quality")
            host = [option_image(KINDS[i % 4], h, w, sampling, seed=i) for i, (h, w) in enumerate(sizes)]
            dev = [torch.from_numpy(f).cuda() for f in host]
            got = video.encode_jpeg(wn, dev, q, progressive=True, **kw)
            assert got == [cv2_prog(f, **opts) for f in host], opts
            assert video.encode_jpeg(wn, host, q, progressive=True, **kw) == got, opts
            for f, g in zip(dev, got):
                assert video.encode_jpeg(wn, [f], q, progressive=True, **kw) == [g], opts


def test_optimize_ignored_and_baseline_unchanged(wn):
    """optimize does not change a progressive file; the same context then still writes the baseline files."""
    from test_jpeg_options_cpu import cv2_file
    from whenet_b200 import video
    frames = [option_image(kind, 61, 97, "444", seed=k) for k, kind in enumerate(KINDS)]
    a = video.encode_jpeg(wn, frames, 90, sampling="444", progressive=True)
    assert video.encode_jpeg(wn, frames, 90, sampling="444", progressive=True, optimize=True) == a
    assert video.encode_jpeg(wn, frames, 90, sampling="444", optimize=True) == [cv2_file(f, quality=90, sampling="444", optimize=True)
                                                                               for f in frames]
    assert video.encode_jpeg(wn, frames, 90) == [cv2_file(f, quality=90) for f in frames]


def test_chain_detect_draw_encode(wn):
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    H, W = 480, 640
    frames = [frame("gradient", H, W, seed=s) for s in range(3)]
    dev = _dev(frames)
    yolo = whenet_b200.YOLO(None, max_frames=4)
    res = pipeline.detect_and_estimate_frames(yolo, wn, dev)
    overlay.draw_heads(wn, dev, res, display="full")
    got = video.encode_jpeg(wn, dev, 95, sampling="444", progressive=True)
    host = dev.cpu().numpy()
    assert got == [cv2_prog(host[i], quality=95, sampling="444") for i in range(3)]
