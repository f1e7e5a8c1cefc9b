"""GPU JPEG encoding with options (``video.encode_jpeg(..., sampling=, restart_interval=, optimize=, chroma_quality=)`` and gray
frames, DESIGN.md section 8.11): every file equals cv2.imencode's bytes with the same parameters, at any batch size, for
ragged lists and host frames, independently of the rest of its batch; the files decode back on the GPU as cv2 decodes cv2's;
they pass through the MJPG writer and reader; and the device optimal-table builder equals the oracle."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_jpeg_cpu import KINDS, frame  # noqa: E402
from test_jpeg_options_cpu import HISTOGRAMS, OPTION_SETS, SAMPLINGS, SIZES, cv2_file, optimal_table, option_image  # noqa: E402

import jpeg_options_oracle as J  # noqa: E402

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


def _opts(sampling, q, r, o):
    return dict(quality=q, sampling="420" if sampling == "gray" else sampling, restart_interval=r, optimize=o)


def _encode_check(wn, frames, opts):
    from whenet_b200 import video
    kw = dict(opts)
    q = kw.pop("quality")
    got = video.encode_jpeg(wn, _dev(frames), q, **kw)
    assert len(got) == len(frames)
    for i, (g, f) in enumerate(zip(got, frames)):
        assert g == cv2_file(f, **opts), (i, f.shape, opts)
    return got


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("h,w", SIZES)
def test_equals_cv2(wn, h, w, sampling):
    for q, r, o in OPTION_SETS:
        frames = [option_image(kind, h, w, sampling, seed=q + k) for k, kind in enumerate(KINDS)]
        _encode_check(wn, frames, _opts(sampling, q, r, o))


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("h,w", [(720, 1280), (1080, 1920), (1081, 1921), (2160, 3840)])
def test_equals_cv2_video_sizes(wn, h, w, sampling):
    frames = [option_image(kind, h, w, sampling, seed=k) for k, kind in enumerate(["noise", "gradient"])]
    for r in (0, 7):
        for o in (False, True):
            _encode_check(wn, frames, _opts(sampling, 95, r, o))


@pytest.mark.parametrize("q,cq", [(90, 40), (40, 90)])
def test_two_qualities(wn, q, cq):
    for h, w in [(37, 53), (1080, 1920)]:
        frames = [frame(kind, h, w, seed=k) for k, kind in enumerate(KINDS)]
        for o in (False, True):
            _encode_check(wn, frames, dict(quality=q, sampling="444", optimize=o, chroma_quality=cq))


@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_restart_every_mcu_1080p(wn, sampling):
    frames = [option_image("noise", 1080, 1920, sampling, seed=1), option_image("gradient", 1080, 1920, sampling, seed=2)]
    for o in (False, True):
        _encode_check(wn, frames, _opts(sampling, 95, 1, o))


@pytest.mark.parametrize("h,w,sampling", [(4096, 4096, "420"), (4096, 4096, "444"), (4096, 4096, "gray"), (16384, 24, "422"),
                                          (24, 16384, "444"), (16384, 24, "gray"), (24, 16384, "420")])
def test_equals_cv2_large(wn, h, w, sampling):
    frames = [option_image("noise", h, w, sampling, seed=5)]
    _encode_check(wn, frames, _opts(sampling, 95, 0, True))
    if h != w:
        _encode_check(wn, frames, _opts(sampling, 50, 3, False))


@pytest.mark.parametrize("n", [1, 8, 64, 65])
def test_batches(wn, n):
    rng = np.random.default_rng(n)
    for sampling in ("444", "gray"):
        frames = [option_image(KINDS[i % 4], 24, 40, sampling, seed=int(rng.integers(1 << 30))) for i in range(n)]
        _encode_check(wn, frames, _opts(sampling, 90, 2, True))


def test_ragged_host_and_device_and_independence(wn):
    """A ragged list on the device, the same as host arrays, and each frame alone: all equal cv2.  With per-frame optimised
    tables, each frame alone against inside the batch catches one frame's histogram or table leaking into another's."""
    import torch
    from whenet_b200 import video
    sizes = [(1, 1), (17, 33), (120, 200), (7, 15), (1081, 1921), (37, 53), (16, 16)]
    for sampling in SAMPLINGS:
        for q, r, o in [(95, 0, True), (50, 1, True), (75, 5, False)]:
            opts = _opts(sampling, q, r, o)
            kw = dict(opts)
            kw.pop("quality")
            host = [option_image(KINDS[i % 4], h, w, sampling, seed=i) for i, (h, w) in enumerate(sizes)]
            dev = [torch.from_numpy(f).cuda() for f in host]
            got = video.encode_jpeg(wn, dev, q, **kw)
            assert got == [cv2_file(f, **opts) for f in host], opts
            assert video.encode_jpeg(wn, host, q, **kw) == got, opts
            for f, g in zip(dev, got):
                assert video.encode_jpeg(wn, [f], q, **kw) == [g], opts


def test_round_trip_through_gpu_decoder(wn):
    """decode_jpeg of every option set's file equals cv2.imdecode of cv2's file."""
    import cv2
    from whenet_b200 import video
    for sampling in SAMPLINGS:
        for q, r, o in [(95, 0, False), (95, 1, True), (30, 4, True), (100, 0, True)]:
            opts = _opts(sampling, q, r, o)
            kw = dict(opts)
            kw.pop("quality")
            host = [option_image(kind, 61, 97, sampling, seed=q + k) for k, kind in enumerate(KINDS)]
            files = video.encode_jpeg(wn, host, q, **kw)
            dec = video.decode_jpeg(wn, files)
            for f, d, img in zip(files, dec, host):
                ref = cv2.imdecode(np.frombuffer(cv2_file(img, **opts), np.uint8), cv2.IMREAD_COLOR)
                assert np.array_equal(d.cpu().numpy(), ref), opts
    for cq in (40, 90):
        host = [frame("noise", 61, 97, seed=cq)]
        files = video.encode_jpeg(wn, host, 70, sampling="444", chroma_quality=cq, optimize=True)
        ref = cv2.imdecode(np.frombuffer(cv2_file(host[0], quality=70, sampling="444", optimize=True, chroma_quality=cq), np.uint8),
                           cv2.IMREAD_COLOR)
        assert np.array_equal(video.decode_jpeg(wn, files)[0].cpu().numpy(), ref)


def test_avi_round_trip(wn, tmp_path):
    import cv2
    from whenet_b200 import video
    H, W = 72, 128
    src = [frame(KINDS[i % 4], H, W, seed=i) for i in range(6)]
    sets = [dict(sampling="444", optimize=True), dict(restart_interval=1), dict(sampling="422", restart_interval=5, optimize=True),
            dict(sampling="444", chroma_quality=40)]
    files = []
    for kw in sets:
        files += video.encode_jpeg(wn, src[:2], 90, **kw)
    files += video.encode_jpeg(wn, [np.ascontiguousarray(f[..., 1:2]) for f in src[:2]], 90, optimize=True)
    path = str(tmp_path / "opts.avi")
    with video.MJPGWriter(path, 30, (W, H)) as w:
        w.write(files)
    with video.MJPGReader(path) as r:
        got = r.read_frames(wn, len(files))
    assert len(got) == len(files)
    for f, d in zip(files, got):
        assert np.array_equal(d.cpu().numpy(), cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR))


def test_chain_detect_draw_encode(wn):
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    H, W = 480, 640
    frames = [frame("gradient", H, W, seed=s) for s in range(3)]
    dev = _dev(frames)
    yolo = whenet_b200.YOLO(None, max_frames=4)
    res = pipeline.detect_and_estimate_frames(yolo, wn, dev)
    overlay.draw_heads(wn, dev, res, display="full")
    got = video.encode_jpeg(wn, dev, 95, sampling="444", optimize=True)
    host = dev.cpu().numpy()
    assert got == [cv2_file(host[i], quality=95, sampling="444", optimize=True) for i in range(3)]


def test_argument_checks(wn):
    import torch
    from whenet_b200 import video
    f = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device="cuda")
    g = torch.zeros((2, 8, 8, 1), dtype=torch.uint8, device="cuda")
    for kw in [dict(sampling="411"), dict(restart_interval=65536), dict(optimize=None), dict(chroma_quality=40)]:
        with pytest.raises(ValueError):
            video.encode_jpeg(wn, f, 95, **kw)
    with pytest.raises(ValueError):
        video.encode_jpeg(wn, g, 95, sampling="422")
    with pytest.raises(ValueError):
        video.encode_jpeg(wn, [f[0], g[0]], 95)
    assert video.encode_jpeg(wn, g, 95) == [cv2_file(g[i].cpu().numpy()) for i in range(2)]


@pytest.mark.parametrize("name", sorted(HISTOGRAMS))
def test_device_optimal_table_equals_oracle(wn, name):
    from whenet_b200 import _lib
    counts = HISTOGRAMS[name]
    assert optimal_table(_lib.load(), counts, wn._h) == J.gen_optimal_table(counts)
