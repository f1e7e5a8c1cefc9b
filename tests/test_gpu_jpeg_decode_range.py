"""GPU JPEG decoding of coefficients outside an encoder's range (DESIGN.md section 8.10): the synthetic files of
jpeg_coef_writer.py through ``video.decode_jpeg`` equal the numpy IDCT model always, and cv2.imdecode where cv2 runs
libjpeg-turbo's x86-64 SIMD IDCT.  Files run alone, in batches of 64 mixed with ordinary cv2 files, with restart intervals,
at 32-bit subsequences, and at 1080p, so that jd_idct_kernel's grid covers many blocks of every IDCT path."""
import os
import platform
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import jpeg_coef_writer as W  # noqa: E402
from test_jpeg_cpu import KINDS, frame  # noqa: E402
from test_jpeg_decode_cpu import encode, imdecode  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import jpeg_decode_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
X86 = platform.machine().lower() in ("x86_64", "amd64")


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _check(wn, files, models=None):
    from whenet_b200 import video
    got = video.decode_jpeg(wn, files)
    assert len(got) == len(files)
    for i, (g, f) in enumerate(zip(got, files)):
        g = g.cpu().numpy()
        model = O.decode(f) if models is None or models[i] is None else models[i]
        assert g.shape == model.shape and np.array_equal(g, model), i
        if X86:
            assert np.array_equal(g, imdecode(f)), i


@pytest.mark.parametrize("sampling", list(W.SAMPLING))
def test_matrix_alone(wn, sampling):
    for name, f in W.matrix(sizes=((16, 32), (37, 53)), restarts=(0, 1), seed=5):
        if "-%s-" % sampling in name:
            _check(wn, [f])


def test_batches_mixed_with_encoder_files(wn):
    """Batches of 64: synthetic files of every kind and sampling between ordinary cv2 files, with restart intervals."""
    synth = W.matrix(sizes=((24, 40), (57, 31)), restarts=(0, 2), seed=6)
    rng = np.random.default_rng(6)
    files = []
    for i, (_, f) in enumerate(synth):
        files.append(f)
        if i % 3 == 0:
            h, w = int(rng.integers(8, 90)), int(rng.integers(8, 90))
            files.append(encode(frame(KINDS[i % 4], h, w, seed=i), int(rng.integers(1, 101)), ["420", "422", "444", "gray"][i % 4],
                                rst=i % 3))
    assert len(files) > 128
    for lo in range(0, len(files), 64):
        _check(wn, files[lo:lo + 64])


def test_short_subsequences(wn):
    from whenet_b200._lib import check
    files = [f for _, f in W.matrix(sizes=((37, 53),), restarts=(0, 3), seed=7)]
    check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 32))
    try:
        for lo in range(0, len(files), 64):
            _check(wn, files[lo:lo + 64])
    finally:
        check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 0))


@pytest.mark.parametrize("sampling", ["420", "422"])
def test_clamped_chroma_through_fancy_upsampling(wn, sampling):
    """Chroma blocks that saturate to 0 and 255 next to each other (alternating DC-only blocks past the shortcut's wrap, and
    dense ones), so the upsampler's neighbours are the clamped and wrapped samples; luma mid-range."""
    for seed, restart in ((0, 0), (1, 2)):
        rng = np.random.default_rng(seed)
        grids = W.grid(48, 80, sampling)
        blocks = [np.zeros(g + (64,), np.int64) for g in grids]
        blocks[0][..., 1:] = rng.integers(-2, 3, blocks[0][..., 1:].shape)
        for c in (1, 2):
            b = blocks[c]
            b[..., 0] = np.where((np.indices(b.shape[:2]).sum(0) % 2) == 0, 1000, -1000) * (1 if c == 1 else -1)
            b[1::2, ..., 1:] = rng.integers(-1023, 1024, b[1::2, ..., 1:].shape)
        q = [np.full(64, 4), np.full(64, 40), rng.integers(1, 256, 64)]
        f = W.write(blocks, q, 48, 80, sampling, restart)
        _, coef = O.coefficients(f)
        px = O.idct_islow(coef[1].reshape(-1, 64), q[1])
        assert px.min() == 0 and px.max() == 255
        _check(wn, [f])


def test_1080p_extreme_coefficients(wn):
    """Full-HD files of extreme coefficients: 32,400 luma blocks each through jd_idct_kernel."""
    files = [W.synthetic(k, 1080, 1920, s, r, seed=8)[0]
             for k, s, r in [("dense", "420", 0), ("mixed", "444", 7), ("dc", "422", 5), ("wild", "gray", 0)]]
    models = [O.decode(f) for f in files]
    _check(wn, files, models)
    _check(wn, files[::-1], models[::-1])
