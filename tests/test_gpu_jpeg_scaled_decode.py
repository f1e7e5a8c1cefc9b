"""Reduced and gray GPU JPEG decoding (``video.decode_jpeg(..., reduce=d, gray=...)``, DESIGN.md section 8.13): every frame
equals cv2.imdecode with IMREAD_REDUCED_COLOR_d, IMREAD_GRAYSCALE or IMREAD_REDUCED_GRAYSCALE_d at every size, quality,
sampling and restart setting, at 32-bit subsequences, at any batch size and for ragged lists; coefficient files outside an
encoder's range equal cv2; corrupt files raise naming their frame; and MJPG transcodes at 1/2 scale and gray
round trips through encode_jpeg match the same work fed by cv2."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import jpeg_coef_writer as CW  # noqa: E402
from test_jpeg_cpu import KINDS, SIZES, frame  # noqa: E402
from test_jpeg_decode_cpu import GOLDEN, SAMPLES, SAMPLINGS, encode, strip_dht, with_exif  # noqa: E402
from test_jpeg_scaled_decode_cpu import MODES, imdecode  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import jpeg_scaled_decode_oracle as S  # noqa: E402

pytestmark = pytest.mark.gpu
QS = [1, 50, 95, 100]
REDUCED = [m for m in MODES if m != (1, False)]


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _check(wn, files, d, g, ref=imdecode):
    from whenet_b200 import video
    got = video.decode_jpeg(wn, files, reduce=d, gray=g)
    assert len(got) == len(files)
    for i, (t, f) in enumerate(zip(got, files)):
        r = ref(f, d, g)
        assert t.is_contiguous() and t.device.index == wn.device
        assert tuple(t.shape) == r.shape and np.array_equal(t.cpu().numpy(), r), (d, g, i, r.shape)


@pytest.mark.parametrize("d,g", REDUCED)
def test_equals_cv2_small(wn, d, g):
    files = [encode(frame(kind, h, w, seed=q + k), q, s, rst=r) for h, w in SIZES for q in QS for k, kind in enumerate(KINDS)
             for s in SAMPLINGS for r in (0, 3)]
    files += [encode(frame("noise", h, w, seed=1), 90, s) for h, w in [(1, 17), (17, 1), (7, 15)] for s in SAMPLINGS]
    for lo in range(0, len(files), 64):
        _check(wn, files[lo:lo + 64], d, g)


@pytest.mark.parametrize("h,w", [(1080, 1920), (1081, 1921), (2160, 3840), (4096, 4096)])
def test_equals_cv2_large(wn, h, w):
    files = [encode(frame(kind, h, w, seed=q), q, s, rst=r) for s in SAMPLINGS for q, kind, r in [(95, "noise", 0), (50, "gradient", 7)]]
    for d, g in REDUCED:
        _check(wn, files, d, g)


@pytest.mark.parametrize("h,w", [(16384, 24), (24, 16384)])
def test_equals_cv2_strips(wn, h, w):
    files = [encode(frame("noise", h, w, seed=3), 75, s, rst=5) for s in SAMPLINGS]
    for d, g in REDUCED:
        _check(wn, files, d, g)


def test_fixtures_exif_and_no_dht(wn):
    base = encode(frame("gradient", 40, 66), 90, "422")
    files = [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    files += [with_exif(base, o, be) for o in range(1, 9) for be in (False, True)]
    files += [strip_dht(encode(frame("noise", 37, 53), 75, s)) for s in SAMPLINGS]
    for d, g in REDUCED:
        _check(wn, files, d, g)


def test_coefficient_files_equal_cv2(wn):
    """Coefficient-writer files outside an encoder's range, and the probe blocks of the CPU test: equal to cv2 (and so to
    the model) at every d."""
    from test_jpeg_scaled_decode_cpu import X86, _probe_files
    files = [CW.synthetic(k, h, w, s, r, seed=5)[0] for k in CW.KINDS for s in CW.SAMPLING
             for (h, w), r in [((16, 32), 0), ((37, 53), 3)]]
    for d, g in REDUCED:
        for lo in range(0, len(files), 64):
            _check(wn, files[lo:lo + 64], d, g, ref=imdecode if X86 else S.decode)
    probes = _probe_files()
    for d in (2, 4, 8):
        _check(wn, probes, d, True, ref=imdecode if X86 else S.decode)
        _check(wn, probes, d, True, ref=S.decode)


def test_short_subsequences(wn):
    from whenet_b200._lib import check
    files = [encode(frame(kind, 1080, 1920, seed=2), q, s, rst=r) for kind in ("noise", "gradient") for q in (10, 95)
             for s in SAMPLINGS for r in (0, 4)]
    check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 32))
    try:
        for d, g in [(2, False), (8, False), (4, True)]:
            _check(wn, files, d, g)
    finally:
        check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 0))


def test_batches_ragged_and_independence(wn):
    from whenet_b200 import video
    rng = np.random.default_rng(5)
    files = []
    for i in range(65):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        files.append(encode(frame(KINDS[i % 4], h, w, seed=i), int(rng.integers(1, 101)), list(SAMPLINGS)[i % 4], rst=i % 3))
    for d, g in REDUCED:
        for n in (1, 8, 64, 65):
            _check(wn, files[:n], d, g)
        alone = [video.decode_jpeg(wn, [f], reduce=d, gray=g)[0].cpu().numpy() for f in files[:8]]
        together = video.decode_jpeg(wn, files[:8], reduce=d, gray=g)
        for a, t in zip(alone, together):
            assert np.array_equal(a, t.cpu().numpy())


def test_corrupt_files_raise_and_context_survives(wn):
    from test_gpu_jpeg_decode import _corrupt_cases
    from whenet_b200 import video
    good, cases = _corrupt_cases()
    for d, g in [(2, False), (8, False), (1, True), (4, True)]:
        for why, bad in cases.items():
            with pytest.raises(ValueError, match="file 1: .*" + why):
                video.decode_jpeg(wn, [good, bad], reduce=d, gray=g)
            _check(wn, [good], d, g)


def test_gray_decode_then_encode_equals_cv2(wn):
    import cv2
    import torch
    from whenet_b200 import video
    files = [encode(frame(kind, 1080, 1920, seed=k), 95, s) for k, kind in enumerate(KINDS) for s in ("420", "gray")]
    got = video.encode_jpeg(wn, torch.stack(video.decode_jpeg(wn, files, gray=True)), 95)
    for f, jpg in zip(files, got):
        ok, buf = cv2.imencode(".jpg", cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_GRAYSCALE), [cv2.IMWRITE_JPEG_QUALITY, 95])
        assert jpg == buf.tobytes()


def test_reader_reduce_and_4k_transcode(wn, tmp_path):
    """MJPGReader.read_frames(reduce=2) per frame, and a 4K transcode at 1/2 scale through detection, pose and drawing equal
    to the same loop fed by cv2.imdecode(f, IMREAD_REDUCED_COLOR_2): the same detections, angles and output bytes."""
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    yolo = whenet_b200.YOLO(None, max_frames=4)
    src = str(tmp_path / "src.avi")
    frames = [frame("gradient", 2160, 3840, seed=i) for i in range(6)]
    with video.MJPGWriter(src, 25, (3840, 2160)) as w:
        w.write([encode(f, 90) for f in frames])
    with video.MJPGReader(src) as r:
        files = r.read(6)
    with video.MJPGReader(src) as r:
        got = r.read_frames(wn, 6, reduce=2)
        assert tuple(got.shape) == (6, 1080, 1920, 3)
        for t, f in zip(got, files):
            assert np.array_equal(t.cpu().numpy(), imdecode(f, 2, False))
    with video.MJPGReader(src) as r:
        got = r.read_frames(wn, 6, reduce=4, gray=True)
        assert tuple(got.shape) == (6, 540, 960, 1)
        for t, f in zip(got, files):
            assert np.array_equal(t.cpu().numpy(), imdecode(f, 4, True))

    def loop(dst, gpu):
        with video.MJPGReader(src) as r, video.MJPGWriter(dst, r.fps, (1920, 1080)) as w:
            res_all = []
            while True:
                if gpu:
                    batch = r.read_frames(wn, 4, reduce=2)
                    if batch is None:
                        break
                else:
                    fs = r.read(4)
                    if not fs:
                        break
                    batch = torch.from_numpy(np.stack([imdecode(f, 2, False) for f in fs])).cuda()
                results = pipeline.detect_and_estimate_frames(yolo, wn, batch)
                overlay.draw_heads(wn, batch, results, display="full")
                w.write(video.encode_jpeg(wn, batch))
                res_all.append([tuple(np.asarray(x).tobytes() for x in r) for r in results])
        return res_all, open(dst, "rb").read()

    a = loop(str(tmp_path / "gpu.avi"), True)
    b = loop(str(tmp_path / "cpu.avi"), False)
    assert a[0] == b[0]
    assert a[1] == b[1]
