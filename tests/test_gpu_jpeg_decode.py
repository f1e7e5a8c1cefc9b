"""GPU JPEG decoding (``video.decode_jpeg``, ``MJPGReader.read_frames``, DESIGN.md section 8.10): every frame equals
cv2.imdecode at every size, quality, sampling and restart setting, at any batch size and for ragged lists, on a context whose
buffers grow and shrink; corrupt files raise naming their frame and leave the context usable; and the MJPG transcode loop
fed by the GPU decoder matches the same loop fed by cv2."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_jpeg_cpu import KINDS, SIZES, frame  # noqa: E402
from test_jpeg_decode_cpu import GOLDEN, SAMPLES, SAMPLINGS, encode, imdecode, strip_dht, with_exif  # noqa: E402

pytestmark = pytest.mark.gpu
QS = [1, 50, 95, 100]


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _check(wn, files):
    from whenet_b200 import video
    got = video.decode_jpeg(wn, files)
    assert len(got) == len(files)
    for i, (g, f) in enumerate(zip(got, files)):
        ref = imdecode(f)
        assert g.is_contiguous() and g.device.index == wn.device
        assert tuple(g.shape) == ref.shape and np.array_equal(g.cpu().numpy(), ref), (i, ref.shape)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_equals_cv2_small(wn, sampling):
    files = [encode(frame(kind, h, w, seed=q + k), q, sampling, rst=r) for h, w in SIZES for q in QS
             for k, kind in enumerate(KINDS) for r in (0, 3)]
    for lo in range(0, len(files), 64):
        _check(wn, files[lo:lo + 64])


@pytest.mark.parametrize("h,w", [(720, 1280), (1080, 1920), (1081, 1921), (2160, 3840)])
@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_equals_cv2_large(wn, h, w, sampling):
    files = [encode(frame(kind, h, w, seed=q), q, sampling, rst=r) for q in QS for kind, r in [("noise", 0), ("gradient", 0), ("noise", 7)]]
    _check(wn, files)


@pytest.mark.parametrize("h,w", [(4096, 4096), (16384, 24), (24, 16384)])
def test_equals_cv2_extreme_sizes(wn, h, w):
    files = [encode(frame("noise", h, w, seed=q), q, s, rst=r) for q in QS for s in SAMPLINGS for r in (0, 5)]
    for lo in range(0, len(files), 8):
        _check(wn, files[lo:lo + 8])


def test_fill_bytes_and_trailing_segments(wn):
    from test_jpeg_decode_cpu import fill_and_trailing_segments
    _check(wn, [fill_and_trailing_segments(encode(frame("noise", 64, 80), 75, s, rst=2)) for s in SAMPLINGS])


def test_fixtures_exif_and_no_dht(wn):
    base = encode(frame("gradient", 40, 64), 90)
    files = [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    files += [with_exif(base, o, be) for o in range(1, 9) for be in (False, True)]
    files += [strip_dht(encode(frame("noise", 37, 53), 75, s)) for s in SAMPLINGS]
    _check(wn, files)


def test_batches_ragged_and_independence(wn):
    from whenet_b200 import video
    rng = np.random.default_rng(5)
    files = []
    for i in range(65):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        files.append(encode(frame(KINDS[i % 4], h, w, seed=i), int(rng.integers(1, 101)), list(SAMPLINGS)[i % 4], rst=i % 3))
    for n in (1, 8, 64, 65):
        _check(wn, files[:n])
    alone = [video.decode_jpeg(wn, [f])[0].cpu().numpy() for f in files[:8]]
    together = video.decode_jpeg(wn, files[:8])
    for a, t in zip(alone, together):
        assert np.array_equal(a, t.cpu().numpy())


def test_grow_then_shrink_fresh_context():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=1)
    try:
        _check(m, [encode(frame("noise", 8, 8), 75)])
        _check(m, [encode(frame("noise", 1080, 1920), 95, rst=5)] * 4)
        _check(m, [encode(frame("gradient", 17, 33), 50, "gray")])
    finally:
        m.close()


def test_encode_then_decode(wn):
    import torch
    from whenet_b200 import video
    frames = [frame(kind, 1080, 1920, seed=k) for k, kind in enumerate(KINDS)]
    dev = torch.from_numpy(np.stack(frames)).cuda()
    got = video.decode_jpeg(wn, video.encode_jpeg(wn, dev, 95))
    for g, f in zip(got, frames):
        ok, buf = __import__("cv2").imencode(".jpg", f, [__import__("cv2").IMWRITE_JPEG_QUALITY, 95])
        assert np.array_equal(g.cpu().numpy(), imdecode(buf.tobytes()))


def test_short_subsequences(wn):
    from whenet_b200._lib import check
    files = [encode(frame(kind, 1080, 1920, seed=2), q, s, rst=r) for kind in ("noise", "gradient") for q in (10, 95)
             for s in SAMPLINGS for r in (0, 4)]
    check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 32))
    try:
        _check(wn, files)
    finally:
        check(wn._L.whenet_debug_jpeg_piece_bits(wn._h, 0))


def _corrupt_cases():
    good = encode(frame("noise", 64, 80), 75, rst=2)
    sos = good.index(b"\xff\xda")
    ecs = sos + 2 + int.from_bytes(good[sos + 2:sos + 4], "big")
    rst = good.index(b"\xff\xd0", ecs)
    cases = {"truncated": good[:len(good) - 40]}
    b = bytearray(good); b[rst + 1] = 0xD3; cases["restart"] = bytes(b)
    b = bytearray(good); b[ecs:ecs + 4] = b"\xff\x00\xff\x00"; cases["Huffman"] = bytes(b)  # 16 one bits: no luma DC code
    b = bytearray(good); b[rst + 1] = 0xC4; cases["marker"] = bytes(b)
    # a block whose AC run passes 63: DC category 0 ('00'), then AC 0xF1 eight times ... built from the standard luma table
    g = encode(np.full((8, 8, 3), 128, np.uint8), 75, "gray")
    s2 = g.index(b"\xff\xda")
    e2 = s2 + 2 + int.from_bytes(g[s2 + 2:s2 + 4], "big")
    bits = "00" + "11111111001" * 4 + "1111111110011101" + "1"     # DC 0, ZRL x4 (64 zeros), run 15 size 1 -> index 80
    bits += "1" * (-len(bits) % 8)
    data = int(bits, 2).to_bytes(len(bits) // 8, "big").replace(b"\xff", b"\xff\x00")
    cases["run past"] = g[:e2] + data + b"\xff\xd9"
    return good, cases


def test_corrupt_files_raise_and_context_survives(wn):
    from whenet_b200 import video
    good, cases = _corrupt_cases()
    for why, bad in cases.items():
        with pytest.raises(ValueError, match="file 1: .*" + why):
            video.decode_jpeg(wn, [good, bad])
        _check(wn, [good])


def test_transcode_loop_matches_cv2_fed_loop(wn, tmp_path):
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    yolo = whenet_b200.YOLO(None, max_frames=4)
    src = str(tmp_path / "src.avi")
    frames = [frame("gradient", 360, 640, seed=i) for i in range(10)]
    with video.MJPGWriter(src, 25, (640, 360)) as w:
        w.write([encode(f, 90) for f in frames])

    def loop(dst, gpu):
        with video.MJPGReader(src) as r, video.MJPGWriter(dst, r.fps, r.frame_size) as w:
            res_all = []
            while True:
                if gpu:
                    batch = r.read_frames(wn, 4)
                    if batch is None:
                        break
                else:
                    files = r.read(4)
                    if not files:
                        break
                    batch = torch.from_numpy(np.stack([imdecode(f) for f in files])).cuda()
                results = pipeline.detect_and_estimate_frames(yolo, wn, batch)
                overlay.draw_heads(wn, batch, results, display="full")
                w.write(video.encode_jpeg(wn, batch))
                res_all.append([tuple(np.asarray(x).tobytes() for x in r) for r in results])
        return res_all, open(dst, "rb").read()

    a = loop(str(tmp_path / "gpu.avi"), True)
    b = loop(str(tmp_path / "cpu.avi"), False)
    assert a[0] == b[0]
    assert a[1] == b[1]
