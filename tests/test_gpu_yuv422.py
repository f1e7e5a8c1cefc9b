"""Packed YUV 4:2:2 frames (YUYV, UYVY) and the YUV -> BGR conversion on the H100: every canvas, detection, crop and head pose
is the bits the BGR path gives on cv2.cvtColor(frame, COLOR_YUV2BGR_YUYV / _UYVY) ("ref" below), across frame and model
sizes, odd heights, detectors, chunking, graph replay, host and device frames, one-size batches and lists of several sizes;
video.to_bgr equals cv2.cvtColor for all four layouts; and a camera loop that stays on the device writes the AVI bytes of the
loop fed cvtColor's frames."""
import ctypes as C

import numpy as np
import pytest

import yolo_oracle as O
import yuv422_oracle as Y4
import yuv_oracle as Y
from test_gpu_pipeline import _crop_boxes, _same
from test_gpu_ragged import _biased_detector, _cuda, _same_dets, classes_file  # noqa: F401  (a fixture)
from test_gpu_yolo import _frame
from test_gpu_yuv import _box_448

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
CODES = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420, "yuyv": cv2.COLOR_YUV2BGR_YUYV, "uyvy": cv2.COLOR_YUV2BGR_UYVY}
LAYOUT = {"nv12": 1, "i420": 2, "yuyv": 3, "uyvy": 4}
FMTS = ["yuyv", "uyvy"]
CANVAS_SIZES = [(1080, 1920), (1081, 1920), (1920, 1080), (479, 640), (2160, 3840), (7, 34), (1, 2)]
DET_SIZES = [(1080, 1920), (719, 1280), (1920, 1080), (481, 640), (416, 416), (301, 1200)]


def _ref(yuv, fmt):
    return cv2.cvtColor(yuv, CODES[fmt])


def _random(rng, H, W, fmt):
    shape = (H, W, 2) if fmt in ("yuyv", "uyvy") else (H * 3 // 2, W)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def _video(H, W, seed, fmt):
    """A smooth scene as a camera (4:2:2) or a decoder (4:2:0) would hand it out."""
    bgr = _frame(H, W, seed=seed)[:, :, ::-1]
    return Y4.bgr_to_yuv422(bgr, fmt) if fmt in ("yuyv", "uyvy") else Y.bgr_to_yuv420(bgr, fmt)


# ----------------------------------------------------------------------------------------------- canvas
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [(416, 416), (448, 608)], ids=lambda s: "%dx%d" % s)
def test_canvas_equals_bgr_path_and_pillow(size, fmt):
    import whenet_b200
    h, w = size
    m = whenet_b200.YOLO(None, model_image_size=size, max_frames=8)
    rng = np.random.default_rng(h + LAYOUT[fmt])
    yuv = [_random(rng, H, W, fmt) for H, W in CANVAS_SIZES + [size]]
    refs = [_ref(f, fmt) for f in yuv]
    want = []
    for f, r in zip(yuv, refs):
        m.detect_frames(r[None])
        want.append(m.tap(-1).reshape(h, w, 3))
        assert np.array_equal(want[-1], O.letterbox(np.ascontiguousarray(r[:, :, ::-1]), (w, h))), r.shape
        for src in (f[None], _cuda([f[None]])[0]):
            m.detect_frames(src, pixel_format=fmt)
            assert np.array_equal(m.tap(-1).reshape(h, w, 3), want[-1]), r.shape
    for src in (yuv, _cuda(yuv)):
        m.detect_frames(src, pixel_format=fmt)
        got = m.tap(-1).reshape(len(yuv), h, w, 3)
        for i in range(len(yuv)):
            assert np.array_equal(got[i], want[i]), refs[i].shape
    m.close()


# ----------------------------------------------------------------------------------------------- detector
@pytest.mark.parametrize("kind", ["full", "tiny", "fp32", "two_classes"])
def test_detect_equals_detect_on_ref(kind, classes_file):  # noqa: F811
    m = _biased_detector(kind, classes_file)
    for fmt in FMTS:
        yuv = [_video(H, W, 10 * i + LAYOUT[fmt], fmt) for i, (H, W) in enumerate(DET_SIZES)]
        refs = [_ref(f, fmt) for f in yuv]
        ref = [m.detect_frames(r[None])[0] for r in refs]
        assert sum(len(r[0]) for r in ref) >= len(yuv)
        _same_dets(m.detect_frames(yuv[0][None], pixel_format=fmt), ref[:1])                     # one frame
        same = [_video(721, 1280, 100 + s, fmt) for s in range(6)]
        batch = np.stack(same)
        want = m.detect_frames(np.stack([_ref(f, fmt) for f in same]))
        _same_dets(m.detect_frames(batch[:4], pixel_format=fmt), want[:4])                        # n = max_frames
        _same_dets(m.detect_frames(batch, pixel_format=fmt), want)                                # chunks of 4 and 2
        _same_dets(m.detect_frames(batch, pixel_format=fmt), want)                                # graph replay
        _same_dets(m.detect_frames(_cuda([batch])[0], pixel_format=fmt), want)
        _same_dets(m.detect_frames(yuv[:4], pixel_format=fmt), ref[:4])                           # ragged, n = max_frames
        _same_dets(m.detect_frames(refs[:4]), ref[:4])                                             # the BGR list of the same sizes
        _same_dets(m.detect_frames(yuv[:4], pixel_format=fmt), ref[:4])                           # ragged replay after it
        _same_dets(m.detect_frames(tuple(yuv), pixel_format=fmt), ref)                            # ragged chunks of 4 and 2
        _same_dets(m.detect_frames(_cuda(yuv), pixel_format=fmt), ref)
    m.close()


def test_graphs_of_one_shape_are_kept_apart(classes_file):  # noqa: F811
    """YUYV, UYVY, NV12 and BGR batches of one (n, H, W), one size and ragged, called in turn: each replays its own graph."""
    m = _biased_detector("full", classes_file)
    batches = {f: np.stack([_video(720, 1280, 300 + 10 * k + s, f) for s in range(4)]) for k, f in enumerate(("yuyv", "uyvy", "nv12"))}
    want = {f: m.detect_frames(np.stack([_ref(x, f) for x in b])) for f, b in batches.items()}
    batches["bgr"] = np.stack([_frame(720, 1280, seed=330 + s)[:, :, ::-1] for s in range(4)])
    want["bgr"] = m.detect_frames(batches["bgr"])
    for f, g in (("yuyv", "uyvy"), ("uyvy", "nv12"), ("nv12", "bgr")):          # each layout's scenes give their own boxes
        assert not all(np.array_equal(a[0], b[0]) for a, b in zip(want[f], want[g])), (f, g)
    sizes = [(720, 1280), (721, 1280)]
    lists = {f: [_video(H, W, 400 + i, f) for i, (H, W) in enumerate(sizes)] for f in ("yuyv", "uyvy")}
    lists["nv12"] = [_video(720, 1280, 400, "nv12"), _video(722, 1280, 401, "nv12")]
    want_l = {f: [m.detect_frames(_ref(x, f)[None])[0] for x in fr] for f, fr in lists.items()}
    for _ in range(2):
        for f in ("yuyv", "uyvy", "nv12", "bgr", "uyvy", "yuyv"):
            _same_dets(m.detect_frames(batches[f], pixel_format=f), want[f])
            if f in lists:
                _same_dets(m.detect_frames(lists[f], pixel_format=f), want_l[f])
    m.close()


# ----------------------------------------------------------------------------------------------- crops
@pytest.fixture(scope="module", params=FMTS)
def crop_case(request):
    """Three frames of different sizes (two odd heights), 96 boxes: random ones, one on every frame edge, the exact 448 x 448
    case and invalid (empty or outside) slices."""
    fmt = request.param
    rng = np.random.default_rng(LAYOUT[fmt])
    sizes = [(1080, 1920), (481, 640), (1919, 1080)]
    yuv = [_random(rng, H, W, fmt) for H, W in sizes]
    boxes, frame_of = [], []
    for i in range(84):
        f = i % 3
        H, W = sizes[f]
        y0, x0 = rng.uniform(-100, H), rng.uniform(-100, W)
        boxes.append((y0, x0, y0 + rng.uniform(1, 500), x0 + rng.uniform(1, 500)))
        frame_of.append(f)
    boxes += [(0, 0, 481, 640), (-50, -50, 100, 100), (1000, 1800, 1100, 1950), (1800, 900, 1950, 1100), tuple(_box_448(1080, 1920)),
              (500.5, 10, 500.9, 200), (-300, -300, -10, -10), (np.nan, 10, 100, 200), (1500, 10, 1700, 200)]
    frame_of += [1, 0, 0, 2, 0, 0, 1, 2, 2]
    return fmt, yuv, np.array(boxes, np.float32), np.array(frame_of, np.int32)


def _crop_yuv422(wn, frames, boxes, frame_of, fmt):
    """whenet_crop_boxes_yuv422_u8 on an (n, H, W, 2) batch, or whenet_crop_boxes_ragged_yuv422_u8 on a list."""
    import torch
    from whenet_b200._lib import check
    from whenet_b200.whenet import _is_device, _ptr
    from whenet_b200.yolo import _frame_table
    m = len(boxes)
    out = torch.full((m, 224, 224, 3), 77, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rects = np.full((m, 4), -1, np.int32)
    valid = np.full(m, -1, np.int32)
    if isinstance(frames, list):
        ptrs, hw = _frame_table(frames, LAYOUT[fmt])
        check(wn._L.whenet_crop_boxes_ragged_yuv422_u8(wn._h, C.addressof(ptrs), _ptr(hw), len(frames), int(_is_device(frames[0])), _ptr(boxes),
                                                       _ptr(frame_of), m, LAYOUT[fmt], _ptr(out), _ptr(rects), _ptr(valid)))
    else:
        n, H, W = frames.shape[:3]
        check(wn._L.whenet_crop_boxes_yuv422_u8(wn._h, _ptr(frames), n, H, W, int(_is_device(frames)), _ptr(boxes), _ptr(frame_of), m,
                                                LAYOUT[fmt], _ptr(out), _ptr(rects), _ptr(valid)))
    wn.synchronize()
    return out.cpu().numpy(), rects, valid


def test_crops_equal_bgr_crops_and_cv2(crop_case):
    import whenet_b200
    fmt, yuv, boxes, frame_of = crop_case
    refs = [_ref(f, fmt) for f in yuv]
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=64)
    want = np.zeros((len(boxes), 224, 224, 3), np.uint8)
    want_rects = np.zeros((len(boxes), 4), np.int32)
    want_valid = np.zeros(len(boxes), np.int32)
    for f, r in enumerate(refs):
        sel = np.flatnonzero(frame_of == f)
        b, fo = np.ascontiguousarray(boxes[sel]), np.zeros(len(sel), np.int32)
        want[sel], want_rects[sel], want_valid[sel] = _crop_boxes(wn, r[None], b, fo)
        for src in (yuv[f][None], _cuda([yuv[f][None]])[0]):                 # the one-size entry, frame by frame
            got, rects, valid = _crop_yuv422(wn, src, b, fo, fmt)
            assert np.array_equal(valid, want_valid[sel]) and np.array_equal(rects, want_rects[sel])
            assert np.array_equal(got, want[sel]), f
    ok = want_rects[want_valid == 1]
    assert 0 < len(ok) < len(boxes) and want_valid[-1] == 1
    assert all((ok[:, j] % 2 == 1).any() for j in range(4))               # slices start and end on odd rows and mid chroma pair
    assert all((ok[:, j] % 2 == 0).any() for j in range(4))
    assert any((r[1] - r[0], r[3] - r[2]) == (448, 448) for r in ok)
    edges = [(ok[:, 0] == 0).any(), any(r[1] == yuv[frame_of[i]].shape[0] for i, r in enumerate(want_rects) if want_valid[i]),
             (ok[:, 2] == 0).any(), any(r[3] == yuv[frame_of[i]].shape[1] for i, r in enumerate(want_rects) if want_valid[i])]
    assert all(edges), edges                                                  # every frame edge is reached
    for src in (yuv, _cuda(yuv)):                                             # the ragged entry
        got, rects, valid = _crop_yuv422(wn, src, boxes, frame_of, fmt)
        assert np.array_equal(valid, want_valid) and np.array_equal(rects, want_rects)
        assert np.array_equal(got, want)
    for i, (y0, y1, x0, x1) in enumerate(want_rects):
        if want_valid[i]:
            cv = cv2.resize(cv2.cvtColor(refs[frame_of[i]][y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224))
            assert np.array_equal(want[i], cv), (i, boxes[i])
        else:
            assert not want[i].any()
    sel = np.flatnonzero(frame_of == 0)                                       # a one-size batch of two frames
    two = np.stack([yuv[0], np.ascontiguousarray(yuv[0][::-1])])
    fo2 = (np.arange(len(sel)) % 2).astype(np.int32)
    got, _r, _v = _crop_yuv422(wn, two, np.ascontiguousarray(boxes[sel]), fo2, fmt)
    exp, _r, _v = _crop_boxes(wn, np.stack([_ref(f, fmt) for f in two]), np.ascontiguousarray(boxes[sel]), fo2)
    assert len(sel) >= 25 and np.array_equal(got, exp)
    wn.close()


# ----------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def wn16():
    import whenet_b200
    m = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=16)
    yield m
    m.close()


@pytest.mark.parametrize("fmt", FMTS)
def test_pipeline_equals_pipeline_on_ref(wn16, classes_file, fmt):  # noqa: F811
    """About 20 heads per frame (more than WHENet's sub-batch of 16 per chunk of 4 frames), one-size batches and lists, host
    and device; the 301 x 1200 frames have heads whose slices are empty (NaN angles)."""
    from whenet_b200 import WhenetError, pipeline
    yolo = _biased_detector("full", classes_file)
    batch = np.stack([_video(1080, 1920, 200 + s, fmt) for s in range(6)])
    ref_batch = np.stack([_ref(f, fmt) for f in batch])
    want = pipeline.detect_and_estimate_frames(yolo, wn16, ref_batch)
    assert max(sum(len(r[0]) for r in want[c:c + 4]) for c in (0, 4)) > 16
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, batch, pixel_format=fmt), want)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, _cuda([batch])[0], pixel_format=fmt), want)
    sizes = DET_SIZES + [(300, 1200), (641, 480), (1081, 1920)]
    frames = [_video(H, W, 50 + i, fmt) for i, (H, W) in enumerate(sizes)]
    want = pipeline.detect_and_estimate_frames(yolo, wn16, [_ref(f, fmt) for f in frames])
    assert any(np.isnan(r[2]).any() for r in want)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, frames, pixel_format=fmt), want)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, _cuda(frames), pixel_format=fmt), want)
    raised = 0
    for f in frames:
        try:
            exp = pipeline.detect_and_estimate(yolo, wn16, _ref(f, fmt))
        except WhenetError as e:
            with pytest.raises(WhenetError) as got:
                pipeline.detect_and_estimate(yolo, wn16, f, pixel_format=fmt)
            assert str(got.value) == str(e) and got.value.code == e.code
            raised += 1
            continue
        _same([pipeline.detect_and_estimate(yolo, wn16, f, pixel_format=fmt)], [exp])
    assert raised
    yolo.close()


# ----------------------------------------------------------------------------------------------- to_bgr
def _to_bgr_sizes(fmt):
    s = [(1080, 1920), (2160, 3840), (2, 2), (16384, 2), (2, 16384)]
    return s + [(1081, 1920), (1, 2), (7, 34)] if fmt in ("yuyv", "uyvy") else s


@pytest.fixture(scope="module")
def wn_plain():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


@pytest.mark.parametrize("fmt", ["nv12", "i420", "yuyv", "uyvy"])
def test_to_bgr_equals_cvtcolor(wn_plain, fmt):
    import torch
    from whenet_b200 import video
    rng = np.random.default_rng(LAYOUT[fmt] + 40)
    for H, W in _to_bgr_sizes(fmt):                                    # one frame, host and device
        f = _random(rng, H, W, fmt)
        want = _ref(f, fmt)
        for src in (f[None], _cuda([f[None]])[0]):
            got = video.to_bgr(wn_plain, src, fmt)
            assert got.is_cuda and got.is_contiguous() and got.dtype == torch.uint8 and tuple(got.shape) == (1, H, W, 3)
            assert np.array_equal(got[0].cpu().numpy(), want), (H, W)
    small = (135, 240) if fmt in ("yuyv", "uyvy") else (136, 240)
    for n, (H, W) in ((1, small), (8, (1080, 1920)), (64, small), (65, small)):   # batches: one group, a full group, two groups
        frames = np.stack([_random(rng, H, W, fmt) for _ in range(n)])
        want = np.stack([_ref(f, fmt) for f in frames])
        for src in (frames, _cuda([frames])[0]):
            got = video.to_bgr(wn_plain, src, fmt)
            assert tuple(got.shape) == (n, H, W, 3) and np.array_equal(got.cpu().numpy(), want), (n, H, W)
        for i in (0, n - 1):                                            # each frame alone equals it inside its batch
            assert np.array_equal(video.to_bgr(wn_plain, frames[i:i + 1], fmt)[0].cpu().numpy(), want[i])
    sizes = _to_bgr_sizes(fmt)[:3] + [small] * 62 + [(480, 640)]       # a ragged list of 66 frames: two groups
    frames = [_random(rng, H, W, fmt) for H, W in sizes]
    want = [_ref(f, fmt) for f in frames]
    for src in (frames, tuple(_cuda(frames))):
        got = video.to_bgr(wn_plain, src, fmt)
        assert isinstance(got, list) and len(got) == len(frames)
        for i, (g, w) in enumerate(zip(got, want)):
            assert g.is_contiguous() and np.array_equal(g.cpu().numpy(), w), (i, sizes[i])
    # device frames whose base is not 4- or 2-byte aligned read their bytes one by one
    for off in (1, 2, 3):
        f = frames[-1]
        buf = torch.empty(f.size + off, dtype=torch.uint8, device="cuda")
        view = buf[off:].view(f.shape)
        view.copy_(torch.from_numpy(f))
        got = video.to_bgr(wn_plain, [view], fmt)
        assert np.array_equal(got[0].cpu().numpy(), want[-1]), off
    assert video.to_bgr(wn_plain, [], fmt) == []
    empty = video.to_bgr(wn_plain, np.zeros((0,) + _random(rng, 4, 4, fmt).shape, np.uint8), fmt)
    assert tuple(empty.shape) == (0, 4, 4, 3)


def test_to_bgr_orders_against_torch_stream(wn_plain):
    """Frames written on torch's current stream behind a held stream, converted, and read on that stream, without a
    synchronisation by the caller."""
    import torch
    from whenet_b200 import video
    rng = np.random.default_rng(7)
    f = rng.integers(0, 256, (4, 1081, 1920, 2), dtype=np.uint8)
    want = np.stack([_ref(x, "uyvy") for x in f])
    host = torch.from_numpy(f).pin_memory()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(2):
            dev = torch.empty(f.shape, dtype=torch.uint8, device="cuda")
            torch.cuda._sleep(50_000_000)                                # hold the stream, then write the frames on it
            dev.copy_(host, non_blocking=True)
            out = video.to_bgr(wn_plain, dev, "uyvy")
            total = out.to(torch.int64).sum()                          # read on the same stream
            assert np.array_equal(out.cpu().numpy(), want)
            assert int(total) == int(want.astype(np.int64).sum())


# ----------------------------------------------------------------------------------------------- end to end
def _loop(yolo, wn, frames, fmt, path):
    """detect_and_estimate_frames -> to_bgr -> draw_heads(display="full") -> encode_jpeg -> MJPGWriter, in chunks of 4; fmt None:
    the frames are BGR already."""
    import torch
    from whenet_b200 import overlay, pipeline, video
    H, W = frames[0].shape[:2] if fmt != "nv12" else (frames[0].shape[0] * 2 // 3, frames[0].shape[1])
    results = []
    with video.MJPGWriter(path, 25, (W, H)) as w:
        for lo in range(0, len(frames), 4):
            chunk = _cuda([np.stack(frames[lo:lo + 4])])[0]
            if fmt is None:
                res = pipeline.detect_and_estimate_frames(yolo, wn, chunk)
                bgr = chunk
            else:
                res = pipeline.detect_and_estimate_frames(yolo, wn, chunk, pixel_format=fmt)
                bgr = video.to_bgr(wn, chunk, fmt)
            overlay.draw_heads(wn, bgr, res, display="full")
            w.write(video.encode_jpeg(wn, bgr))
            results += res
            torch.cuda.synchronize()
    with open(path, "rb") as f:
        return results, f.read()


@pytest.mark.parametrize("fmt", ["nv12", "yuyv"])
def test_device_loop_equals_cvtcolor_loop(wn16, classes_file, fmt, tmp_path):  # noqa: F811
    yolo = _biased_detector("full", classes_file)
    frames = [_video(1080, 1920, 600 + s, fmt) for s in range(6)]
    got, avi = _loop(yolo, wn16, frames, fmt, str(tmp_path / "device.avi"))
    want, want_avi = _loop(yolo, wn16, [_ref(f, fmt) for f in frames], None, str(tmp_path / "host.avi"))
    assert sum(len(r[0]) for r in want) > 16
    _same(got, want)
    assert avi == want_avi
    yolo.close()
