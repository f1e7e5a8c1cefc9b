"""NV12 and I420 frames on the H100: every canvas, detection, crop and head pose is the bits the BGR path gives on
cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420) ("ref" below), across frame and model sizes, detectors, chunking, graph
replay, host and device frames, one-size batches and lists of several sizes."""
import ctypes as C

import numpy as np
import pytest

import yolo_oracle as O
import yuv_oracle as Y
from test_gpu_pipeline import _crop_boxes, _same
from test_gpu_ragged import _biased_detector, _cuda, _same_dets, classes_file  # noqa: F401  (a fixture)
from test_gpu_yolo import _frame

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
CODES = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420}
LAYOUT = {"nv12": 1, "i420": 2}
CANVAS_SIZES = [(1080, 1920), (1920, 1080), (720, 1280), (480, 640), (2160, 3840), (2, 2)]
DET_SIZES = [(1080, 1920), (720, 1280), (1920, 1080), (480, 640), (416, 416), (300, 1200)]


def _ref(yuv, fmt):
    return cv2.cvtColor(yuv, CODES[fmt])


def _video(H, W, seed, fmt):
    """A smooth scene as a decoder would hand it out (4:2:0 in cv2's layout)."""
    return Y.bgr_to_yuv420(_frame(H, W, seed=seed)[:, :, ::-1], fmt)


# ----------------------------------------------------------------------------------------------- canvas
@pytest.mark.parametrize("fmt", ["nv12", "i420"])
@pytest.mark.parametrize("size", [(416, 416), (448, 608)], ids=lambda s: "%dx%d" % s)
def test_canvas_equals_bgr_path_and_pillow(size, fmt):
    import whenet_b200
    h, w = size
    m = whenet_b200.YOLO(None, model_image_size=size, max_frames=8)
    rng = np.random.default_rng(h + LAYOUT[fmt])
    yuv = [rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8) for H, W in CANVAS_SIZES + [size]]
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
    for fmt in ("nv12", "i420"):
        yuv = [_video(H, W, 10 * i + LAYOUT[fmt], fmt) for i, (H, W) in enumerate(DET_SIZES)]
        refs = [_ref(f, fmt) for f in yuv]
        ref = [m.detect_frames(r[None])[0] for r in refs]
        assert sum(len(r[0]) for r in ref) >= len(yuv)
        _same_dets(m.detect_frames(yuv[0][None], pixel_format=fmt), ref[:1])                     # one frame
        same = [_video(720, 1280, 100 + s, fmt) for s in range(6)]
        batch = np.stack(same)
        want = m.detect_frames(np.stack([_ref(f, fmt) for f in same]))
        _same_dets(m.detect_frames(batch[:4], pixel_format=fmt), want[:4])                        # n = max_frames
        _same_dets(m.detect_frames(batch, pixel_format=fmt), want)                                # chunks of 4 and 2
        _same_dets(m.detect_frames(batch, pixel_format=fmt), want)                                # graph replay
        for _ in range(2):                                                                         # BGR and YUV graphs of one shape
            _same_dets(m.detect_frames(np.stack([_ref(f, fmt) for f in same[:4]])), want[:4])
            _same_dets(m.detect_frames(batch[:4], pixel_format=fmt), want[:4])
        _same_dets(m.detect_frames(_cuda([batch])[0], pixel_format=fmt), want)
        _same_dets(m.detect_frames(yuv[:4], pixel_format=fmt), ref[:4])                           # ragged, n = max_frames
        _same_dets(m.detect_frames(refs[:4]), ref[:4])                                             # the BGR list of the same sizes
        _same_dets(m.detect_frames(yuv[:4], pixel_format=fmt), ref[:4])                           # ragged replay after it
        _same_dets(m.detect_frames(tuple(yuv), pixel_format=fmt), ref)                            # ragged chunks of 4 and 2
        _same_dets(m.detect_frames(_cuda(yuv), pixel_format=fmt), ref)
    m.close()


# ----------------------------------------------------------------------------------------------- crops
def _box_448(H, W):
    """A float32 box whose enlarged slice is exactly 448 x 448 (the 2x2 box path of the resize)."""
    from whenet_b200 import crops
    hs = [h for h in np.arange(360.0, 380.0, 0.01) if np.diff(crops.enlarge_box(np.array([101, 101, 101 + h, 301], np.float32), H, W)[:2])[0] == 448]
    ws = [w for w in np.arange(300.0, 320.0, 0.01) if np.diff(crops.enlarge_box(np.array([101, 101, 301, 101 + w], np.float32), H, W)[2:])[0] == 448]
    return np.array([101, 101, 101 + hs[0], 101 + ws[0]], np.float32)


@pytest.fixture(scope="module", params=["nv12", "i420"])
def crop_case(request):
    """Three frames of different sizes, 96 boxes: random ones, one on every frame edge, the exact 448 x 448 case and invalid
    (empty or outside) slices."""
    fmt = request.param
    rng = np.random.default_rng(LAYOUT[fmt])
    sizes = [(1080, 1920), (480, 640), (1920, 1080)]
    yuv = [rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8) for H, W in sizes]
    boxes, frame_of = [], []
    for i in range(84):
        f = i % 3
        H, W = sizes[f]
        y0, x0 = rng.uniform(-100, H), rng.uniform(-100, W)
        boxes.append((y0, x0, y0 + rng.uniform(1, 500), x0 + rng.uniform(1, 500)))
        frame_of.append(f)
    boxes += [(0, 0, 480, 640), (-50, -50, 100, 100), (1000, 1800, 1100, 1950), (1800, 900, 1950, 1100), tuple(_box_448(1080, 1920)),
              (500.5, 10, 500.9, 200), (-300, -300, -10, -10), (np.nan, 10, 100, 200), (1500, 10, 1700, 200)]
    frame_of += [1, 0, 0, 2, 0, 0, 1, 2, 2]
    return fmt, yuv, np.array(boxes, np.float32), np.array(frame_of, np.int32)


def _crop_yuv(wn, frames, boxes, frame_of, fmt):
    """whenet_crop_boxes_yuv_u8 on an (n, H * 3/2, W) batch, or whenet_crop_boxes_ragged_yuv_u8 on a list."""
    import torch
    from whenet_b200._lib import check
    from whenet_b200.whenet import _is_device, _ptr
    from whenet_b200.yolo import _frame_table
    m = len(boxes)
    out = torch.full((m, 224, 224, 3), 77, dtype=torch.uint8, device="cuda")
    rects = np.full((m, 4), -1, np.int32)
    valid = np.full(m, -1, np.int32)
    if isinstance(frames, list):
        ptrs, hw = _frame_table(frames, LAYOUT[fmt])
        check(wn._L.whenet_crop_boxes_ragged_yuv_u8(wn._h, C.addressof(ptrs), _ptr(hw), len(frames), int(_is_device(frames[0])), _ptr(boxes),
                                                    _ptr(frame_of), m, LAYOUT[fmt], _ptr(out), _ptr(rects), _ptr(valid)))
    else:
        n, rows, W = frames.shape
        check(wn._L.whenet_crop_boxes_yuv_u8(wn._h, _ptr(frames), n, rows // 3 * 2, W, int(_is_device(frames)), _ptr(boxes), _ptr(frame_of), m,
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
            got, rects, valid = _crop_yuv(wn, src, b, fo, fmt)
            assert np.array_equal(valid, want_valid[sel]) and np.array_equal(rects, want_rects[sel])
            assert np.array_equal(got, want[sel]), f
    ok = want_rects[want_valid == 1]
    assert 0 < len(ok) < len(boxes) and want_valid[-1] == 1
    assert all((ok[:, j] % 2 == 1).any() for j in range(4))               # slices start and end mid chroma pair
    assert any((r[1] - r[0], r[3] - r[2]) == (448, 448) for r in ok)
    for src in (yuv, _cuda(yuv)):                                             # the ragged entry
        got, rects, valid = _crop_yuv(wn, src, boxes, frame_of, fmt)
        assert np.array_equal(valid, want_valid) and np.array_equal(rects, want_rects)
        assert np.array_equal(got, want)
    for i, (y0, y1, x0, x1) in enumerate(want_rects):
        if want_valid[i]:
            cv = cv2.resize(cv2.cvtColor(refs[frame_of[i]][y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224))
            assert np.array_equal(want[i], cv), (i, boxes[i])
        else:
            assert not want[i].any()
    sel = np.flatnonzero(frame_of != 1)                                       # a one-size batch of two frames, m >= 60
    two = np.stack([yuv[0], np.ascontiguousarray(yuv[0][:, ::-1])])
    fo2 = (frame_of[sel] == 2).astype(np.int32)
    got, _r, _v = _crop_yuv(wn, two, np.ascontiguousarray(boxes[sel]), fo2, fmt)
    exp, _r, _v = _crop_boxes(wn, np.stack([_ref(f, fmt) for f in two]), np.ascontiguousarray(boxes[sel]), fo2)
    assert len(sel) >= 60 and np.array_equal(got, exp)
    wn.close()


# ----------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def wn16():
    import whenet_b200
    m = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=16)
    yield m
    m.close()


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
def test_pipeline_equals_pipeline_on_ref(wn16, classes_file, fmt):  # noqa: F811
    """About 20 heads per frame (more than WHENet's sub-batch of 16 per chunk of 4 frames), one-size batches and lists, host
    and device; the 300 x 1200 frames have heads whose slices are empty (NaN angles)."""
    from whenet_b200 import WhenetError, pipeline
    yolo = _biased_detector("full", classes_file)
    batch = np.stack([_video(1080, 1920, 200 + s, fmt) for s in range(6)])
    ref_batch = np.stack([_ref(f, fmt) for f in batch])
    want = pipeline.detect_and_estimate_frames(yolo, wn16, ref_batch)
    assert max(sum(len(r[0]) for r in want[c:c + 4]) for c in (0, 4)) > 16
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, batch, pixel_format=fmt), want)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, _cuda([batch])[0], pixel_format=fmt), want)
    sizes = DET_SIZES + [(300, 1200), (640, 480), (1080, 1920)]
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
