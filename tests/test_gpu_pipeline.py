"""Multi-frame pipeline on the H100: whenet_crop_boxes_u8 bit for bit against cv2 on the crops of several frames, and
pipeline.detect_and_estimate_frames against pipeline.detect_and_estimate frame by frame - bitwise, because the detector and
WHENet are batch invariant - across chunkings, WHENet sub-batches, frames without detections, detectors and frame sizes, with
NaN angles for exactly the heads whose slice is empty."""
import numpy as np
import pytest

from test_gpu_yolo import _frame

pytestmark = pytest.mark.gpu


def _hook(boxes, H, W):
    from whenet_b200 import _lib
    boxes = np.ascontiguousarray(boxes, np.float32).reshape(-1, 4)
    rects = np.zeros((len(boxes), 4), np.int32)
    valid = np.zeros(len(boxes), np.int32)
    if len(boxes):
        assert _lib.load().whenet_debug_enlarge_boxes(boxes.ctypes.data, len(boxes), H, W, rects.ctypes.data, valid.ctypes.data) == 0
    return rects, valid.astype(bool)


# ----------------------------------------------------------------------------------------------- crops of many frames
def _crop_boxes(wn, frames, boxes, frame_of):
    import torch
    from whenet_b200._lib import check
    from whenet_b200.whenet import _is_device, _ptr
    n, H, W = frames.shape[:3]
    m = len(boxes)
    out = torch.full((m, 224, 224, 3), 77, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rects = np.full((m, 4), -1, np.int32)
    valid = np.full(m, -1, np.int32)
    check(wn._L.whenet_crop_boxes_u8(wn._h, _ptr(frames), n, H, W, int(_is_device(frames)), _ptr(boxes), _ptr(frame_of), m, 1,
                                     _ptr(out), _ptr(rects), _ptr(valid)))
    wn.synchronize()
    return out.cpu().numpy(), rects, valid


def test_crop_boxes_equal_cv2_on_three_frames():
    import torch
    import whenet_b200
    from whenet_b200._lib import check
    from whenet_b200.whenet import _ptr
    cv2 = pytest.importorskip("cv2")
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=64)
    rng = np.random.default_rng(11)
    H, W = 1080, 1920
    frames = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    boxes = []
    for _ in range(54):                         # inside or straddling a border
        y0, x0 = rng.uniform(-100, H), rng.uniform(-100, W)
        boxes.append((y0, x0, y0 + rng.uniform(1, 500), x0 + rng.uniform(1, 500)))
    boxes += [(0, 0, H, W), (0, 0, 448 / 1.2, 448 / 1.4),      # the whole frame; a slice near 448 x 448 (2x box path)
              (500.5, 10, 500.9, 200), (-300, -300, -10, -10), (np.nan, 10, 100, 200), (10, 10, -np.inf, 200)]
    boxes = np.array(boxes, np.float32)
    frame_of = rng.integers(0, 3, len(boxes)).astype(np.int32)
    ref_rects, ref_valid = _hook(boxes, H, W)
    assert 0 < ref_valid.sum() < len(boxes)
    for src in (frames, torch.from_numpy(frames).cuda()):
        got, rects, valid = _crop_boxes(wn, src, boxes, frame_of)
        assert np.array_equal(valid.astype(bool), ref_valid) and np.array_equal(rects, ref_rects)
        for i, (y0, y1, x0, x1) in enumerate(rects):
            if valid[i]:
                ref = cv2.resize(cv2.cvtColor(frames[frame_of[i]][y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224))
                assert np.array_equal(got[i], ref), (i, boxes[i], rects[i])
            else:
                assert not got[i].any(), (i, boxes[i])
    # one frame's boxes: the same bytes as whenet_crop_resize_u8 with the same slices
    one = np.flatnonzero(ref_valid & (frame_of == 1))
    got, _r, _v = _crop_boxes(wn, frames[1:2], boxes[one], np.zeros(len(one), np.int32))
    out = torch.empty((len(one), 224, 224, 3), dtype=torch.uint8, device="cuda")
    check(wn._L.whenet_crop_resize_u8(wn._h, _ptr(frames[1]), H, W, 0, _ptr(np.ascontiguousarray(ref_rects[one])), len(one), 1, _ptr(out)))
    wn.synchronize()
    assert np.array_equal(got, out.cpu().numpy())
    wn.close()


# ----------------------------------------------------------------------------------------------- detect_and_estimate_frames
@pytest.fixture(scope="module")
def wn16():
    import whenet_b200
    m = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=16)
    yield m
    m.close()


@pytest.fixture(scope="module")
def classes_file(tmp_path_factory):
    p = tmp_path_factory.mktemp("classes") / "classes_2.txt"
    p.write_text("head\nface")
    return str(p)


def _detector(kind, classes_file):
    import whenet_b200
    import yolo_tiny_cases as TC
    kw = {"tiny": {"anchors_path": TC.ANCHORS}, "two_classes": {"classes_path": classes_file}}.get(kind, {})
    return whenet_b200.YOLO(None, max_frames=4, **kw)


def _same(got, ref):
    assert len(got) == len(ref)
    for f, (g, r) in enumerate(zip(got, ref)):
        for x, y, what in zip(g, r, ("boxes", "scores", "angles")):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y, equal_nan=True), (f, what)


def _frames_with_empty_ones(yolo):
    """Square 832 x 832 frames (every box centre lies inside: no slice is empty) and flat ones; the detector's score is set
    between the two lowest per-frame top scores, so the frame(s) with the lowest top score have no detection while the
    textured ones keep theirs.  -> (frames in mixed order, indices of the empty frames)."""
    frames = [_frame(832, 832, seed=s) for s in range(7)] + [np.full((832, 832, 3), v, np.uint8) for v in (0, 128, 255)]
    frames = [frames[i] for i in (0, 7, 1, 2, 3, 8, 4, 5, 9, 6)]
    yolo.score = 0.0
    top = [float(d[1].max()) for d in yolo.detect_frames(np.stack(frames))]
    lo = sorted(set(top))
    yolo.score = (lo[0] + lo[1]) / 2
    empty = [i for i, t in enumerate(top) if t < yolo.score]
    return frames, empty


def _check_against_per_frame(yolo, wn, frames, empty, sources=("host", "device"), ns=(1, 3, 9)):
    import torch
    from whenet_b200 import pipeline
    ref = [pipeline.detect_and_estimate(yolo, wn, f) for f in frames]
    assert all(len(ref[i][0]) == 0 for i in empty) and any(len(r[0]) for r in ref)
    stack = np.stack(frames)
    for n in ns:
        for src in sources:
            x = stack[:n] if src == "host" else torch.from_numpy(stack[:n]).cuda()
            _same(pipeline.detect_and_estimate_frames(yolo, wn, x), ref[:n])
    return ref


def test_frames_equal_per_frame_full_detector(wn16, classes_file):
    """n = 1, 3 and 9 with max_frames = 4 (9 frames: chunks of 4, 4 and 1), host and device frames, WHENet sub-batches of 16
    with more than 16 crops per chunk, frames without detections mixed in, and a batch without any detection."""
    import torch
    from whenet_b200 import pipeline
    yolo = _detector("full", classes_file)
    frames, empty = _frames_with_empty_ones(yolo)
    assert empty and empty[0] < 9
    ref = _check_against_per_frame(yolo, wn16, frames[:9], [i for i in empty if i < 9])
    assert max(sum(len(r[0]) for r in ref[c:c + 4]) for c in (0, 4)) > 16
    none = np.stack([frames[empty[0]]] * 3)
    for x in (none, torch.from_numpy(none).cuda()):
        got = pipeline.detect_and_estimate_frames(yolo, wn16, x)
        _same(got, [ref[empty[0]]] * 3)
        assert all(len(g[0]) == 0 and g[2].shape == (0, 3) for g in got)
    assert pipeline.detect_and_estimate_frames(yolo, wn16, none[:0]) == []
    yolo.close()


@pytest.mark.parametrize("kind,source", [("tiny", "device"), ("two_classes", "host")])
def test_frames_equal_per_frame_other_detectors(wn16, classes_file, kind, source):
    yolo = _detector(kind, classes_file)
    assert yolo.tiny == (kind == "tiny") and yolo.num_classes == (2 if kind == "two_classes" else 1)
    frames, empty = _frames_with_empty_ones(yolo)
    _check_against_per_frame(yolo, wn16, frames[:6], [i for i in empty if i < 6], sources=(source,), ns=(6,))
    yolo.close()


def _per_frame_with_nan(yolo, wn, frame):
    """What detect_and_estimate_frames promises for one frame: detect_and_estimate where it succeeds; where it raises
    (an empty slice), the detector's boxes and scores with NaN angles for exactly the heads whose enlarge_box slice is
    empty and get_angle_from_frame's angles on the other boxes."""
    from whenet_b200 import WhenetError, crops, pipeline
    try:
        return pipeline.detect_and_estimate(yolo, wn, frame)
    except WhenetError as e:
        assert e.code == -1 and "box" in str(e) and "cv2.resize would raise" in str(e)
    boxes, scores, _c = yolo.detect_frames(frame[None])[0]
    H, W = frame.shape[:2]
    ok = np.array([r[0] < r[1] and r[2] < r[3] and 0 <= r[0] and r[1] <= H and 0 <= r[2] and r[3] <= W
                   for r in (crops.enlarge_box(b, H, W) for b in boxes)], bool)
    assert not ok.all()
    angles = np.full((len(boxes), 3), np.nan, np.float32)
    if ok.any():
        angles[ok] = np.stack(wn.get_angle_from_frame(frame, boxes[ok]), 1)
    return boxes, scores, angles


def test_empty_slices_get_nan(wn16, classes_file):
    """Wide frames letterboxed to 416 x 416: boxes centred in the padding enlarge to empty slices."""
    import torch
    from whenet_b200 import pipeline
    yolo = _detector("full", classes_file)
    yolo.score = 0.26
    frames = np.stack([_frame(300, 1200, seed=s) for s in range(3)])
    ref = [_per_frame_with_nan(yolo, wn16, f) for f in frames]
    n_nan = sum(int(np.isnan(r[2][:, 0]).sum()) for r in ref)
    assert n_nan >= 1 and all(np.isnan(r[2]).all(1).sum() == np.isnan(r[2]).any(1).sum() for r in ref)
    for x in (frames, torch.from_numpy(frames).cuda()):
        _same(pipeline.detect_and_estimate_frames(yolo, wn16, x), ref)
    yolo.close()


def test_changing_frame_size(wn16, classes_file):
    from whenet_b200 import pipeline
    yolo = _detector("full", classes_file)
    yolo.score = 0.26
    for h, w, n, seed in ((832, 832, 3, 20), (300, 1200, 5, 30), (640, 640, 2, 40)):
        frames = np.stack([_frame(h, w, seed=seed + s) for s in range(n)])
        ref = [_per_frame_with_nan(yolo, wn16, f) for f in frames] if h != w else \
            [pipeline.detect_and_estimate(yolo, wn16, f) for f in frames]
        _same(pipeline.detect_and_estimate_frames(yolo, wn16, frames), ref)
    yolo.close()
