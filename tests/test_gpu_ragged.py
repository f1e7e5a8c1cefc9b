"""Frames of several sizes in one call on the H100: each frame's canvas, detections, crops and head poses are the bits the
one-size path gives that frame alone (the canvas also Pillow's, the crops also cv2's), across detectors, chunking, graph
replay, host and device frames, WHENet sub-batches and frames without detections."""
import ctypes as C

import numpy as np
import pytest

import yolo_oracle as O
from test_gpu_pipeline import _per_frame_with_nan, _same
from test_gpu_yolo import _frame

pytestmark = pytest.mark.gpu

CANVAS_SIZES = [(1080, 1920), (1920, 1080), (720, 1280), (480, 640), (2160, 3840), (417, 417), (1, 1)]
DET_SIZES = [(1080, 1920), (720, 1280), (1920, 1080), (480, 640), (417, 417), (300, 1200)]


def _cuda(frames):
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames]
    torch.cuda.synchronize()
    return d


def _same_dets(got, ref):
    assert len(got) == len(ref)
    for f, (g, r) in enumerate(zip(got, ref)):
        for x, y, what in zip(g, r, ("boxes", "scores", "classes")):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), (f, what)


# ----------------------------------------------------------------------------------------------- canvas
@pytest.mark.parametrize("size", [(416, 416), (448, 608)], ids=lambda s: "%dx%d" % s)
def test_ragged_canvas_equals_pillow_and_the_one_size_path(size):
    import whenet_b200
    h, w = size
    m = whenet_b200.YOLO(None, model_image_size=size, max_frames=8)
    rng = np.random.default_rng(h)
    rgb = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in CANVAS_SIZES + [size]]
    bgr = [np.ascontiguousarray(f[:, :, ::-1]) for f in rgb]
    alone = []
    for f in bgr:
        m.detect_frames(f[None])
        alone.append(m.tap(-1).reshape(h, w, 3))
    for src in (bgr, _cuda(bgr)):
        m.detect_frames(src)
        got = m.tap(-1).reshape(len(rgb), h, w, 3)
        for i, f in enumerate(rgb):
            assert np.array_equal(got[i], alone[i]), (i, f.shape)
            assert np.array_equal(got[i], O.letterbox(f, (w, h))), (i, f.shape)
    m.close()


# ----------------------------------------------------------------------------------------------- detector
@pytest.fixture(scope="module")
def classes_file(tmp_path_factory):
    p = tmp_path_factory.mktemp("classes") / "classes_2.txt"
    p.write_text("head\nface")
    return str(p)


def _biased_detector(kind, classes_file, max_frames=4):
    """A detector whose head objectness biases give about 20 boxes on a 1080p frame (tools/detect_bench.py); the two-class
    model keeps its random weights and takes every box above score 0.2 instead."""
    import whenet_b200
    import yolo_tiny_cases as TC
    from tools.detect_bench import frame1080, set_objectness_for_boxes
    kw = {"tiny": {"anchors_path": TC.ANCHORS}, "fp32": {"precision": "fp32"}, "two_classes": {"classes_path": classes_file}}.get(kind, {})
    m = whenet_b200.YOLO(None, max_frames=max_frames, **kw)
    if kind == "two_classes":
        m.score = 0.2
    else:
        set_objectness_for_boxes(m, frame1080(), m.tiny)
    return m


@pytest.mark.parametrize("kind", ["full", "tiny", "fp32", "two_classes"])
def test_ragged_detect_equals_detect_frame_by_frame(kind, classes_file):
    m = _biased_detector(kind, classes_file)
    frames = [np.ascontiguousarray(_frame(H, W, seed=i)[:, :, ::-1]) for i, (H, W) in enumerate(DET_SIZES)]
    ref = [m.detect_frames(f[None])[0] for f in frames]
    assert sum(len(r[0]) for r in ref) >= len(frames)
    _same_dets(m._detect_ragged(frames[:1], False), ref[:1])               # n = 1 through the ragged entry
    _same_dets(m.detect_frames(frames[:4]), ref[:4])                        # n = max_frames
    _same_dets(m.detect_frames(frames[:4]), ref[:4])                        # the same list again: graph replay
    _same_dets(m.detect_frames(frames[3::-1]), ref[3::-1])                  # another order: another graph
    _same_dets(m.detect_frames(tuple(frames)), ref)                         # 6 > max_frames: chunks of 4 and 2
    _same_dets(m.detect_frames(_cuda(frames)), ref)
    same = [frames[1], frames[1], frames[1]]
    _same_dets(m.detect_frames(same), m.detect_frames(np.stack(same)))     # one size: the stacked batch
    _same_dets(m.detect_frames(same), [ref[1]] * 3)
    m.close()


def test_ragged_graph_cache_eviction_and_buffer_growth():
    """More than 16 size lists empty the ragged cache without touching the one-size graphs; a larger list grows the frame
    buffer and frees both caches; every later call still gives the same bits."""
    import whenet_b200
    m = whenet_b200.YOLO(None, max_frames=2, score=0.2)
    small = [np.ascontiguousarray(_frame(120 + 8 * s, 160, seed=s)[:, :, ::-1]) for s in range(2)]
    first_ragged = m.detect_frames(small)
    first_uniform = m.detect_frames(np.stack([small[0]] * 2))
    for k in range(17):
        m.detect_frames([small[0], np.ascontiguousarray(_frame(40 + k, 64, seed=k))])
    _same_dets(m.detect_frames(small), first_ragged)
    _same_dets(m.detect_frames(np.stack([small[0]] * 2)), first_uniform)
    m.detect_frames([np.ascontiguousarray(_frame(1080, 1920, seed=3)), np.ascontiguousarray(_frame(720, 1280, seed=4))])
    _same_dets(m.detect_frames(small), first_ragged)
    _same_dets(m.detect_frames(np.stack([small[0]] * 2)), first_uniform)
    from whenet_b200 import WhenetError
    with pytest.raises(WhenetError, match="max_frames=2"):
        m._detect_ragged(small + small[:1], False)
    m.close()


# ----------------------------------------------------------------------------------------------- crops
def _crop_ragged(wn, frames, boxes, frame_of):
    import torch
    from whenet_b200._lib import check
    from whenet_b200.whenet import _is_device, _ptr
    from whenet_b200.yolo import _frame_table
    m = len(boxes)
    ptrs, hw = _frame_table(frames)
    out = torch.full((m, 224, 224, 3), 77, dtype=torch.uint8, device="cuda")
    rects = np.full((m, 4), -1, np.int32)
    valid = np.full(m, -1, np.int32)
    check(wn._L.whenet_crop_boxes_ragged_u8(wn._h, C.addressof(ptrs), _ptr(hw), len(frames), int(_is_device(frames[0])), _ptr(boxes),
                                            _ptr(frame_of), m, 1, _ptr(out), _ptr(rects), _ptr(valid)))
    wn.synchronize()
    return out.cpu().numpy(), rects, valid


@pytest.fixture(scope="module")
def crop_case():
    """Three frames of different sizes, 90 boxes inside, straddling a border or invalid (empty slices)."""
    rng = np.random.default_rng(5)
    sizes = [(1080, 1920), (480, 640), (1920, 1080)]
    frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in sizes]
    boxes, frame_of = [], []
    for i in range(84):
        f = i % 3
        H, W = sizes[f]
        y0, x0 = rng.uniform(-100, H), rng.uniform(-100, W)
        boxes.append((y0, x0, y0 + rng.uniform(1, 500), x0 + rng.uniform(1, 500)))
        frame_of.append(f)
    boxes += [(0, 0, 480, 640), (0, 0, 448 / 1.2, 448 / 1.4), (500.5, 10, 500.9, 200), (-300, -300, -10, -10), (np.nan, 10, 100, 200),
              (1500, 10, 1700, 200)]                                    # ... the last one is inside frame 2 only
    frame_of += [1, 0, 0, 1, 2, 2]
    return frames, np.array(boxes, np.float32), np.array(frame_of, np.int32)


def test_ragged_crops_equal_one_frame_crops(crop_case):
    import whenet_b200
    from test_gpu_pipeline import _crop_boxes
    frames, boxes, frame_of = crop_case
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=64)
    ref = np.zeros((len(boxes), 224, 224, 3), np.uint8)
    ref_rects = np.zeros((len(boxes), 4), np.int32)
    ref_valid = np.zeros(len(boxes), np.int32)
    for f, fr in enumerate(frames):
        sel = np.flatnonzero(frame_of == f)
        ref[sel], ref_rects[sel], ref_valid[sel] = _crop_boxes(wn, fr[None], np.ascontiguousarray(boxes[sel]), np.zeros(len(sel), np.int32))
    assert 0 < ref_valid.sum() < len(boxes) and ref_valid[-1] == 1
    for src in (frames, _cuda(frames)):
        got, rects, valid = _crop_ragged(wn, src, boxes, frame_of)
        assert np.array_equal(valid, ref_valid) and np.array_equal(rects, ref_rects)
        assert np.array_equal(got, ref)
    wn.close()


def test_ragged_crops_equal_cv2(crop_case):
    import whenet_b200
    cv2 = pytest.importorskip("cv2")
    frames, boxes, frame_of = crop_case
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=64)
    got, rects, valid = _crop_ragged(wn, frames, boxes, frame_of)
    for i, (y0, y1, x0, x1) in enumerate(rects):
        if valid[i]:
            ref = cv2.resize(cv2.cvtColor(frames[frame_of[i]][y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224))
            assert np.array_equal(got[i], ref), (i, boxes[i], rects[i])
        else:
            assert not got[i].any(), (i, boxes[i])
    wn.close()


# ----------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def wn16():
    import whenet_b200
    m = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=16)
    yield m
    m.close()


def test_ragged_pipeline_equals_per_frame(wn16, classes_file):
    """About 20 heads per frame (more than WHENet's sub-batch of 16 per chunk), chunks of 4, 4 and 1, host and device lists;
    the 300 x 1200 frames have heads in the letterbox padding whose slices are empty (NaN angles)."""
    from whenet_b200 import pipeline
    yolo = _biased_detector("full", classes_file)
    sizes = DET_SIZES + [(300, 1200), (640, 480), (1080, 1920)]
    frames = [np.ascontiguousarray(_frame(H, W, seed=50 + i)[:, :, ::-1]) for i, (H, W) in enumerate(sizes)]
    ref = [_per_frame_with_nan(yolo, wn16, f) for f in frames]
    assert max(sum(len(r[0]) for r in ref[c:c + 4]) for c in (0, 4)) > 16
    assert any(np.isnan(r[2]).any() for r in ref)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, frames), ref)
    _same(pipeline.detect_and_estimate_frames(yolo, wn16, _cuda(frames)), ref)
    yolo.close()


def test_ragged_pipeline_frames_without_detections(wn16, classes_file):
    from whenet_b200 import pipeline
    yolo = _biased_detector("two_classes", classes_file)
    sizes = [(832, 832), (600, 800), (700, 700), (900, 640), (832, 1000)]
    frames = [np.ascontiguousarray(_frame(H, W, seed=70 + i)) for i, (H, W) in enumerate(sizes)]
    frames += [np.full((H, W, 3), v, np.uint8) for (H, W), v in zip(((500, 500), (640, 900)), (0, 255))]
    frames = [frames[i] for i in (0, 5, 1, 2, 6, 3, 4)]
    yolo.score = 0.0
    top = [float(d[1].max()) for d in yolo.detect_frames(frames)]
    lo = sorted(set(top))
    yolo.score = (lo[0] + lo[1]) / 2
    ref = [_per_frame_with_nan(yolo, wn16, f) for f in frames]
    assert any(len(r[0]) == 0 for r in ref) and any(len(r[0]) for r in ref)
    for src in (frames, _cuda(frames)):
        _same(pipeline.detect_and_estimate_frames(yolo, wn16, src), ref)
    yolo.close()
