"""YOLOv3 head detector, everything that runs without a GPU: the letterbox restatement against Pillow, the two float64 body
restatements against each other, the decode/NMS restatement on hand-built cases, weight mapping and argument validation."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLD
import yolo_oracle as O
from yolo_cases import SIZES, int_round_differ as _int_round_differ, pil_letterbox as _pil_letterbox, nan_iou_heads
from whenet_b200 import yolo_arch as Y


@pytest.mark.parametrize("wh", SIZES)
def test_letterbox_oracle_equals_pillow(wh):
    W, H = wh
    img = np.random.default_rng(W * 7919 + H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    for size in ((416, 416), (608, 320)):
        assert np.array_equal(O.letterbox(img, size), _pil_letterbox(img, size)), (wh, size)


def test_int_and_round_extents_differ_somewhere():
    W, H = _int_round_differ()
    nw, nh, _, _ = O.letterbox_geometry(W, H, 416, 416)
    _off, scale = O.correct_params(416, 416, H, W)
    assert (nh, nw) != tuple(int(v) for v in np.float32(416) / scale)      # the letterbox and the box correction disagree here


def test_numpy_body_equals_torch_body():
    names, w = Y.random_weights(3)
    layers, _ = Y.map_weights(names, w)
    x = np.random.default_rng(1).random((1, 64, 96, 3))
    outs = O.body_numpy(x, layers)
    heads_t = O.body_torch(x, layers)
    for i, t in zip(Y.HEADS, heads_t):
        assert outs[i].shape == t.shape
        assert np.abs(outs[i] - t).max() <= 1e-9 * np.abs(t).max(), i
        assert 0.05 < np.abs(t).max() < 50          # activations stay O(1) through 75 layers


def test_bn_folding_equals_unfolded():
    names, w = Y.random_weights(4)
    layers, _ = Y.map_weights(names, w)
    x = np.random.default_rng(2).random((1, 32, 64, 3))
    ref = O.body_numpy(x, layers)
    got = O.body_numpy(x, [Y.fold_bn(d) for d in layers], folded=True)
    for a, b in zip(ref, got):
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(a).max())


def test_table_and_flops():
    assert Y.N_CONV == 75 and sum(L.bn for L in Y.LAYERS) == 72
    assert abs(2 * Y.macs_per_frame(416, 416) / 1e9 - 65.3) < 0.05
    assert Y.num_candidates(416, 416) == 10647 and Y.num_candidates(608, 608) == 22743
    hw = Y.out_hw(416, 416)
    assert [(hw[i], Y.LAYERS[i].cout) for i in Y.SKIP_LAYERS] == [((52, 52), 256), ((26, 26), 512)]
    assert [hw[i] for i in Y.HEADS] == [(13, 13), (26, 26), (52, 52)]


def test_default_anchors_equal_reference_file():
    assert np.array_equal(Y.read_anchors(os.path.join(GOLD, "yolo_anchors.txt")), Y.DEFAULT_ANCHORS)


def test_weight_mapping_by_order_with_offset_numbering():
    names, w = Y.random_weights(5)
    ref, C = Y.map_weights(names, w)
    assert C == 1
    # the same model built second in a session: every conv2d_N / batch_normalization_N shifted
    def shift(n):
        base, _, rest = n.partition("/")
        kind, _, num = base.rpartition("_")
        return "%s_%d%s%s" % (kind, int(num) + 100, "/" if rest else "", rest)
    names2 = [shift(n) for n in names]
    w2 = {shift(k): v for k, v in w.items()}
    got, _ = Y.map_weights(names2, w2)
    for a, b in zip(ref, got):
        for k in a:
            if k != "name":
                assert np.array_equal(a[k], b[k])


def test_weight_mapping_refuses_bad_files():
    names, w = Y.random_weights(6)
    w1 = dict(w)
    del w1["batch_normalization_3/gamma:0"]
    with pytest.raises(ValueError, match="batch_normalization_3"):
        Y.map_weights(names, w1)
    w2 = dict(w)
    w2["conv2d_5/kernel:0"] = np.zeros((3, 3, 64, 65), np.float32)
    with pytest.raises(ValueError, match="conv2d_5"):
        Y.map_weights(names, w2)
    w3 = {k: v for k, v in w.items() if not k.startswith("conv2d_75/")}
    with pytest.raises(ValueError, match="conv"):
        Y.map_weights([n for n in names if n != "conv2d_75"], w3)


# ----------------------------------------------------------------------------------------------- decode / NMS restatement
def _box(y0, x0, y1, x1):
    return np.array([y0, x0, y1, x1], np.float32)


def test_iou_threshold_is_strict():
    a = _box(0, 0, 10, 10)
    b = _box(0, 0, 10, 5)          # IoU exactly 0.5
    assert O.iou_tf(a, b) == np.float32(0.5)
    boxes = np.stack([a, b])
    s = np.array([0.9, 0.8], np.float32)
    assert O.nms_tf(boxes, s, 20, 0.5) == [0, 1]                     # 0.5 is not > 0.5: kept
    assert O.nms_tf(boxes, s, 20, np.nextafter(np.float32(0.5), np.float32(0))) == [0]    # just below: suppressed
    assert O.nms_tf(boxes, s, 20, np.nextafter(np.float32(0.5), np.float32(1))) == [0, 1]


def test_zero_and_negative_areas_never_suppress():
    boxes = np.stack([_box(0, 0, 10, 10), _box(5, 5, 5, 9), _box(10, 10, 0, 0), _box(0, 0, -1, 10)])
    s = np.array([0.9, 0.8, 0.7, 0.6], np.float32)
    # the flipped box (10,10,0,0) has positive area after min/max and overlaps box 0 fully: suppressed
    assert O.nms_tf(boxes, s, 20, 0.3) == [0, 1, 3]


def test_more_survivors_than_max_boxes():
    boxes = np.stack([_box(20 * i, 0, 20 * i + 10, 10) for i in range(30)])
    s = np.linspace(0.9, 0.4, 30).astype(np.float32)
    assert O.nms_tf(boxes, s, 20, 0.45) == list(range(20))


def test_two_classes_and_threshold_inclusive():
    boxes = np.stack([_box(0, 0, 10, 10), _box(1, 1, 11, 11), _box(50, 50, 60, 60)])
    scores = np.array([[0.3, 0.1], [0.9, 0.5], [0.2999, 0.6]], np.float32)
    b, s, c, idx = O.yolo_eval(boxes, scores, 0.3, 0.45)
    # class 0: candidates 0 (score exactly 0.3, kept by >=) and 1; 1 suppresses 0.  class 1: 2 then 1.
    assert idx.tolist() == [1, 2, 1] and c.tolist() == [0, 1, 1]
    assert s.tolist() == [np.float32(0.9), np.float32(0.6), np.float32(0.5)]
    scores[0, 0] = np.float32(0.3)
    b, s, c, idx = O.yolo_eval(boxes[:1], scores[:1], 0.3, 0.45)
    assert idx.tolist() == [0]


def test_equal_scores_keep_lower_index_first():
    boxes = np.stack([_box(0, 0, 10, 10), _box(0, 0, 10, 10)])
    assert O.nms_tf(boxes, np.array([0.5, 0.5], np.float32), 20, 0.45) == [0]


def test_nan_iou_suppresses_nothing():
    heads = nan_iou_heads()
    with np.errstate(over="ignore", invalid="ignore"):
        boxes, scores = O.decode([h[0] for h in heads], Y.DEFAULT_ANCHORS, 1, 480, 640)
        i, j = np.nonzero(scores[:, 0] == 1)[0]
        assert np.isnan(O.iou_tf(boxes[i], boxes[j]))
        _b, s, _c, idx = O.yolo_eval(boxes, scores, 0.3, 0.45)
    assert idx.tolist() == [i, j] and s.tolist() == [1.0, 1.0]         # TF suppresses only when IoU > threshold


def test_correct_boxes_reproduce_round_and_int():
    W, H = _int_round_differ()
    off, scale = O.correct_params(416, 416, H, W)
    new = np.float32(416) / scale
    m = np.float32(min(np.float32(416) / np.float32(H), np.float32(416) / np.float32(W)))
    assert np.allclose(new, np.round(np.array([H, W], np.float32) * m))


# ----------------------------------------------------------------------------------------------- library, no GPU
def test_detector_argument_validation_without_gpu():
    from whenet_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    assert L.whenet_det_create(None, 0, 416, 416, 1) == -1
    for hw in ((400, 416), (416, 0), (640, 416), (0, 0), (16, 32)):
        assert L.whenet_det_create(C.byref(h), 0, hw[0], hw[1], 1) == -1, hw
        assert b"multiples of 32" in L.whenet_last_error()
    assert L.whenet_det_create(C.byref(h), 0, 416, 416, 0) == -1 and b"max_frames" in L.whenet_last_error()
    assert L.whenet_det_load_weights(None, None, 0, None, 0) == -1
    assert L.whenet_det_detect_u8(None, None, 1, 10, 10, 0, 1, 0.3, 0.45, 20, None, None, None, None) == -1
    assert L.whenet_det_debug_conv(None, None, None, 1, 13, 13, 64, 0, None, None, 3, 1, 64, 1, None, None) == -1
    assert L.whenet_det_num_classes(None) == 0
    L.whenet_det_destroy(None)
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        assert L.whenet_det_create(C.byref(h), 0, 416, 416, 1) == -2


def test_yolo_refuses_image_sized_input():
    import whenet_b200
    with pytest.raises(ValueError, match="None"):
        whenet_b200.YOLO(model_image_size=(None, None))
    with pytest.raises(ValueError, match="multiples of 32"):
        whenet_b200.YOLO(model_image_size=(400, 416))
