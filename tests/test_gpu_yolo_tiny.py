"""Tiny YOLOv3 head detector on the H100: every conv and every max-pool on its own GPU input against the float64 oracle, the
3x3 concat conv, the max-pool kernel bit for bit, end-to-end heads, the two-head decode + NMS against the float32
restatement, batch invariance, graph replay, switching networks on a live detector and the frame pipeline."""
import functools

import numpy as np
import pytest

import yolo_oracle as O
import yolo_tiny_cases as TC
import yolo_tiny_oracle as TO
from test_gpu_yolo import _assert_same, _check_ulp, _frame, _scale
from whenet_b200 import yolo_arch as Y

pytestmark = pytest.mark.gpu


def _tiny(**kw):
    import whenet_b200
    return whenet_b200.YOLO(None, anchors_path=TC.ANCHORS, **kw)


@pytest.fixture(scope="module")
def tiny():
    m = _tiny(max_frames=4)
    assert m.tiny
    yield m
    m.close()


@functools.lru_cache(maxsize=None)
def _layers(seed=0, classes=1):
    names, w = Y.random_weights(seed, classes, tiny=True)
    return Y.map_weights(names, w, tiny=True)[0]


def _folded_bf16(seed=0, classes=1):
    return [(Y.bf16_round(k).astype(np.float64), b) for k, b in (Y.fold_bn(d) for d in _layers(seed, classes))]


def _run_model(size):
    m = _tiny(model_image_size=size, max_frames=1)
    rgb = _frame(*TC.FRAMES[size], seed=3)
    m.detect(rgb)
    taps = [m.tap(i) for i in range(Y.TINY_N_CONV)]
    pooled = {i: m.tap(100 + i) for i in Y.TINY_POOLED}
    canvas = m.tap(-1).reshape(1, size[0], size[1], 3)
    m.close()
    return size, rgb, taps, pooled, canvas


@pytest.fixture(scope="module", params=TC.MODEL_SIZES, ids=lambda s: "%dx%d" % s)
def run_model(request):
    return _run_model(request.param)


def _outs(size, taps, classes=1):
    hw = Y.out_hw(*size, tiny=True)
    return [t.reshape(1, hw[i][0], hw[i][1], Y.cout(L, classes)).astype(np.float64) for i, (t, L) in enumerate(zip(taps, Y.TINY_LAYERS))]


def test_every_tiny_layer_and_pool_matches_oracle_on_its_own_input(run_model):
    size, _rgb, taps, pooled, canvas = run_model
    outs = _outs(size, taps)
    folded = _folded_bf16()
    ins = Y.in_hw(*size, tiny=True)
    shares, ratios, lin = [], [], []
    for i, L in enumerate(Y.TINY_LAYERS):
        x, up = TO.layer_inputs(i, outs, canvas / np.float32(255.0))
        if L.pool:      # the in-graph pool is exact: bit-identical to the max over the GPU's tap of the conv before it
            assert np.array_equal(pooled[i].reshape(x.shape), x), "pool before conv %d" % i
            assert x.shape[1:3] == ins[i]
        w, b = folded[i]
        ref = O.conv_layer(x, w, b, L.k, L.stride, L.bn, None, up)
        if L.bn:
            share, ratio = _check_ulp(outs[i], ref, "tiny layer %d" % i, _scale(x, w, L.k, L.stride, None, up))
            shares.append(share)
            ratios.append(ratio)
        else:
            lin.append(np.abs(outs[i] - ref).max() / np.abs(ref).max())
            assert lin[-1] <= 1e-5, i
    print("MEASURED tiny %dx%d layers: min share within 1 ulp %.5f, max |err| / (2 ulp + acc bound) %.3f, output convs max rel %.2g"
          % (size + (min(shares), max(ratios), max(lin))))


def test_tiny_end_to_end_heads_within_bound(run_model):
    size, rgb, taps, _pooled, canvas = run_model
    lb = O.letterbox(rgb, (size[1], size[0]))
    assert np.array_equal(lb, canvas[0].astype(np.uint8))
    outs = TO.body_numpy(lb[None] / np.float32(255.0), _layers())
    errs = [np.abs(taps[i].reshape(outs[i].shape) - outs[i]).max() / np.abs(outs[i]).max() for i in Y.TINY_HEADS]
    print("MEASURED tiny %dx%d heads: max abs err / max abs = %s" % (size + (", ".join("%.4g" % e for e in errs),)))
    assert max(errs) < 0.05, errs


@pytest.mark.parametrize("classes,size", [(c, s) for c, sizes in TC.CLASS_SIZES.items() for s in sizes])
def test_tiny_output_convs_with_more_classes(tmp_path, classes, size):
    p = tmp_path / "classes.txt"
    p.write_text("\n".join("class_%d" % i for i in range(classes)))
    m = _tiny(classes_path=str(p), model_image_size=size, max_frames=1)
    assert m.num_classes == classes
    m.detect(_frame(*TC.FRAMES[size], seed=classes))
    outs = _outs(size, [m.tap(i) for i in range(Y.TINY_N_CONV)], classes)
    folded = _folded_bf16(0, classes)
    for i in Y.TINY_HEADS:
        L = Y.TINY_LAYERS[i]
        w, b = folded[i]
        ref = O.conv_layer(outs[L.src], w, b, 1, 1, leaky=False)
        assert ref.shape[3] == Y.head_channels(classes)
        assert np.abs(outs[i] - ref).max() <= 1e-5 * np.abs(ref).max(), i
    m.close()


@pytest.mark.parametrize("case", TC.DEBUG_CONVS, ids=lambda c: "n%d-%dx%d-%d-%d-un%d" % (c[0], c[1], c[2], c[3], c[5], c[9]))
def test_debug_conv_3x3_concat(tiny, case):
    n, H, W, cin, c_up, cout, k, stride, _mode, _un = case
    rng = np.random.default_rng(H * 1000 + W + cout + n)
    x = Y.bf16_round(rng.standard_normal((n, H, W, cin - c_up)))
    up = Y.bf16_round(rng.standard_normal((n, H // 2, W // 2, c_up)))
    w = Y.bf16_round(rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin))
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    got = tiny.debug_conv(x, w, b, k, stride, up=up)
    ref = O.conv_layer(x, w, b, k, stride, up=up)
    _check_ulp(got, ref, str(case), _scale(x, w, k, stride, up=up))


@pytest.mark.parametrize("case", TC.POOLS, ids=lambda c: "n%d-%dx%d-c%d-s%d" % c)
def test_debug_maxpool_is_bit_exact(tiny, case):
    n, H, W, C, s = case
    x = Y.bf16_round(np.random.default_rng(H * 100 + W + C + s).standard_normal((n, H, W, C)) - 0.5)
    got = tiny.debug_maxpool(x, s)
    ref = TO.maxpool_same(x, s)
    assert got.shape == ref.shape and np.array_equal(got, ref)


# ----------------------------------------------------------------------------------------------- decode + NMS, two heads
@pytest.mark.parametrize("size,score", [((416, 416), 0.3), ((608, 608), 0.0), ((448, 608), 0.3)])
def test_tiny_decode_matches_restatement(size, score):
    m = _tiny(score=score, iou=0.45, model_image_size=size, max_frames=2)
    rng = np.random.default_rng(size[0] + size[1])
    heads = [rng.standard_normal((2, size[0] // 32 << l, size[1] // 32 << l, 18)).astype(np.float32) for l in range(2)]
    got = m.debug_decode(heads, 1080, 1920)
    for f in range(2):
        boxes, scores = TO.decode([h[f] for h in heads], m.anchors, 1, 1080, 1920)
        assert len(boxes) == Y.num_candidates(*size, tiny=True)
        rb, rs, rc, _ = O.yolo_eval(boxes, scores, score, 0.45)
        gb, gs, gc = got[f]
        assert len(gb) == len(rb) and np.array_equal(gc, rc)
        assert np.allclose(gb, rb, rtol=1e-4, atol=1e-3) and np.allclose(gs, rs, rtol=1e-5)
    m.close()


def test_tiny_decode_exact_logits_and_anchor_slots(tiny):
    """Exactly representable logits (t_w = t_h = 0: the box is its anchor) on a 416 x 416 frame: bit for bit against the
    restatement, and the box sizes are anchors 3, 4, 5 on head 0 and 1, 2, 3 on head 1 - never anchor 0."""
    hs = [np.zeros((1, 13 << l, 13 << l, 3, 6), np.float32) for l in range(2)]
    for h in hs:
        h[..., 2:5] = -200                  # score 0, zero-area box
    cells = {0: [(2, 3), (6, 9), (10, 1)], 1: [(4, 20), (12, 5), (22, 14)]}
    for l, yx in cells.items():
        for a, (y, x) in enumerate(yx):
            hs[l][0, y, x, a, 2:6] = (0, 0, 200, 200)           # score 1, the anchor's own size
    tiny.score, tiny.iou = 0.5, 1.0                             # nothing suppressed
    flat = [np.ascontiguousarray(h.reshape(h.shape[:3] + (-1,))) for h in hs]
    try:
        (gb, gs, gc), = tiny.debug_decode(flat, 416, 416)
    finally:
        tiny.score, tiny.iou = 0.3, 0.45
    with np.errstate(under="ignore", over="ignore"):
        boxes, scores = TO.decode([h[0] for h in flat], tiny.anchors, 1, 416, 416)
        rb, rs, rc, idx = O.yolo_eval(boxes, scores, 0.5, 1.0)
    assert np.array_equal(gb, rb) and np.array_equal(gs, rs) and np.array_equal(gc, rc) and len(gb) == 6
    sizes = {(int(round(b[3] - b[1])), int(round(b[2] - b[0]))) for b in gb}
    anchors = [tuple(int(v) for v in a) for a in tiny.anchors]
    assert sizes == {anchors[i] for i in (1, 2, 3, 4, 5)} and anchors[0] not in sizes
    by_head = {l: {(int(round(b[3] - b[1])), int(round(b[2] - b[0]))) for b, i in zip(gb, idx) if (i >= 507) == l} for l in (0, 1)}
    assert by_head == {0: {anchors[i] for i in (3, 4, 5)}, 1: {anchors[i] for i in (1, 2, 3)}}


# ----------------------------------------------------------------------------------------------- lifecycle and pipeline
def _run(m, frames):
    return m.detect_frames(frames), [m.tap(i) for i in Y.TINY_HEADS]


def test_tiny_batch_invariance_and_graph_replay(tiny):
    frames = np.stack([_frame(360, 640, seed=50 + s)[:, :, ::-1] for s in range(3)])
    tiny.score = 0.2
    try:
        batch, heads_b = _run(tiny, frames)
        assert all(len(r[0]) for r in batch)
        _assert_same(_run(tiny, frames), (batch, heads_b))       # replay of the captured graph
        for f in range(3):
            single = tiny.detect_frames(frames[f:f + 1])[0]
            for x, y in zip(single, batch[f]):
                assert np.array_equal(x, y), f
            for hb, i in zip(heads_b, Y.TINY_HEADS):
                assert np.array_equal(tiny.tap(i), hb.reshape(3, -1)[f]), (f, i)
    finally:
        tiny.score = 0.3


def test_switching_networks_on_a_live_detector_equals_a_fresh_one():
    import whenet_b200
    frames = np.stack([_frame(300, 400, seed=60 + s)[:, :, ::-1] for s in range(2)])
    full = whenet_b200.YOLO(None, max_frames=2, score=0.2)
    tiny = _tiny(max_frames=2, score=0.2)
    fresh_full, fresh_tiny = _run(full, frames), _run(tiny, frames)
    assert len(fresh_tiny[1]) == 2 and len(fresh_full[1]) == 2
    tiny_anchors, full_anchors = tiny.anchors, full.anchors
    names, w = Y.random_weights(0)
    tiny.load_layers(Y.map_weights(names, w)[0], anchors=full_anchors)      # tiny -> full
    assert not tiny.tiny
    got = tiny.detect_frames(frames), [tiny.tap(i) for i in Y.HEADS]
    _assert_same(got, (full.detect_frames(frames), [full.tap(i) for i in Y.HEADS]))
    full.load_layers(_layers(), anchors=tiny_anchors)                       # full -> tiny
    assert full.tiny
    _assert_same(_run(full, frames), fresh_tiny)
    with pytest.raises(RuntimeError, match="tiny YOLOv3: 13 convs"):
        full.load_layers(Y.map_weights(names, w)[0], anchors=tiny_anchors)  # 75 convs with 6 anchors
    _assert_same(_run(full, frames), fresh_tiny)                            # a refused load changes nothing
    full.close()
    tiny.close()


def test_tiny_detect_and_estimate_equals_detect_then_whenet(tiny):
    import whenet_b200
    from whenet_b200 import crops
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=32)
    tiny.score = 0.26
    try:
        for seed in range(20):
            frame = _frame(832, 832, seed=seed)
            rb, rs, _rc = tiny.detect(np.ascontiguousarray(frame[:, :, ::-1]))
            r = crops.rects_from_boxes(rb, 832, 832)
            if len(rb) and ((r[:, 0] < r[:, 1]) & (r[:, 2] < r[:, 3])).all():
                break
        else:
            pytest.fail("no frame with boxes inside it")
        boxes, scores, angles = whenet_b200.pipeline.detect_and_estimate(tiny, wn, frame)
        assert np.array_equal(boxes, rb) and np.array_equal(scores, rs)
        yaw, pitch, roll = wn.get_angle_from_frame(frame, rb)
        assert np.array_equal(angles, np.stack([yaw, pitch, roll], 1))
    finally:
        tiny.score = 0.3
        wn.close()
