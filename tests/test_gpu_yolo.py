"""YOLOv3 head detector on the H100: letterbox vs Pillow, the implicit-GEMM conv and every layer vs the float64 oracle,
end-to-end heads, decode + NMS vs the float32 restatement, batch invariance, graph replay and the frame pipeline."""
import functools

import numpy as np
import pytest

import yolo_cases as YC
import yolo_oracle as O
from whenet_b200 import yolo_arch as Y

pytestmark = pytest.mark.gpu

ULP1_SHARE = 0.999      # >= 99.9 % of elements within 1 bf16 ulp (DESIGN.md section 8)
ACC_REL = 2.0 ** -14    # fp32 accumulation over K ~ 1000 terms: K * 2^-24 of the sum of |terms|


@pytest.fixture(scope="module")
def yolo():
    import whenet_b200
    m = whenet_b200.YOLO(None, max_frames=4)
    yield m
    m.close()


def _ulp_bf16(ref):
    """bf16 ulp at |ref| (2^(e-7) for |ref| in [2^e, 2^(e+1)); values below 2^-30 use 2^-37)."""
    a = np.maximum(np.abs(ref), 2.0 ** -30)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


def _scale(x, w, k, stride, resid=None, up=None):
    """Per output: the conv of |x| with |w| (+ |resid|), the magnitude the fp32 sum cancels from."""
    ab = lambda a: None if a is None else np.abs(a)
    return O.conv_layer(np.abs(x), np.abs(w), None, k, stride, leaky=False, resid=ab(resid), up=ab(up))


def _check_ulp(got, ref, what, scale):
    """>= 99.9 % within 1 bf16 ulp of the float64 result; every element within 2 ulp plus the fp32 accumulation error bound
    (outputs that cancel to near zero have a tiny ulp but keep the absolute error of the sum).  Returns the share within 1 ulp
    and the largest error as a fraction of the bound."""
    d = np.abs(got.astype(np.float64) - ref)
    err = d / _ulp_bf16(ref)
    share = float(np.mean(err <= 1.0))
    bound = 2.0 * _ulp_bf16(ref) + ACC_REL * scale
    excess = d - bound
    assert share >= ULP1_SHARE and excess.max() <= 0, "%s: %.5f within 1 ulp, max %.2f ulp, bound exceeded by %.3g" % (
        what, share, err.max(), excess.max())
    return share, float((d / bound).max())


def _frame(h, w, seed):
    """A smooth synthetic frame (random noise resamples to near-gray, which exercises nothing)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([127 + 120 * np.sin(x / (7 + 3 * c) + y / (11 + c) + rng.random() * 6) for c in range(3)], -1)
    img += rng.normal(0, 6, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.mark.parametrize("hw", [(720, 1280), (1080, 1920), (416, 416), (37, 501), (300, 200)])
def test_letterbox_kernel_equals_pillow(yolo, hw):
    rgb = _frame(*hw, seed=hw[0])
    yolo.detect(rgb)
    got = yolo.tap(-1).reshape(416, 416, 3)
    assert np.array_equal(got, O.letterbox(rgb, (416, 416)).astype(np.float32))
    yolo.detect_frames(rgb[None, :, :, ::-1].copy())        # BGR in, swap_rb
    assert np.array_equal(yolo.tap(-1).reshape(416, 416, 3), got)


@pytest.mark.parametrize("k,stride", [(1, 1), (3, 1), (3, 2)])
@pytest.mark.parametrize("cout", [18, 32, 64, 1024])
@pytest.mark.parametrize("n", [1, 3])
def test_debug_conv_matches_float64(yolo, k, stride, cout, n):
    rng = np.random.default_rng(cout * 10 + k + n)
    cin = 64
    x = Y.bf16_round(rng.standard_normal((n, 13, 13, cin)))
    w = Y.bf16_round(rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin))
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    leaky = cout != 18
    got = yolo.debug_conv(x, w, b, k, stride, leaky=leaky)
    ref = O.conv_layer(x, w, b, k, stride, leaky=leaky)
    if leaky:
        _check_ulp(got, ref, "conv k%d s%d cout %d" % (k, stride, cout), _scale(x, w, k, stride))
    else:
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("n", [1, 2])
def test_debug_conv_residual_and_concat(yolo, n):
    rng = np.random.default_rng(7 + n)
    x = Y.bf16_round(rng.standard_normal((n, 14, 14, 128)))
    r = Y.bf16_round(rng.standard_normal((n, 14, 14, 128)))
    w = Y.bf16_round(rng.standard_normal((3, 3, 128, 128)) / 34)
    b = rng.standard_normal(128).astype(np.float32) * 0.1
    _check_ulp(yolo.debug_conv(x, w, b, 3, 1, resid=r), O.conv_layer(x, w, b, 3, 1, resid=r), "residual", _scale(x, w, 3, 1, resid=r))
    up = Y.bf16_round(rng.standard_normal((n, 7, 7, 128)))
    wc = Y.bf16_round(rng.standard_normal((1, 1, 256, 64)) / 16)
    _check_ulp(yolo.debug_conv(x, wc, b[:64], 1, 1, up=up), O.conv_layer(x, wc, b[:64], 1, 1, up=up), "concat", _scale(x, wc, 1, 1, up=up))


def _run_model(size):
    """One frame through a one-class detector at model input ``size``: the detections, every conv's tap and the canvas."""
    import whenet_b200
    m = whenet_b200.YOLO(None, model_image_size=size, max_frames=1)
    rgb = _frame(*YC.FRAMES[size], seed=3)
    res = m.detect(rgb)
    taps = [m.tap(i) for i in range(Y.N_CONV)]
    canvas = m.tap(-1).reshape(1, size[0], size[1], 3)
    m.close()
    return size, rgb, res, taps, canvas


@pytest.fixture(scope="module")
def run720():
    return _run_model(YC.MODEL_SIZES[0])          # 416 x 416, a 720p frame


@pytest.fixture(scope="module", params=YC.MODEL_SIZES[1:], ids=lambda s: "%dx%d" % s)
def run_model(request):
    return _run_model(request.param)


@functools.lru_cache(maxsize=None)
def _folded_bf16(seed=0):
    names, w = Y.random_weights(seed)
    layers, _ = Y.map_weights(names, w)
    return [(Y.bf16_round(k).astype(np.float64), b) for k, b in (Y.fold_bn(d) for d in layers)]


def _check_layer_taps(run):
    size, _rgb, _res, taps, canvas = run
    folded = _folded_bf16()
    hw = Y.out_hw(*size)
    outs = []
    for i, L in enumerate(Y.LAYERS):
        co = Y.cout(L, 1)
        outs.append(taps[i].reshape(1, hw[i][0], hw[i][1], co).astype(np.float64))
    shares, ratios, lin = [], [], []
    for i, L in enumerate(Y.LAYERS):
        x, up, res = O.layer_inputs(i, outs, canvas / np.float32(255.0))
        w, b = folded[i]
        ref = O.conv_layer(x, w, b, L.k, L.stride, L.bn, res, up)
        if L.bn:
            share, ratio = _check_ulp(outs[i], ref, "layer %d" % i, _scale(x, w, L.k, L.stride, res, up))
            shares.append(share)
            ratios.append(ratio)
        else:
            lin.append(np.abs(outs[i] - ref).max() / np.abs(ref).max())
            assert lin[-1] <= 1e-5, i
    print("MEASURED %dx%d layers: min share within 1 ulp %.5f, max |err| / (2 ulp + acc bound) %.3f, output convs max rel %.2g"
          % (size + (min(shares), max(ratios), max(lin))))


def _check_end_to_end(run):
    """The canvas equals Pillow's letterbox, and the three heads are within 5 % of the float64 body."""
    size, rgb, _res, taps, canvas = run
    lb = O.letterbox(rgb, (size[1], size[0]))
    assert np.array_equal(lb, canvas[0].astype(np.uint8))
    assert np.array_equal(YC.pil_letterbox(rgb, (size[1], size[0])), lb)
    names, w = Y.random_weights(0)
    layers, _ = Y.map_weights(names, w)
    outs = O.body_numpy(lb[None] / np.float32(255.0), layers)
    errs = []
    for i in Y.HEADS:
        got = taps[i].reshape(outs[i].shape)
        errs.append(np.abs(got - outs[i]).max() / np.abs(outs[i]).max())
    print("MEASURED %dx%d heads: max abs err / max abs = %s" % (size + (", ".join("%.4g" % e for e in errs),)))
    assert max(errs) < 0.05, errs         # bound from measurement, DESIGN.md section 8


def test_every_layer_tap_matches_oracle_on_its_own_input(run720):
    _check_layer_taps(run720)


def test_every_layer_tap_matches_oracle_at_other_input_sizes(run_model):
    _check_layer_taps(run_model)


def test_end_to_end_heads_within_bound(run720):
    _check_end_to_end(run720)


def test_end_to_end_heads_within_bound_at_other_input_sizes(run_model):
    _check_end_to_end(run_model)


@pytest.mark.parametrize("size,score", [((416, 416), 0.3), ((608, 608), 0.0)])
def test_debug_decode_matches_restatement(size, score):
    import whenet_b200
    m = whenet_b200.YOLO(None, score=score, iou=0.45, model_image_size=size, max_frames=2)
    rng = np.random.default_rng(size[0])
    heads = [rng.standard_normal((2, size[0] // 32 << l, size[1] // 32 << l, 18)).astype(np.float32) for l in range(3)]
    img_h, img_w = 1080, 1920
    got = m.debug_decode(heads, img_h, img_w)
    for f in range(2):
        boxes, scores = O.decode([h[f] for h in heads], m.anchors, 1, img_h, img_w)
        if score == 0.0:
            assert (scores >= 0).all()          # every candidate passes the mask
        rb, rs, rc, _ = O.yolo_eval(boxes, scores, score, 0.45)
        gb, gs, gc = got[f]
        assert len(gb) == len(rb) and np.array_equal(gc, rc)
        assert np.allclose(gb, rb, rtol=1e-4, atol=1e-3) and np.allclose(gs, rs, rtol=1e-5)
    m.close()


def test_batch_invariance_and_graph_replay(yolo):
    frames = np.stack([_frame(360, 640, seed=s)[:, :, ::-1] for s in range(4)])
    batch = yolo.detect_frames(frames)
    heads_b = [yolo.tap(i) for i in Y.HEADS]
    again = yolo.detect_frames(frames)          # replay of the captured graph
    for a, b in zip(batch, again):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    for f in range(4):
        single = yolo.detect_frames(frames[f:f + 1])[0]
        for x, y in zip(single, batch[f]):
            assert np.array_equal(x, y), f
        for hb, i in zip(heads_b, Y.HEADS):
            s = yolo.tap(i)
            assert np.array_equal(s, hb.reshape(4, -1)[f]), (f, i)


def test_detect_and_estimate_equals_detect_then_whenet(yolo):
    import whenet_b200
    from whenet_b200 import crops
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=32)
    yolo.score = 0.26           # the random-weight detector's scores sit near 0.25
    try:
        for seed in range(20):
            # a square frame fills the letterbox: every box centre lies inside the frame
            frame = _frame(832, 832, seed=seed)
            rb, rs, _rc = yolo.detect(np.ascontiguousarray(frame[:, :, ::-1]))
            r = crops.rects_from_boxes(rb, 832, 832)
            # boxes are not clipped (model.py:176): the reference's slice would be empty for one outside the frame
            if len(rb) and ((r[:, 0] < r[:, 1]) & (r[:, 2] < r[:, 3])).all():
                break
        else:
            pytest.fail("no frame with boxes inside it")
        boxes, scores, angles = whenet_b200.pipeline.detect_and_estimate(yolo, wn, frame)
        assert np.array_equal(boxes, rb) and np.array_equal(scores, rs)
        yaw, pitch, roll = wn.get_angle_from_frame(frame, rb)
        assert np.array_equal(angles, np.stack([yaw, pitch, roll], 1))
    finally:
        yolo.score = 0.3
        wn.close()


# ----------------------------------------------------------------------------------------------- more shapes and class counts
@pytest.mark.parametrize("case", YC.DEBUG_CONVS, ids=lambda c: "%s-n%d-%dx%d-%d-%d-k%ds%d-un%d" % (c[8], c[0], c[1], c[2], c[3], c[5], c[6], c[7], c[9]))
def test_debug_conv_shapes_and_tile_widths(yolo, case):
    """Non-square frames, odd sides at stride 2, concat with H != W, and shapes that plan 64- and 128-wide tiles (the plans are
    checked by test_yolo_plans.py)."""
    n, H, W, cin, c_up, cout, k, stride, mode, _un = case
    rng = np.random.default_rng(H * 1000 + W + cout)
    x = Y.bf16_round(rng.standard_normal((n, H, W, cin - c_up)))
    up = Y.bf16_round(rng.standard_normal((n, H // 2, W // 2, c_up))) if mode == "cat" else None
    r = Y.bf16_round(rng.standard_normal((n, H // stride, W // stride, cout))) if mode == "res" else None
    w = Y.bf16_round(rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin))
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    leaky = mode != "f32"
    got = yolo.debug_conv(x, w, b, k, stride, leaky=leaky, resid=r, up=up)
    ref = O.conv_layer(x, w, b, k, stride, leaky=leaky, resid=r, up=up)
    if leaky:
        _check_ulp(got, ref, str(case), _scale(x, w, k, stride, resid=r, up=up))
    else:
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


def test_batch_invariance_non_square_odd_batch():
    import whenet_b200
    m = whenet_b200.YOLO(None, model_image_size=(448, 608), max_frames=4, score=0.2)
    frames = np.stack([_frame(360, 640, seed=10 + s)[:, :, ::-1] for s in range(3)])
    batch = m.detect_frames(frames)
    heads_b = [m.tap(i).reshape(3, -1) for i in Y.HEADS]
    assert all(len(r[0]) for r in batch)
    for f in range(3):
        single = m.detect_frames(frames[f:f + 1])[0]
        for x, y in zip(single, batch[f]):
            assert np.array_equal(x, y), f
        for hb, i in zip(heads_b, Y.HEADS):
            assert np.array_equal(m.tap(i), hb[f]), (f, i)
    m.close()


@pytest.fixture(scope="module")
def classes_file(tmp_path_factory):
    def make(c):
        p = tmp_path_factory.mktemp("classes") / ("classes_%d.txt" % c)
        p.write_text("\n".join("class_%d" % i for i in range(c)))
        return str(p)
    return make


@pytest.mark.parametrize("classes,size", [(c, s) for c, sizes in YC.CLASS_SIZES.items() for s in sizes])
def test_output_convs_with_more_classes(classes_file, classes, size):
    """Head widths 3 * (5 + C) = 21 and 255 (a 63-column tail tile at 608 x 608) against the oracle on the GPU's own input."""
    import whenet_b200
    m = whenet_b200.YOLO(None, classes_path=classes_file(classes), model_image_size=size, max_frames=1)
    assert m.num_classes == classes
    m.detect(_frame(*YC.FRAMES[size], seed=classes))
    names, w = Y.random_weights(0, classes)
    layers, _ = Y.map_weights(names, w)
    hw = Y.out_hw(*size)
    for i in Y.HEADS:
        L = Y.LAYERS[i]
        x = m.tap(L.src).reshape(1, hw[L.src][0], hw[L.src][1], Y.LAYERS[L.src].cout).astype(np.float64)
        k, b = Y.fold_bn(layers[i])
        ref = O.conv_layer(x, Y.bf16_round(k).astype(np.float64), b, 1, 1, leaky=False)
        assert ref.shape[3] == Y.head_channels(classes)
        got = m.tap(i).reshape(ref.shape)
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), i
    m.close()


@pytest.mark.parametrize("classes,score", [(2, 0.0), (2, 0.6), (80, 0.5)])
def test_decode_nms_with_more_classes(classes_file, classes, score):
    """Per-class masks, NMS and the class-by-class output slots; the class logits get a per-class offset so that the classes
    keep different numbers of boxes."""
    import whenet_b200
    m = whenet_b200.YOLO(None, classes_path=classes_file(classes), score=score, iou=0.45, max_frames=2)
    rng = np.random.default_rng(classes)
    heads = [rng.standard_normal((2, 13 << l, 13 << l, 3, 5 + classes)).astype(np.float32) for l in range(3)]
    for h in heads:
        h[..., 5:] += np.linspace(-3, 0.5, classes, dtype=np.float32)
    heads = [h.reshape(h.shape[:3] + (-1,)) for h in heads]
    got = m.debug_decode(heads, 1080, 1920)
    for f in range(2):
        boxes, scores = O.decode([h[f] for h in heads], m.anchors, classes, 1080, 1920)
        rb, rs, rc, _ = O.yolo_eval(boxes, scores, score, 0.45)
        gb, gs, gc = got[f]
        assert len(gb) == len(rb) and np.array_equal(gc, rc), f
        assert np.allclose(gb, rb, rtol=1e-4, atol=1e-3) and np.allclose(gs, rs, rtol=1e-5), f
        if score > 0:
            assert len(set(np.bincount(gc, minlength=classes).tolist())) > 1
    m.close()


# ----------------------------------------------------------------------------------------------- decode / NMS edge cases
# Logits whose float32 results are exact on both sides: t = 0 gives sigmoid 0.5 and exp 1, t = -200 gives 0, t = 200 gives 1,
# t = 100 gives exp = inf.  So the kernel must equal the restatement bit for bit.
_SCORE_LOGITS = {1.0: (200, 200), 0.5: (200, 0), 0.25: (0, 0), 0.0: (-200, 200)}


def _blank(n, size=(416, 416)):
    """One-class heads (n, gh, gw, 3, 6) whose every candidate scores 0 with a zero-area box."""
    hs = []
    for l in range(3):
        h = np.zeros((n, size[0] // 32 << l, size[1] // 32 << l, 3, 6), np.float32)
        h[..., 2:5] = -200
        hs.append(h)
    return hs


def _cand(size, i):
    """candidate index -> (layer, y, x, anchor): layer 0, 1, 2, then (y, x, anchor) as the decode orders them"""
    gh, gw = size[0] // 32, size[1] // 32
    for l in range(3):
        if i < 3 * gh * gw:
            cell, a = divmod(i, 3)
            return l, cell // gw, cell % gw, a
        i -= 3 * gh * gw
        gh, gw = 2 * gh, 2 * gw
    raise IndexError(i)


def _put(hs, i, score, twh=(0, 0), f=0, size=(416, 416)):
    l, y, x, a = _cand(size, i)
    t = hs[l][f, y, x, a]
    t[2:4] = twh
    t[4:6] = _SCORE_LOGITS[score]


def _decode_exact(m, hs, img_h=480, img_w=640, max_boxes=20):
    """Device decode + NMS equal to the float32 restatement bit for bit, per frame; returns the kept candidate indices."""
    flat = [np.ascontiguousarray(h.reshape(h.shape[:3] + (-1,))) for h in hs]
    got = m.debug_decode(flat, img_h, img_w, max_boxes)
    kept = []
    for f, (gb, gs, gc) in enumerate(got):
        with np.errstate(over="ignore", invalid="ignore", under="ignore"):
            boxes, scores = O.decode([h[f] for h in flat], m.anchors, 1, img_h, img_w)
            rb, rs, rc, idx = O.yolo_eval(boxes, scores, m.score, m.iou, max_boxes)
        assert np.array_equal(gb, rb) and np.array_equal(gs, rs) and np.array_equal(gc, rc), (f, len(gb), len(rb))
        kept.append(idx.tolist())
    return kept


@pytest.fixture(scope="module")
def dec():
    import whenet_b200
    m = whenet_b200.YOLO(None, max_frames=4)
    yield m
    m.close()


def _f32_next(v, toward):
    return float(np.nextafter(np.float32(v), np.float32(toward)))


def test_kernel_score_threshold_is_inclusive(dec):
    hs = _blank(1)
    _put(hs, 40, 0.25)
    dec.iou = 0.45
    dec.score = 0.25
    assert _decode_exact(dec, hs) == [[40]]
    dec.score = _f32_next(0.25, 1)
    assert _decode_exact(dec, hs) == [[]]


def test_kernel_iou_threshold_is_strict(dec):
    hs = _blank(1)
    i, j = 3 * (5 * 13 + 5), 3 * (5 * 13 + 6)          # anchor 0 of two neighbouring 13 x 13 cells
    _put(hs, i, 1.0)
    _put(hs, j, 0.5)
    with np.errstate(over="ignore"):
        boxes, _ = O.decode([h[0].reshape(h.shape[1:3] + (-1,)) for h in hs], dec.anchors, 1, 480, 640)
    thr = O.iou_tf(boxes[i], boxes[j])
    assert 0.3 < thr < 1
    dec.score = 0.25
    dec.iou = float(thr)
    assert _decode_exact(dec, hs) == [[i, j]]          # IoU == threshold: not suppressed
    dec.iou = _f32_next(thr, 0)
    assert _decode_exact(dec, hs) == [[i]]


def test_kernel_equal_scores_keep_lower_index_first(dec):
    """Ties within one thread (i, i + 1024, i + 2048: different alive bits), across warps and across the three head layers."""
    hs = _blank(1)
    ties = [3, 3 + 1024, 3 + 2048, 100, 700, 5000, 3 + 5 * 1024]
    assert [_cand((416, 416), i)[0] for i in (3, 700, 5000)] == [0, 1, 2]
    for i in ties:
        _put(hs, i, 0.5, twh=(-200, -200))
    for i in (9000, 50):
        _put(hs, i, 1.0, twh=(-200, -200))
    for i in (8000, 7):
        _put(hs, i, 0.25, twh=(-200, -200))
    dec.score, dec.iou = 0.25, 0.45
    assert _decode_exact(dec, hs) == [[50, 9000] + sorted(ties) + [7, 8000]]


def test_kernel_zero_area_boxes_neither_suppress_nor_are_suppressed(dec):
    hs = _blank(1)
    c = 3 * (6 * 13 + 6)                                # the three anchors of one 13 x 13 cell
    _put(hs, c, 0.5)
    _put(hs, c + 1, 1.0, twh=(-200, 0))                 # zero width, the best score, on top of both boxes
    _put(hs, c + 2, 0.25)                               # the largest anchor: IoU 0.086 with anchor 0's box
    z = 507 + 3 * (12 * 26 + 12)                        # zero height, inside anchor 0's box, on the 26 x 26 grid
    _put(hs, z, 0.25, twh=(0, -200))
    dec.score, dec.iou = 0.25, 0.05
    assert _decode_exact(dec, hs) == [[c + 1, c, z]]


def test_kernel_keeps_score_zero_candidates_after_positive_ones(dec):
    hs = _blank(1)
    for i, s in ((500, 1.0), (20, 0.5), (7000, 0.25)):
        _put(hs, i, s, twh=(-200, -200))
    dec.score, dec.iou = 0.0, 0.45
    assert _decode_exact(dec, hs) == [[500, 20, 7000] + list(range(17))]


@pytest.mark.parametrize("max_boxes", [1, 20, 256])
def test_kernel_max_boxes(dec, max_boxes):
    hs = _blank(1)
    cands = list(range(0, 9000, 30))                    # 300 survivors
    for i in cands:
        _put(hs, i, 0.5, twh=(-200, -200))
    dec.score, dec.iou = 0.25, 0.45
    assert _decode_exact(dec, hs, max_boxes=max_boxes) == [cands[:max_boxes]]


def test_kernel_nan_iou_suppresses_nothing(dec):
    dec.score, dec.iou = 0.3, 0.45
    kept = _decode_exact(dec, [h.reshape(h.shape[:3] + (3, 6)) for h in YC.nan_iou_heads()])
    assert len(kept[0]) == 2


def _sparse_heads(rng, n, size, k=80):
    """n frames of k random candidates each: scores and box kinds drawn from the exact set, different per frame."""
    hs = _blank(n, size)
    nc = Y.num_candidates(*size)
    for f in range(n):
        for i in rng.choice(nc, k, replace=False):
            twh = [(0, 0), (-200, -200), (0, -200), (-200, 0)][rng.integers(4)]
            _put(hs, int(i), [1.0, 0.5, 0.25][rng.integers(3)], twh=twh, f=f, size=size)
    return hs


@pytest.mark.parametrize("size,img", [((416, 416), "int_round"), ((448, 608), (1080, 1920)), ((608, 448), (480, 640)),
                                      ((96, 160), (333, 500))], ids=str)
def test_kernel_decode_frames_non_square_and_letterbox_extents(size, img):
    """Four frames of different content in one call (per-frame workspaces), non-square heads (gh0 != gw0) and an image size
    whose int() and round() letterbox extents differ."""
    import whenet_b200
    if img == "int_round":
        W, H = YC.int_round_differ()
        img = (H, W)
    m = whenet_b200.YOLO(None, model_image_size=size, max_frames=4, score=0.25, iou=0.45)
    kept = _decode_exact(m, _sparse_heads(np.random.default_rng(size[0] + size[1]), 4, size), *img)
    assert all(kept) and len({tuple(k) for k in kept}) == 4
    m.close()


# ----------------------------------------------------------------------------------------------- detector lifecycle
def _run(m, frames, rgb=False):
    """Detections of a batch plus the three head taps: what must repeat bit for bit."""
    res = [m.detect(f) for f in frames] if rgb else m.detect_frames(frames)
    return res, [m.tap(i) for i in Y.HEADS]


def _assert_same(a, b):
    (ra, ha), (rb, hb) = a, b
    assert len(ra) == len(rb)
    for x, y in zip(ra, rb):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)
    for u, v in zip(ha, hb):
        assert np.array_equal(u, v)


def test_buffer_growth_and_graph_eviction_replay_nothing_stale():
    import whenet_b200
    m = whenet_b200.YOLO(None, max_frames=4, score=0.2)
    small = np.stack([_frame(120, 160, seed=s) for s in range(2)])
    first = _run(m, small)
    assert all(len(r[0]) for r in first[0])
    _run(m, np.stack([_frame(720, 1280, seed=s) for s in range(3)]))        # the frame buffer grows: every graph is freed
    _assert_same(_run(m, small), first)
    for k in range(17):                                                     # 17 more keys: the 16-graph cache is emptied
        _run(m, _frame(40 + k, 64 + 3 * k, seed=k)[None], rgb=k % 2 == 1)
    _assert_same(_run(m, small), first)
    m.close()


def test_load_layers_on_a_live_detector_equals_a_fresh_one():
    import whenet_b200
    frames = np.stack([_frame(300, 400, seed=s) for s in range(2)])
    live = whenet_b200.YOLO(None, max_frames=2, score=0.2)
    before = _run(live, frames)
    names, w = Y.random_weights(1)
    live.load_layers(Y.map_weights(names, w)[0])
    after = _run(live, frames)
    fresh = whenet_b200.YOLO(None, seed=1, max_frames=2, score=0.2)
    _assert_same(after, _run(fresh, frames))
    assert not np.array_equal(after[1][0], before[1][0])
    live.close()
    fresh.close()


def test_device_frames_equal_host_frames(yolo):
    import torch
    frames = np.stack([_frame(360, 480, seed=20 + s)[:, :, ::-1] for s in range(3)])
    host = _run(yolo, frames)
    _assert_same(_run(yolo, torch.from_numpy(frames).cuda()), host)


def test_more_frames_than_max_frames_run_in_chunks(yolo):
    frames = np.stack([_frame(240, 320, seed=30 + s)[:, :, ::-1] for s in range(6)])
    yolo.score = 0.2
    try:
        whole = yolo.detect_frames(frames)
        parts = yolo.detect_frames(frames[:4]) + yolo.detect_frames(frames[4:])
    finally:
        yolo.score = 0.3
    assert len(whole) == 6 and all(len(r[0]) for r in whole)
    for a, b in zip(whole, parts):
        for u, v in zip(a, b):
            assert np.array_equal(u, v)


def test_empty_letterbox_raises_and_the_detector_recovers(yolo):
    frames = np.stack([_frame(200, 300, seed=40 + s)[:, :, ::-1] for s in range(2)])
    first = _run(yolo, frames)
    with pytest.raises(RuntimeError, match="empty"):
        yolo.detect(np.zeros((2, 1920, 3), np.uint8))                       # 1920 x 2 -> 416 x 0
    _assert_same(_run(yolo, frames), first)


# ----------------------------------------------------------------------------------------------- letterbox against Pillow
@pytest.fixture(scope="module", params=[(416, 416), (320, 608)], ids=lambda s: "%dx%d" % s)
def lb_det(request):
    import whenet_b200
    m = whenet_b200.YOLO(None, model_image_size=request.param, max_frames=1)
    yield m
    m.close()


@pytest.mark.parametrize("wh", YC.SIZES, ids=str)
def test_letterbox_kernel_equals_pillow_every_size(lb_det, wh):
    W, H = wh
    h, w = lb_det.model_image_size
    img = np.random.default_rng(W * 7919 + H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref = YC.pil_letterbox(img, (w, h))
    lb_det.detect(img)
    assert np.array_equal(lb_det.tap(-1).reshape(h, w, 3), ref)
    lb_det.detect_frames(np.ascontiguousarray(img[None, :, :, ::-1]))      # BGR in, swap_rb
    assert np.array_equal(lb_det.tap(-1).reshape(h, w, 3), ref)
