"""YOLOv3 head detector on the H100: letterbox vs Pillow, the implicit-GEMM conv and every layer vs the float64 oracle,
end-to-end heads, decode + NMS vs the float32 restatement, batch invariance, graph replay and the frame pipeline."""
import numpy as np
import pytest

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
    (outputs that cancel to near zero have a tiny ulp but keep the absolute error of the sum)."""
    d = np.abs(got.astype(np.float64) - ref)
    err = d / _ulp_bf16(ref)
    share = float(np.mean(err <= 1.0))
    excess = d - (2.0 * _ulp_bf16(ref) + ACC_REL * scale)
    assert share >= ULP1_SHARE and excess.max() <= 0, "%s: %.5f within 1 ulp, max %.2f ulp, bound exceeded by %.3g" % (
        what, share, err.max(), excess.max())


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


@pytest.fixture(scope="module")
def run720(yolo):
    rgb = _frame(720, 1280, seed=3)
    res = yolo.detect(rgb)
    taps = [yolo.tap(i) for i in range(Y.N_CONV)]
    canvas = yolo.tap(-1).reshape(1, 416, 416, 3)
    return rgb, res, taps, canvas


def _folded_bf16(seed=0):
    names, w = Y.random_weights(seed)
    layers, _ = Y.map_weights(names, w)
    return [(Y.bf16_round(k).astype(np.float64), b) for k, b in (Y.fold_bn(d) for d in layers)]


def test_every_layer_tap_matches_oracle_on_its_own_input(run720):
    _rgb, _res, taps, canvas = run720
    folded = _folded_bf16()
    hw = Y.out_hw(416, 416)
    outs = []
    for i, L in enumerate(Y.LAYERS):
        co = Y.cout(L, 1)
        outs.append(taps[i].reshape(1, hw[i][0], hw[i][1], co).astype(np.float64))
    for i, L in enumerate(Y.LAYERS):
        x, up, res = O.layer_inputs(i, outs, canvas / np.float32(255.0))
        w, b = folded[i]
        ref = O.conv_layer(x, w, b, L.k, L.stride, L.bn, res, up)
        if L.bn:
            _check_ulp(outs[i], ref, "layer %d" % i, _scale(x, w, L.k, L.stride, res, up))
        else:
            assert np.abs(outs[i] - ref).max() <= 1e-5 * np.abs(ref).max(), i


def test_end_to_end_heads_within_bound(run720):
    rgb, _res, taps, _canvas = run720
    assert np.array_equal(O.letterbox(rgb, (416, 416)), _canvas[0].astype(np.uint8))
    names, w = Y.random_weights(0)
    layers, _ = Y.map_weights(names, w)
    outs = O.body_numpy(O.letterbox(rgb, (416, 416))[None] / np.float32(255.0), layers)
    hw = Y.out_hw(416, 416)
    for i in Y.HEADS:
        got = taps[i].reshape(outs[i].shape)
        err = np.abs(got - outs[i]).max() / np.abs(outs[i]).max()
        print("head %d: max abs err / max abs = %.4g" % (i, err))
        assert err < 0.05, (i, err)         # bound from measurement, DESIGN.md section 8


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
