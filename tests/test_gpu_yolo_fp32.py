"""The detector's fp32 parity mode (YOLO(precision="fp32")) on the H100: the split-bf16 implicit-GEMM conv and every layer of
YOLOv3 and tiny YOLOv3 on its own GPU input against float64 on the unrounded operands, end-to-end heads, detections against
the float32 decode of the float64 heads, frame -> angles against the CPU restatement of the reference's video loop, batch
invariance, graph replay, the fp32 max-pool bit for bit, and a bf16 detector next to an fp32 one.

Every conv output is held to |got - ref| <= 2^-14 * sum|x * w| + 2^-20 * |ref|: the fp32 accumulation of K ~ 1000 terms
(K * 2^-24 of the sum of |terms|, the bf16 tests' ACC_REL) plus the fp32 rounding of the result; the split drops at most about
3 * 2^-18 of each |product| (two split residuals and the Alo * Wlo term), which sits under the first term."""
import functools

import numpy as np
import pytest

import yolo_cases as YC
import yolo_oracle as O
import yolo_tiny_cases as TC
import yolo_tiny_oracle as TO
from test_gpu_yolo import _frame, _scale
from whenet_b200 import yolo_arch as Y

pytestmark = pytest.mark.gpu

ACC_REL = 2.0 ** -14
OUT_REL = 2.0 ** -20
# output convs: largest error over the largest |value|.  The bf16 tests hold 1e-5 on bf16 inputs, whose products are exact in
# fp32; here the inputs are fp32 and the split's ~2^-17 per product, summed over K = 256..1024 with cancellation, measured
# 1.4-1.7e-5 on the 52 x 52 head (DESIGN.md 8.3).  The per-element bound above is the derived one and holds everywhere.
HEAD_REL = 3e-5


def _yolo(tiny=False, **kw):
    import whenet_b200
    return whenet_b200.YOLO(None, anchors_path=TC.ANCHORS if tiny else None, precision=kw.pop("precision", "fp32"), **kw)


@pytest.fixture(scope="module")
def yolo32():
    m = _yolo(max_frames=4)
    assert m.precision == "fp32" and m._L.whenet_det_precision(m._h) == 0
    yield m
    m.close()


def _check(got, ref, scale, what):
    """Every element within the bound; returns the largest error as a share of it."""
    d = np.abs(got.astype(np.float64) - ref)
    bound = ACC_REL * scale + OUT_REL * np.abs(ref)
    ratio = float((d / bound).max())
    assert ratio <= 1.0, "%s: error %.3g of the bound (max |err| %.3g)" % (what, ratio, d.max())
    return ratio


# ----------------------------------------------------------------------------------------------- 1. debug conv vs float64
def _debug_case(m, rng, n, H, W, cin, c_up, cout, k, stride, mode):
    x = rng.standard_normal((n, H, W, cin - c_up)).astype(np.float32)
    up = rng.standard_normal((n, H // 2, W // 2, c_up)).astype(np.float32) if mode == "cat" else None
    r = rng.standard_normal((n, H // stride, W // stride, cout)).astype(np.float32) if mode == "res" else None
    w = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    leaky = mode != "f32"
    got = m.debug_conv(x, w, b, k, stride, leaky=leaky, resid=r, up=up)
    ref = O.conv_layer(x, w, b, k, stride, leaky=leaky, resid=r, up=up)
    ratio = _check(got, ref, _scale(x, w, k, stride, resid=r, up=up), (n, H, W, cin, c_up, cout, k, stride, mode))
    print("MEASURED fp32 debug conv %s: max |err| / bound %.3f" % ((n, H, W, cin, c_up, cout, k, stride, mode), ratio))


@pytest.mark.parametrize("k,stride", [(1, 1), (3, 1), (3, 2)])
@pytest.mark.parametrize("cout", [18, 32, 64, 1024])
@pytest.mark.parametrize("n", [1, 3])
def test_debug_conv_grid(yolo32, k, stride, cout, n):
    _debug_case(yolo32, np.random.default_rng(cout * 10 + k + n), n, 13, 13, 64, 0, cout, k, stride, "leaky" if cout != 18 else "f32")


@pytest.mark.parametrize("n", [1, 2])
def test_debug_conv_residual_and_concat(yolo32, n):
    rng = np.random.default_rng(7 + n)
    _debug_case(yolo32, rng, n, 14, 14, 128, 0, 128, 3, 1, "res")
    _debug_case(yolo32, rng, n, 14, 14, 256, 128, 64, 1, 1, "cat")


@pytest.mark.parametrize("case", YC.DEBUG_CONVS + TC.DEBUG_CONVS, ids=lambda c: "%s-n%d-%dx%d-%d-%d-%d-k%ds%d" % ((c[8],) + c[:8]))
def test_debug_conv_shapes(yolo32, case):
    n, H, W, cin, c_up, cout, k, stride, mode, _un = case
    _debug_case(yolo32, np.random.default_rng(H * 1000 + W + cout + n), n, H, W, cin, c_up, cout, k, stride, mode)


# ----------------------------------------------------------------------------------------------- 2, 3. every layer, heads
@functools.lru_cache(maxsize=None)
def _layers(tiny, seed=0):
    names, w = Y.random_weights(seed, tiny=tiny)
    return Y.map_weights(names, w, tiny=tiny)[0]


def _folded32(tiny):
    """BatchNorm folded in float64 and the kernel rounded to fp32, as whenet_det_load_weights does in fp32 (no bf16 rounding)."""
    return [(k.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)) for k, b in (Y.fold_bn(d) for d in _layers(tiny))]


def _run_model(tiny, size):
    m = _yolo(tiny, model_image_size=size, max_frames=1)
    rgb = _frame(*YC.FRAMES[size], seed=3)
    m.detect(rgb)
    T = Y.table(tiny)
    taps = [m.tap(i) for i in range(len(T))]
    pooled = {i: m.tap(100 + i) for i in Y.TINY_POOLED} if tiny else {}
    canvas = m.tap(-1).reshape(1, size[0], size[1], 3)
    m.close()
    hw = Y.out_hw(*size, tiny=tiny)
    outs = [t.reshape(1, hw[i][0], hw[i][1], Y.cout(L, 1)).astype(np.float64) for i, (t, L) in enumerate(zip(taps, T))]
    return tiny, size, rgb, outs, pooled, canvas


@pytest.fixture(scope="module", params=[(t, s) for t in (False, True) for s in YC.MODEL_SIZES],
                ids=lambda p: "%s-%dx%d" % (("tiny" if p[0] else "full",) + p[1]))
def run_model(request):
    return _run_model(*request.param)


def test_every_layer_tap_on_its_own_input(run_model):
    tiny, size, _rgb, outs, pooled, canvas = run_model
    folded = _folded32(tiny)
    image = canvas / np.float32(255.0)
    ratios, lin = [], []
    for i, L in enumerate(Y.table(tiny)):
        if tiny:
            x, up = TO.layer_inputs(i, outs, image)
            res = None
            if L.pool:      # the fp32 pool is exact: bit-identical to the max over the GPU's tap of the conv before it
                assert np.array_equal(pooled[i].reshape(x.shape), x), "pool before conv %d" % i
        else:
            x, up, res = O.layer_inputs(i, outs, image)
        w, b = folded[i]
        ref = O.conv_layer(x, w, b, L.k, L.stride, L.bn, res, up)
        ratios.append(_check(outs[i], ref, _scale(x, w, L.k, L.stride, res, up), "layer %d" % i))
        if not L.bn:
            lin.append(np.abs(outs[i] - ref).max() / np.abs(ref).max())
            assert lin[-1] <= HEAD_REL, i
    print("MEASURED fp32 %s %dx%d layers: max |err| / bound %.3f, output convs max rel %.2g"
          % (("tiny" if tiny else "full",) + size + (max(ratios), max(lin))))


def test_end_to_end_heads(run_model):
    tiny, size, rgb, outs, _pooled, canvas = run_model
    lb = O.letterbox(rgb, (size[1], size[0]))
    assert np.array_equal(lb, canvas[0].astype(np.uint8))
    ref = (TO if tiny else O).body_numpy(lb[None] / np.float32(255.0), _layers(tiny))
    errs = [np.abs(outs[i] - ref[i]).max() / np.abs(ref[i]).max() for i in Y.heads(tiny)]
    print("MEASURED fp32 %s %dx%d heads: max abs err / max abs = %s" % (("tiny" if tiny else "full",) + size + (", ".join("%.3g" % e for e in errs),)))
    assert max(errs) <= 1e-3, errs


# ----------------------------------------------------------------------------------------------- 4, 5. detections, frame -> angles
SCORE_MARGIN = 1e-3
IOU_MARGIN = 1e-3
BOUND_MARGIN = 0.05         # px: every enlarged slice bound this far from an integer (or from its clamp)
BOX_PX = 1.0               # px: the largest box error; measured 0.42 px on boxes up to ~700 px wide (DESIGN.md 8.3)
GAP_MARGIN = 1e-5           # score gap of two candidates that suppress one another: NMS meets them in the same order


def _set_objectness(m, frame_bgr, target=20):
    """Seeded weights with the objectness bias of every head anchor set to the value in -12..3 (steps of 0.5) whose detections
    on ``frame_bgr`` come closest to ``target`` boxes -> the layers loaded.  The output convs' objectness and class columns are
    scaled by 10 and 3 first: the seeded weights give every candidate nearly the same score, and a threshold can only sit
    clear of all of them once the scores spread."""
    layers = [dict(d) for d in _layers(False)]
    for i in Y.HEADS:
        k = np.array(layers[i]["kernel"])
        k[..., 4::6] *= 10
        k[..., 5::6] *= 3
        layers[i]["kernel"] = k

    def load(bias):
        for i in Y.HEADS:
            bb = np.zeros_like(layers[i]["bias"])
            bb[4::6] = bias
            layers[i]["bias"] = bb
        m.load_layers(layers)

    best = None
    for bias in np.arange(-12.0, 3.01, 0.5):
        load(bias)
        k = len(m.detect_frames(frame_bgr[None])[0][0])
        if best is None or abs(k - target) < abs(best[1] - target):
            best = (bias, k)
    load(best[0])
    return layers


def _margins(boxes, scores, thr, iou):
    """How far the yolo_eval decisions on (boxes, scores) sit from flipping: the smallest |score - threshold| over all
    candidates, and the smallest |IoU - iou threshold| and score gap over the pairs NMS compares (both candidates pass)."""
    s = scores[:, 0].astype(np.float64)
    score_m = float(np.abs(s - thr).min())
    idx = np.flatnonzero(s >= thr)
    iou_m, gap_m = np.inf, np.inf
    for a in range(len(idx)):
        for b in range(a + 1, len(idx)):
            v = float(O.iou_tf(boxes[idx[a]], boxes[idx[b]]))
            iou_m = min(iou_m, abs(v - iou))
            if v > iou:
                gap_m = min(gap_m, abs(s[idx[a]] - s[idx[b]]))
    return score_m, iou_m, gap_m


def _bound_margin(box, H, W):
    """enlarge_bounds (demo_video.py:15-19) with the distance of every bound from an integer, or from the clamp it crosses."""
    y_min, x_min, y_max, x_max = [np.float32(v) for v in box]
    out = []

    def frac(t):
        t = float(t)
        return min(t - np.floor(t), np.ceil(t) - t)
    t = y_min - abs(y_min - y_max) / 10
    out.append(-float(t) if t < 0 else frac(t)); y_min = max(0, t)
    t = y_max + abs(y_min - y_max) / 10
    out.append(float(t) - H if t > H else frac(t)); y_max = min(H, t)
    t = x_min - abs(x_min - x_max) / 5
    out.append(-float(t) if t < 0 else frac(t)); x_min = max(0, t)
    t = x_max + abs(x_min - x_max) / 5
    out.append(float(t) - W if t > W else frac(t))
    return min(out)


def _gap_threshold(values, lo, hi):
    """The midpoint of the widest gap between the sorted ``values`` (and lo, hi) inside [lo, hi]: the threshold in that range
    that is farthest from every value."""
    v = np.sort(np.concatenate([[lo, hi], values[(values > lo) & (values < hi)]]))
    j = int(np.argmax(np.diff(v)))
    return float(np.float32((v[j] + v[j + 1]) / 2))


def _pair_ious(boxes, scores, thr):
    idx = np.flatnonzero(scores[:, 0] >= thr)
    return np.array([float(O.iou_tf(boxes[a], boxes[b])) for i, a in enumerate(idx) for b in idx[i + 1:]])


def _pick_thresholds(boxes, scores, k_lo, k_hi):
    """Score and IoU thresholds in the widest gaps of one frame's scores and pair IoUs, such that NMS keeps about k_lo..k_hi
    boxes.  Greedy NMS keeps, at a higher score threshold, the prefix of what it keeps at a lower one, so the score threshold
    goes between the k_lo-th and the (k_hi + 1)-th box kept at 0.2."""
    idx = np.flatnonzero(scores[:, 0] >= 0.2)
    ks = np.sort(scores[idx[O.nms_tf(boxes[idx], scores[idx, 0], k_hi + 1, 0.45)], 0])[::-1]
    if len(ks) < k_lo:
        return 0.2, 0.45
    thr = _gap_threshold(scores[:, 0], float(ks[k_hi]) if len(ks) > k_hi else 0.2, float(ks[k_lo - 1]))
    return thr, _gap_threshold(_pair_ious(boxes, scores, thr), 0.3, 0.6)


@pytest.fixture(scope="module")
def det():
    """An fp32 detector at 416 x 416 with seeded weights whose objectness bias gives about 20 boxes on an 832 x 832 frame."""
    m = _yolo(max_frames=3, score=0.3, iou=0.45)
    layers = _set_objectness(m, np.ascontiguousarray(_frame(832, 832, seed=0)[:, :, ::-1]))
    yield m, layers
    m.close()


def _scene(det, k_lo, k_hi, bounds):
    """The first square 832 x 832 frame (the letterbox fills it: no box centre lies outside) whose detections, with the
    thresholds of _pick_thresholds, clear every margin on the GPU's heads (with some room) and then on the float64 heads; with
    ``bounds`` also the margin of every enlarged slice bound.  Sets the detector's thresholds -> (frame, oracle detections)."""
    m, layers = det
    for seed in range(30):              # pick on the GPU's heads, then confirm on the oracle's
        frame = _frame(832, 832, seed=seed)
        m.detect_frames(frame[None])
        heads = [m.tap(i).reshape(13 << l, 13 << l, 18) for l, i in enumerate(Y.HEADS)]
        boxes, scores = O.decode(heads, m.anchors, 1, 832, 832)
        thr, iou = _pick_thresholds(boxes, scores, k_lo, k_hi)
        sm, im, gm = _margins(boxes, scores, thr, iou)
        kept = O.yolo_eval(boxes, scores, thr, iou)[0]
        bm = min(_bound_margin(b, 832, 832) for b in kept) if len(kept) else 0.0
        if len(kept) >= k_lo and sm >= SCORE_MARGIN + 1e-4 and im >= IOU_MARGIN + 1e-4 and gm >= 2 * GAP_MARGIN and \
                (not bounds or bm >= BOUND_MARGIN + 5e-3):
            break
    else:
        pytest.fail("no seed gives a frame whose detections clear the margins")
    m.score, m.iou = thr, iou
    lb = O.letterbox(np.ascontiguousarray(frame[:, :, ::-1]), (416, 416))
    outs = O.body_numpy(lb[None] / np.float32(255.0), layers)
    boxes, scores = O.decode([outs[i][0].astype(np.float32) for i in Y.HEADS], m.anchors, 1, 832, 832)
    sm, im, gm = _margins(boxes, scores, thr, iou)
    ref = O.yolo_eval(boxes, scores, thr, iou)
    bm = min(_bound_margin(b, 832, 832) for b in ref[0])
    print("MEASURED scene seed %d, score threshold %.4f, IoU threshold %.4f: %d boxes; float64 margins: score %.3g, IoU %.3g, "
          "score gap of suppressing pairs %.3g, slice bounds %.3g px" % (seed, thr, iou, len(ref[0]), sm, im, gm, bm))
    assert sm >= SCORE_MARGIN and im >= IOU_MARGIN and gm >= GAP_MARGIN and (not bounds or bm >= BOUND_MARGIN), (sm, im, gm, bm)
    return frame, ref


def test_detections_equal_float64_heads(det):
    m, _layers_ = det
    frame, (rb, rs, rc, _idx) = _scene(det, 15, 20, bounds=False)
    gb, gs, gc = m.detect_frames(frame[None])[0]
    assert len(gb) == len(rb) >= 15 and np.array_equal(gc, rc)
    err = np.abs(gb.astype(np.float64) - rb).max()
    print("MEASURED fp32 detections: %d boxes, max box error %.3g px, max score error %.3g" % (len(gb), err, np.abs(gs - rs).max()))
    assert err <= BOX_PX, err


def test_frame_to_angles_equal_the_reference_restatement(det, oracle64):
    """pipeline.detect_and_estimate with both networks in fp32 against reference demo_video.py:13-27 on the CPU: oracle
    boxes -> enlarge_box -> cv2 slice, BGR -> RGB, resize -> float64 WHENet."""
    cv2 = pytest.importorskip("cv2")
    import whenet_b200
    from whenet_b200 import crops
    m, layers = det
    frame, (rb, _rs, _rc, _idx) = _scene(det, 3, 6, bounds=True)
    H, W = frame.shape[:2]
    rects = [crops.enlarge_box(b, H, W) for b in rb]
    ref_crops = np.stack([cv2.resize(cv2.cvtColor(frame[y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224)) for y0, y1, x0, x1 in rects])
    ref = np.stack(oracle64.get_angle(ref_crops), 1)
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="fp32", max_batch=32)
    try:
        boxes, _scores, angles = whenet_b200.pipeline.detect_and_estimate(m, wn, frame)
        assert [crops.enlarge_box(b, H, W) for b in boxes] == rects
        d = np.abs(angles.astype(np.float64) - ref).max()
        print("MEASURED fp32 detector + fp32 WHENet: %d heads, max |angle - reference| %.4f deg" % (len(boxes), d))
        assert d <= 0.01, d
        bf = _yolo(precision="bf16", max_frames=1, score=m.score, iou=m.iou)
        bf.load_layers(layers)
        b16, _s16, a16 = whenet_b200.pipeline.detect_and_estimate(bf, wn, frame)
        same = [crops.enlarge_box(b, H, W) for b in b16] == rects
        print("MEASURED bf16 detector + fp32 WHENet on the same frame: %d heads (%s slices as the reference)%s" % (
            len(b16), "the same" if same else "other", ", max |angle - reference| %.3f deg" % np.abs(a16 - ref).max() if len(b16) == len(rb) else ""))
        bf.close()
    finally:
        wn.close()


# ----------------------------------------------------------------------------------------------- 6. batch invariance, replay
def _run(m, frames):
    return m.detect_frames(frames), [m.tap(i) for i in Y.HEADS]


def _same(a, b):
    (ra, ha), (rb, hb) = a, b
    assert len(ra) == len(rb)
    for x, y in zip(ra, rb):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)
    for u, v in zip(ha, hb):
        assert np.array_equal(u, v)


def test_batch_invariance_graph_replay_and_device_frames(yolo32):
    import torch
    frames = np.stack([_frame(360, 640, seed=70 + s)[:, :, ::-1] for s in range(3)])
    yolo32.score = 0.2
    try:
        batch = _run(yolo32, frames)
        assert all(len(r[0]) for r in batch[0])
        _same(_run(yolo32, frames), batch)                                  # replay of the captured graph
        _same(_run(yolo32, torch.from_numpy(frames).cuda()), batch)         # device frames
        for f in range(3):
            single = _run(yolo32, frames[f:f + 1])
            _same(single, ([batch[0][f]], [h.reshape(3, -1)[f] for h in batch[1]]))
    finally:
        yolo32.score = 0.3


def test_detect_and_estimate_frames_equals_per_frame(yolo32):
    import whenet_b200
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="fp32", max_batch=32)
    yolo32.score = 0.26
    try:
        frames = np.stack([_frame(832, 832, seed=80 + s) for s in range(5)])
        ref = [whenet_b200.pipeline.detect_and_estimate(yolo32, wn, f) for f in frames]
        assert any(len(r[0]) for r in ref)
        got = whenet_b200.pipeline.detect_and_estimate_frames(yolo32, wn, frames)
        assert len(got) == len(ref)
        for g, r in zip(got, ref):
            for x, y in zip(g, r):
                assert x.dtype == y.dtype and np.array_equal(x, y)
    finally:
        yolo32.score = 0.3
        wn.close()


# ----------------------------------------------------------------------------------------------- 7. max-pool, 8. bf16 next to fp32
@pytest.mark.parametrize("case", TC.POOLS, ids=lambda c: "n%d-%dx%d-c%d-s%d" % c)
def test_debug_maxpool_is_bit_exact(yolo32, case):
    n, H, W, C, s = case
    x = (np.random.default_rng(H * 100 + W + C + s).standard_normal((n, H, W, C)) - 0.5).astype(np.float32)
    got = yolo32.debug_maxpool(x, s)
    ref = TO.maxpool_same(x, s)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_bf16_detector_after_an_fp32_one_is_unchanged():
    frames = np.stack([_frame(300, 400, seed=90 + s)[:, :, ::-1] for s in range(2)])
    alone = _yolo(precision="bf16", max_frames=2, score=0.2)
    assert alone.precision == "bf16" and alone._L.whenet_det_precision(alone._h) == 1
    ref = _run(alone, frames)
    alone.close()
    f32 = _yolo(max_frames=2, score=0.2)
    r32 = _run(f32, frames)
    after = _yolo(precision="bf16", max_frames=2, score=0.2)
    _same(_run(after, frames), ref)
    assert not all(np.array_equal(a, b) for a, b in zip(r32[1], ref[1]))
    after.close()
    f32.close()
