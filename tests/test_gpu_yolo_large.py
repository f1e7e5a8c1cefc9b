"""The head detector at model inputs above 608 (whenet_det_create_large, DESIGN.md 8.6) on the H100: letterbox canvases, the
decode + NMS route for more than 24,576 candidates against the float32 restatement and against the one-CTA kernel, every conv
on its own GPU input at sampled pixels against float64, the conv launch split into frame groups, the pipeline, and a clean
failure when the activations cannot fit; bf16 and the fp32 parity mode.  Device memory stays under about 8 GB (YOLOv3 bf16 at
2176 x 3840, two frames)."""
import numpy as np
import pytest

import yolo_cases as YC
import yolo_oracle as O
import yolo_tiny_cases as TC
import yolo_tiny_oracle as TO
from test_gpu_yolo import ACC_REL, _blank, _cand, _decode_exact, _f32_next, _frame, _put, _sparse_heads, _ulp_bf16
from test_gpu_yolo_fp32 import HEAD_REL, OUT_REL
from whenet_b200 import yolo_arch as Y

pytestmark = pytest.mark.gpu

FHD, UHD = (1088, 1920), (2176, 3840)


def _yolo(size, **kw):
    import whenet_b200
    return whenet_b200.YOLO(None, model_image_size=size, **kw)


# ----------------------------------------------------------------------------------------------- letterbox
@pytest.mark.parametrize("size,frames", [(FHD, [(1080, 1920), (720, 1280), (2160, 3840)]), ((1056, 1920), [(1080, 1920)]),
                                         (UHD, [(2160, 3840)])], ids=str)
def test_letterbox_canvases_bit_exact(size, frames):
    import torch
    m = _yolo(size, max_frames=len(frames))
    imgs = [_frame(h, w, seed=h + w) for h, w in frames]
    refs = [O.letterbox(im, (size[1], size[0])) for im in imgs]
    if size == (1056, 1920):        # the reference's image-sized mode on 1080p: (1080 - 1080 % 32, 1920 - 1920 % 32)
        assert size == (1080 - 1080 % 32, 1920 - 1920 % 32)
        assert np.array_equal(YC.pil_letterbox(imgs[0], (1920, 1056)), refs[0])
    for im, ref in zip(imgs, refs):
        m.detect(im)
        assert np.array_equal(m.tap(-1).reshape(ref.shape), ref)
        m.detect_frames(im[None, :, :, ::-1].copy())                                      # host BGR
        assert np.array_equal(m.tap(-1).reshape(ref.shape), ref)
        m.detect_frames(torch.from_numpy(im[None, :, :, ::-1].copy()).cuda())             # device BGR
        assert np.array_equal(m.tap(-1).reshape(ref.shape), ref)
    if len(frames) > 1:
        bgr = [np.ascontiguousarray(im[:, :, ::-1]) for im in imgs]
        for fr in (bgr, [torch.from_numpy(b).cuda() for b in bgr]):                      # ragged, host and device
            m.detect_frames(fr)
            canv = m.tap(-1).reshape((len(frames),) + refs[0].shape)
            for c, ref in zip(canv, refs):
                assert np.array_equal(c, ref)
    m.close()


# ----------------------------------------------------------------------------------------------- decode + NMS, second route
def _blank_c(n, size, classes=1, tiny=False):
    """_blank for any class count and network: every candidate scores 0 with a zero-area box."""
    hs = []
    for l in range(2 if tiny else 3):
        h = np.zeros((n, size[0] // 32 << l, size[1] // 32 << l, 3, 5 + classes), np.float32)
        h[..., 2:] = -200
        hs.append(h)
    return hs


@pytest.fixture(scope="module", params=[FHD, UHD], ids=lambda s: "%dx%d" % s)
def big(request):
    m = _yolo(request.param, max_frames=2)
    yield m
    m.close()


def test_large_route_exact_cases(big):
    """The exact-logit cases of test_gpu_yolo.py at 1088 x 1920 and 2176 x 3840, far past the one-CTA kernel's capacity."""
    size = big.model_image_size
    nc = Y.num_candidates(*size)
    assert nc > 24576
    big.score, big.iou = 0.25, 0.45
    hs = _blank(1, size)                                # threshold inclusive
    _put(hs, nc - 1, 0.25, size=size)
    assert _decode_exact(big, hs) == [[nc - 1]]
    big.score = _f32_next(0.25, 1)
    assert _decode_exact(big, hs) == [[]]
    # equal scores across words, warps, threads' strides and heads: lower index first
    hs = _blank(1, size)
    ties = [3, 35, 3 + 1024 * 32, 31, 32, nc // 2, nc - 1, 3 * (size[0] // 32) * (size[1] // 32) + 5]
    for i in ties:
        _put(hs, i, 0.5, twh=(-200, -200), size=size)
    for i in (nc - 2, 50):
        _put(hs, i, 1.0, twh=(-200, -200), size=size)
    big.score, big.iou = 0.25, 0.45
    assert _decode_exact(big, hs) == [[50, nc - 2] + sorted(ties)]
    # IoU == threshold does not suppress, the next float below does
    hs = _blank(1, size)
    gw = size[1] // 32
    i, j = 3 * (5 * gw + 5), 3 * (5 * gw + 6)
    _put(hs, i, 1.0, size=size)
    _put(hs, j, 0.5, size=size)
    with np.errstate(over="ignore"):
        boxes, _ = O.decode([h[0].reshape(h.shape[1:3] + (-1,)) for h in hs], big.anchors, 1, 1080, 1920)
    thr = O.iou_tf(boxes[i], boxes[j])
    big.iou = float(thr)
    assert _decode_exact(big, hs, 1080, 1920) == [[i, j]]
    big.iou = _f32_next(thr, 0)
    assert _decode_exact(big, hs, 1080, 1920) == [[i]]
    # NaN IoU suppresses nothing: two boxes of (-inf, -inf, inf, inf)
    hs = _blank(1, size)
    for y, x in ((2, 3), (9, 7)):
        hs[0][0, y, x, 0, 2:4] = 100
        hs[0][0, y, x, 0, 4:6] = 200
    big.score, big.iou = 0.3, 0.45
    assert len(_decode_exact(big, hs)[0]) == 2


@pytest.mark.parametrize("max_boxes", [1, 20, 256])
def test_large_route_max_boxes(big, max_boxes):
    size = big.model_image_size
    hs = _blank(2, size)
    cands = list(range(7, Y.num_candidates(*size), 1601))[:300]
    for f in range(2):
        for i in cands:
            _put(hs, i, 0.5, twh=(-200, -200), f=f, size=size)
    big.score, big.iou = 0.25, 0.45
    assert _decode_exact(big, hs, max_boxes=max_boxes) == [cands[:max_boxes]] * 2


def test_large_route_every_candidate_passes(big):
    """Threshold 0 with every score 0: every alive bit is set, and the 256 lowest indices are kept."""
    size = big.model_image_size
    big.score, big.iou = 0.0, 0.45
    assert _decode_exact(big, _blank(1, size), max_boxes=256) == [list(range(256))]


def test_large_route_sparse_frames(big):
    size = big.model_image_size
    big.score, big.iou = 0.25, 0.45
    kept = _decode_exact(big, _sparse_heads(np.random.default_rng(size[0]), 2, size, k=400), 1080, 1920)
    assert all(kept) and kept[0] != kept[1]


def test_large_route_random_heads(big):
    """Random logits: the same kept candidates in the same order as the float32 restatement.  The device returns boxes, so
    each kept box is matched to the nearest candidate box of the restatement."""
    size = big.model_image_size
    rng = np.random.default_rng(11)
    flat = [rng.normal(0, 2, (1, size[0] // 32 << l, size[1] // 32 << l, 18)).astype(np.float32) for l in range(3)]
    big.score, big.iou = 0.5, 0.3
    gb, gs, gc = big.debug_decode(flat, 1080, 1920, 100)[0]
    boxes, scores = O.decode([h[0] for h in flat], big.anchors, 1, 1080, 1920)
    rb, rs, rc, idx = O.yolo_eval(boxes, scores, big.score, big.iou, 100)
    assert len(gb) == len(rb) == 100
    got_idx = [int(np.argmin(np.abs(boxes - b).sum(1))) for b in gb]
    assert got_idx == idx.tolist()
    assert np.allclose(gb, rb, rtol=1e-5, atol=1e-3) and np.allclose(gs, rs, rtol=1e-6)


@pytest.mark.parametrize("classes,tiny", [(2, False), (80, False), (1, True), (2, True)])
def test_large_route_classes_and_tiny(classes, tiny):
    """Per-class NMS CTAs and the class-by-class pack: 2 and 80 classes, and tiny YOLOv3 (two heads) at 1088 x 1920."""
    m = _yolo(FHD, max_frames=1, **({"anchors_path": TC.ANCHORS} if tiny else {}))
    names, w = Y.random_weights(0, classes, tiny=tiny)
    m.load_layers(Y.map_weights(names, w, tiny=tiny)[0])
    m.score, m.iou = 0.25, 0.45
    nc = Y.num_candidates(*FHD, tiny=tiny)
    assert nc > 24576
    hs = _blank_c(1, FHD, classes, tiny)
    rng = np.random.default_rng(classes)
    picks = rng.choice(nc, 200, replace=False)
    for i in picks:
        l, y, x, a = _cand(FHD, int(i))
        t = hs[l][0, y, x, a]
        t[2:4] = (-200, -200)
        t[4] = 200
        t[5:] = -200
        t[5 + int(rng.integers(classes))] = [200, 0][int(rng.integers(2))]
    flat = [np.ascontiguousarray(h.reshape(h.shape[:3] + (-1,))) for h in hs]
    gb, gs, gc = m.debug_decode(flat, 1080, 1920, 64)[0]
    boxes, scores = (TO if tiny else O).decode([h[0] for h in flat], m.anchors, classes, 1080, 1920)
    rb, rs, rc, _ = O.yolo_eval(boxes, scores, m.score, m.iou, 64)
    assert len(gb) > 0 and np.array_equal(gb, rb) and np.array_equal(gs, rs) and np.array_equal(gc, rc)
    m.close()


@pytest.mark.parametrize("size", [(416, 416), (608, 608)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("n", [1, 8])
def test_forced_large_route_equals_one_cta_kernel(size, n):
    """Where both routes run, the second one gives the one-CTA kernel's outputs bit for bit."""
    m = _yolo(size, max_frames=8)
    rng = np.random.default_rng(n + size[0])
    flat = [rng.normal(0, 2, (n, size[0] // 32 << l, size[1] // 32 << l, 18)).astype(np.float32) for l in range(3)]
    for score, iou, mb in ((0.3, 0.45, 20), (0.0, 0.45, 256), (0.6, 0.1, 1)):
        m.score, m.iou = score, iou
        a = m.debug_decode(flat, 720, 1280, mb)
        m.debug_force_large_decode(True)
        b = m.debug_decode(flat, 720, 1280, mb)
        m.debug_force_large_decode(False)
        for x, y in zip(a, b):
            assert len(x[0]) > 0
            for u, v in zip(x, y):
                assert np.array_equal(u, v)
    m.close()


# ----------------------------------------------------------------------------------------------- convs on their own GPU input
def _samples(n, H, W, rng, k_random=1500):
    """(f, y, x) output pixels: every border (every 5th pixel), both sides of each 128-row tile that straddles frames, the last
    pixel of the last frame, random pixels."""
    pts = set()
    for f in range(n):
        for x in range(0, W, 5):
            pts |= {(f, 0, x), (f, H - 1, x)}
        for y in range(0, H, 5):
            pts |= {(f, y, 0), (f, y, W - 1)}
    hw = H * W
    for f in range(1, n):
        m = f * hw
        if m % 128:
            for q in (m - 1, m):                        # the pixels on both sides of the frame edge inside one tile
                pts.add((q // hw, q % hw // W, q % W))
    pts.add((n - 1, H - 1, W - 1))
    for _ in range(k_random):
        pts.add((int(rng.integers(n)), int(rng.integers(H)), int(rng.integers(W))))
    return np.array(sorted(pts))


def _conv_at(x, w, k, stride, pts):
    """The conv's sum at output pixels pts in float64 (padding as O.conv_layer), and the same of |x| and |w|."""
    f, y, xx = pts[:, 0], pts[:, 1], pts[:, 2]
    pad_after = 1 if stride == 1 and k == 3 else 0
    xp = np.pad(x, ((0, 0), (k // 2, pad_after), (k // 2, pad_after), (0, 0))) if k == 3 else x
    acc = np.zeros((len(pts), w.shape[3]))
    sc = np.zeros_like(acc)
    for ky in range(k):
        for kx in range(k):
            p = xp[f, y * stride + ky, xx * stride + kx].astype(np.float64)
            acc += p @ w[ky, kx]
            sc += np.abs(p) @ np.abs(w[ky, kx])
    return acc, sc


def _check_convs_sampled(m, tiny, n, classes, what):
    """Every conv of detector m's last call at sampled output pixels against float64 on the GPU's own input.  bf16: 8's bound,
    2 bf16 ulp plus the fp32 accumulation error; fp32: 8.3's, 2^-14 of the sum of |terms| plus 2^-20 of |ref|.  The output convs:
    1e-5 (fp32: 3e-5) of the largest value.  Taps are dropped after their last use, so that 2176 x 3840 fits in host memory."""
    T = Y.table(tiny)
    f32 = m.precision == "fp32"
    size = m.model_image_size
    outs_hw = Y.out_hw(*size, tiny)
    ins_hw = Y.in_hw(*size, tiny)
    names, w = Y.random_weights(0, classes, tiny=tiny)
    layers, _ = Y.map_weights(names, w, tiny=tiny)
    if f32:     # as whenet_det_load_weights folds in fp32: kernel and bias rounded to fp32, no bf16 rounding
        folded = [(k.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)) for k, b in (Y.fold_bn(d) for d in layers)]
    else:
        folded = [(Y.bf16_round(k).astype(np.float64), b) for k, b in (Y.fold_bn(d) for d in layers)]
    canvas = m.tap(-1).reshape(n, size[0], size[1], 3) / np.float32(255.0)
    last_use = {}
    for i, L in enumerate(T):
        for j in ([] if L.pool or L.src < 0 else [L.src]) + [v for v in (L.res, L.up) if v is not None]:
            last_use[j] = i
    taps = {}
    rng = np.random.default_rng(5)
    worst = 0.0
    for i, L in enumerate(T):
        co = Y.cout(L, classes)
        out = m.tap(i).reshape(n, outs_hw[i][0], outs_hw[i][1], co)
        if L.pool:
            x = m.tap(100 + i).reshape(n, ins_hw[i][0], ins_hw[i][1], L.cin)      # the GPU's max-pool (exact, tested apart)
        else:
            x = canvas if L.src < 0 else taps[L.src]
        if L.up is not None:
            u = taps[L.up].repeat(2, axis=1).repeat(2, axis=2)
            x = np.concatenate([u, x], axis=3)
        pts = _samples(n, out.shape[1], out.shape[2], rng)
        wk, b = folded[i]
        acc, sc = _conv_at(x, wk, L.k, L.stride, pts)
        del x
        got = out[pts[:, 0], pts[:, 1], pts[:, 2]].astype(np.float64)
        ref = acc + b
        if L.bn:
            ref = np.where(ref > 0, ref, 0.1 * ref)
            if L.res is not None:
                r = taps[L.res][pts[:, 0], pts[:, 1], pts[:, 2]].astype(np.float64)
                ref = ref + r
                sc = sc + np.abs(r)
            d = np.abs(got - ref)
            if f32:
                bound = ACC_REL * sc + OUT_REL * np.abs(ref)
                assert (d <= bound).all(), (what, i, float((d / bound).max()))
            else:
                # the 99.9 %-within-1-ulp share of the full-tap tests is loosened to 99.5 % for a few thousand samples
                bound = 2.0 * _ulp_bf16(ref) + ACC_REL * sc
                share = float(np.mean(d <= _ulp_bf16(ref)))
                assert (d <= bound).all() and share >= 0.995, (what, i, share, float((d / bound).max()))
            worst = max(worst, float((d / bound).max()))
        else:
            assert np.abs(got - ref).max() <= (HEAD_REL if f32 else 1e-5) * np.abs(ref).max(), (what, i)
        if last_use.get(i, -1) > i:
            taps[i] = out
        for j in [j for j in taps if last_use[j] <= i]:
            del taps[j]
    print("MEASURED %s: %d convs at sampled pixels, max |err| / bound %.3f" % (what, len(T), worst))


# (tiny, classes, h, w, precision): together they run every tile configuration either planner picks above 608
# (test_yolo_large_cpu.GPU_CONV_RUNS holds the same list)
CONV_RUNS = [(False, 1, 1088, 1920, "bf16"), (False, 80, 1088, 1920, "bf16"), (False, 1, 2176, 3840, "bf16"),
             (True, 1, 1088, 1920, "bf16"), (True, 80, 1088, 1920, "bf16"), (True, 80, 2176, 3840, "bf16"), (True, 1, 4096, 4096, "bf16"),
             (False, 80, 1088, 1920, "fp32"), (True, 1, 1088, 1920, "fp32"), (True, 80, 2176, 3840, "fp32"), (True, 1, 4096, 4096, "fp32")]


@pytest.mark.parametrize("tiny,classes,h,w,precision", CONV_RUNS, ids=str)
def test_every_conv_on_its_own_input(tiny, classes, h, w, precision):
    """Tiny bf16 at 1088 x 1920 runs two frames, which puts a 128-row tile across the frame edge in every conv whose Ho * Wo
    is not a multiple of 128."""
    n = 2 if (tiny, classes, h, precision) == (True, 1, 1088, "bf16") else 1
    m = _yolo((h, w), max_frames=n, score=0.3, precision=precision, **({"anchors_path": TC.ANCHORS} if tiny else {}))
    if classes > 1:
        names, wt = Y.random_weights(0, classes, tiny=tiny)
        m.load_layers(Y.map_weights(names, wt, tiny=tiny)[0])
    frames = np.stack([_frame(1080, 1920, seed=s)[:, :, ::-1] for s in range(n)])
    m.detect_frames(np.ascontiguousarray(frames))
    _check_convs_sampled(m, tiny, n, classes, "%s %s %dx%d n=%d classes=%d" % ("tiny" if tiny else "yolov3", precision, h, w, n, classes))
    m.close()


@pytest.mark.parametrize("precision,bound", [("bf16", 0.05), ("fp32", 1e-3)])
def test_end_to_end_heads_within_bound_at_640(precision, bound):
    """640 x 640 (25,200 candidates: the second decode route) against the float64 body, within 8's 5 % head bound (fp32:
    8.3's 1e-3)."""
    m = _yolo((640, 640), max_frames=1, precision=precision)
    rgb = _frame(720, 1280, seed=3)
    m.detect(rgb)
    lb = O.letterbox(rgb, (640, 640))
    assert np.array_equal(m.tap(-1).reshape(640, 640, 3), lb)
    names, w = Y.random_weights(0)
    layers, _ = Y.map_weights(names, w)
    outs = O.body_numpy(lb[None] / np.float32(255.0), layers)
    errs = [np.abs(m.tap(i).reshape(outs[i].shape) - outs[i]).max() / np.abs(outs[i]).max() for i in Y.HEADS]
    print("MEASURED %s 640x640 heads: max abs err / max abs = %s" % (precision, ", ".join("%.4g" % e for e in errs)))
    assert max(errs) < bound
    m.close()


# ----------------------------------------------------------------------------------------------- conv launch split
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_tiny_17_frames_split_into_frame_groups(precision):
    """Tiny YOLOv3 at 1088 x 1920 with 17 frames in one call: conv 1 needs 69,360 M tiles, more than gridDim.y holds, so
    launch_igemm (fp32: launch_igemm32) runs it as groups of 16 and 1 frames.  Every frame's boxes, scores and conv taps equal
    that frame run alone."""
    m = _yolo(FHD, max_frames=17, score=0.0, anchors_path=TC.ANCHORS, precision=precision)   # threshold 0: 20 boxes per frame
    hw = Y.out_hw(*FHD, tiny=True)[1]
    assert -(-17 * hw[0] * hw[1] // 128) == 69360
    frames = np.stack([_frame(1080, 1920, seed=s)[:, :, ::-1] for s in range(17)])
    frames = np.ascontiguousarray(frames)
    res = m.detect_frames(frames)
    per = [m.tap(i).reshape(17, -1) for i in range(Y.TINY_N_CONV)]
    for f in (0, 7, 15, 16):
        alone = m.detect_frames(frames[f:f + 1])[0]
        for u, v in zip(res[f], alone):
            assert np.array_equal(u, v), f
        for i in range(Y.TINY_N_CONV):
            assert np.array_equal(per[i][f], m.tap(i)), (f, i)
    assert all(len(r[0]) == 20 for r in res)
    m.close()


# ----------------------------------------------------------------------------------------------- pipeline
def test_pipeline_frames_at_1088x1920():
    import torch
    import whenet_b200
    from whenet_b200 import pipeline
    m = _yolo(FHD, max_frames=4, score=0.2, max_boxes=40)
    wh = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=64)
    frames = np.stack([_frame(1080, 1920, seed=s)[:, :, ::-1] for s in range(3)])
    frames = np.ascontiguousarray(frames)
    got = pipeline.detect_and_estimate_frames(m, wh, frames)
    assert max(len(g[0]) for g in got) > 20                        # max_boxes above the reference's 20
    for f in range(3):
        one = pipeline.detect_and_estimate(m, wh, frames[f])                   # boxes in frame pixels, every slice valid
        for u, v in zip(got[f], one):
            assert np.array_equal(u, v, equal_nan=True)
    dev = pipeline.detect_and_estimate_frames(m, wh, torch.from_numpy(frames).cuda())
    ragged = pipeline.detect_and_estimate_frames(m, wh, [frames[0], np.ascontiguousarray(frames[1, :720, :1280])])
    for u, v in zip(got[0], dev[0]):
        assert np.array_equal(u, v, equal_nan=True)
    for u, v in zip(got[0], ragged[0]):
        assert np.array_equal(u, v, equal_nan=True)
    m.close()


# ----------------------------------------------------------------------------------------------- memory
def _bytes_per_frame(tiny, h, w, classes, f32):
    """What whenet_det_load_weights allocates per frame (conv outputs, pooled inputs, boxes, class scores) plus the canvas"""
    b = 0
    for L, (ih, iw), (oh, ow) in zip(Y.table(tiny), Y.in_hw(h, w, tiny), Y.out_hw(h, w, tiny)):
        b += oh * ow * Y.cout(L, classes) * (4 if L.head is not None or f32 else 2)
        if L.pool:
            b += ih * iw * L.cin * (4 if f32 else 2)
    nc = Y.num_candidates(h, w, tiny)
    return b + nc * 16 + classes * nc * 4 + h * w * 3


def test_over_large_detector_fails_cleanly():
    """A detector larger than the device is refused before its first large buffer, naming the bytes: fp32 at 4096 x 4096 with
    64 frames at create (even tiny YOLOv3 with one class needs 187 GB), YOLOv3 fp32 at 4096 x 4096 with 8 frames when the weights
    are loaded (120 GB; only the 400 MB of canvases exist by then, and they are freed).  A detector made afterwards works."""
    import whenet_b200
    from whenet_b200._lib import WhenetError
    least = 64 * _bytes_per_frame(True, 4096, 4096, 1, True)
    assert least > 80e9
    with pytest.raises(WhenetError, match="needs %d bytes" % least) as e:
        whenet_b200.YOLO(None, model_image_size=(4096, 4096), max_frames=64, precision="fp32")
    assert e.value.code == -2
    with pytest.raises(WhenetError, match="this network at this size") as e:
        whenet_b200.YOLO(None, model_image_size=(4096, 4096), max_frames=8, precision="fp32")
    assert e.value.code == -2 and 8 * _bytes_per_frame(False, 4096, 4096, 1, True) > 80e9
    m = _yolo((640, 640), max_frames=1, score=0.2)
    assert len(m.detect(_frame(480, 640, seed=1))[0]) > 0
    m.close()
