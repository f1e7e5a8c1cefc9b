"""GPU head overlay (``overlay.draw_heads``, DESIGN.md section 8.7): frames drawn on the device equal, bit for bit, the same
frames drawn on the host with oracle/overlay_oracle's cv2 calls on float32 boxes and angles."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))

pytestmark = pytest.mark.gpu


def _ref_draw(img, box, ang):
    """What process_detection_ref draws for one head on img (in place), or nothing where the reference raises."""
    import overlay_oracle as O
    y_min, x_min, y_max, x_max = (np.float32(v) for v in box)
    y_min = max(0, y_min - abs(y_min - y_max) / 10)
    y_max = min(img.shape[0], y_max + abs(y_min - y_max) / 10)
    x_min = max(0, x_min - abs(x_min - x_max) / 5)
    x_max = min(img.shape[1], x_max + abs(x_min - x_max) / 5)
    x_max = min(x_max, img.shape[1])
    if not (int(y_min) < int(y_max) and int(x_min) < int(x_max)):
        return False        # the slice enlarge_box refuses (the pipeline gives such a head NaN angles)
    tmp = img.copy()
    try:
        with np.errstate(over="ignore", invalid="ignore"):
            import cv2
            cv2.rectangle(tmp, (int(x_min), int(y_min)), (int(x_max), int(y_max)), (0, 0, 0), 2)
            O.draw_axis_ref(tmp, np.float32(ang[0]), np.float32(ang[1]), np.float32(ang[2]), tdx=(x_min + x_max) / 2,
                            tdy=(y_min + y_max) / 2, size=abs(x_max - x_min) // 2)
    except (ValueError, OverflowError):
        return False
    img[:] = tmp
    return True


def _heads(rng, H, W, k):
    """k heads: random boxes partly off the frame, edge-touching, whole-frame and tiny ones; angles incl. NaN and inf."""
    boxes, angs = [], []
    for i in range(k):
        kind = i % 6
        if kind == 0:
            y0, x0 = rng.uniform(-0.2, 1.0) * H, rng.uniform(-0.2, 1.0) * W
            y1, x1 = y0 + rng.uniform(0, 0.5) * H, x0 + rng.uniform(0, 0.5) * W
        elif kind == 1:
            y0, x0, y1, x1 = 0.0, 0.0, float(H), float(W)
        elif kind == 2:
            y0, x0 = rng.uniform(0, H), rng.uniform(0, W)
            y1, x1 = y0 + rng.uniform(0, 3), x0 + rng.uniform(0, 3)
        elif kind == 3:
            y0, y1 = rng.uniform(0, H), float(H) - rng.uniform(0, 1)
            x0, x1 = float(W) * rng.uniform(0.5, 1), float(W) + rng.uniform(0, 5)
        else:
            y0, x0 = rng.uniform(0, H), rng.uniform(0, W)
            y1, x1 = y0 + rng.uniform(2, 0.3 * H + 3), x0 + rng.uniform(2, 0.3 * W + 3)
        boxes.append((y0, x0, y1, x1))
        a = rng.uniform(-180, 180, 3)
        if i % 17 == 5:
            a[i % 3] = np.nan
        if i % 23 == 7:
            a[i % 3] = np.inf
        if i % 29 == 11:
            a[i % 3] = 3e38
        angs.append(a)
    return np.array(boxes, np.float32).reshape(-1, 4), np.array(angs, np.float32).reshape(-1, 3)


def _results(rng, shapes, k):
    return [(b, np.ones(len(b), np.float32), a) for b, a in (_heads(rng, H, W, k) for H, W in shapes)]


def _host(frames, results):
    out = [f.copy() for f in frames]
    drawn = []
    for img, (b, _s, a) in zip(out, results):
        drawn.append(np.array([_ref_draw(img, b[i], a[i]) for i in range(len(b))], bool))
    return out, drawn


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


@pytest.mark.parametrize("H,W,n", [(1080, 1920, 8), (720, 1280, 1), (2160, 3840, 1), (417, 417, 64), (3, 5, 8), (1, 1, 8)])
def test_draw_heads_equals_host(wn, H, W, n):
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(H * 7 + W + n)
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    res = _results(rng, [(H, W)] * n, 20 if H * W > 100 else 6)
    ref, ref_drawn = _host(list(frames), res)
    dev = torch.from_numpy(frames).cuda()
    drawn = overlay.draw_heads(wn, dev, res)
    got = dev.cpu().numpy()
    for f in range(n):
        assert np.array_equal(drawn[f], ref_drawn[f]), f
        assert np.array_equal(got[f], ref[f]), (f, np.argwhere((got[f] != ref[f]).any(-1))[:5].tolist())
    # each frame drawn alone equals the same frame drawn in the batch
    for f in (0, n - 1):
        one = torch.from_numpy(frames[f:f + 1]).cuda()
        overlay.draw_heads(wn, one, res[f:f + 1])
        assert np.array_equal(one.cpu().numpy()[0], got[f])


def test_draw_heads_ragged(wn):
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(3)
    shapes = [(1080, 1920), (417, 417), (3, 5), (720, 1280), (1, 1), (2160, 3840)]
    frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in shapes]
    res = _results(rng, shapes, 20)
    ref, ref_drawn = _host(frames, res)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    drawn = overlay.draw_heads(wn, dev, res)
    for f in range(len(shapes)):
        assert np.array_equal(drawn[f], ref_drawn[f]), f
        assert np.array_equal(dev[f].cpu().numpy(), ref[f]), f


def test_draw_heads_overlap_order_and_untouched_pixels(wn):
    """Identical boxes with different angles: the later head's axes win; pixels off every primitive keep their value."""
    import torch
    from whenet_b200 import overlay
    H, W = 240, 320
    frame = np.full((1, H, W, 3), 77, np.uint8)
    b = np.array([[40, 60, 200, 260]] * 3, np.float32)
    a = np.array([[10, 20, 30], [-40, 5, 80], [170, -60, -10]], np.float32)
    res = [(b, np.ones(3, np.float32), a)]
    ref, _ = _host(list(frame), res)
    dev = torch.from_numpy(frame).cuda()
    overlay.draw_heads(wn, dev, res)
    got = dev.cpu().numpy()[0]
    assert np.array_equal(got, ref[0])
    assert ((got == 77).all(-1)).sum() > 0.9 * H * W


@pytest.mark.parametrize("kind", ["yolov3", "tiny"])
def test_detect_then_draw_end_to_end(wn, kind):
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline
    from test_gpu_yolo import _frame
    kw = {}
    if kind == "tiny":
        import yolo_tiny_cases as TC
        kw = {"anchors_path": TC.ANCHORS}
    yolo = whenet_b200.YOLO(None, max_frames=4, score=0.0, **kw)
    frames = np.stack([_frame(480, 640, seed=s) for s in range(3)])
    dev = torch.from_numpy(frames).cuda()
    res = pipeline.detect_and_estimate_frames(yolo, wn, dev)
    assert sum(len(r[0]) for r in res) > 0
    ref, _ = _host(list(frames), res)
    overlay.draw_heads(wn, dev, res)
    got = dev.cpu().numpy()
    for f in range(3):
        assert np.array_equal(got[f], ref[f]), f
    ragged = [_frame(480, 640, seed=5), _frame(360, 500, seed=6)]
    devr = [torch.from_numpy(f).cuda() for f in ragged]
    res = pipeline.detect_and_estimate_frames(yolo, wn, devr)
    ref, _ = _host(ragged, res)
    overlay.draw_heads(wn, devr, res)
    for f in range(2):
        assert np.array_equal(devr[f].cpu().numpy(), ref[f]), f
