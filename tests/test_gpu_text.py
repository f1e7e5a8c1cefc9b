"""GPU text (``overlay.draw_heads(display="full")`` and ``overlay.put_text``, DESIGN.md section 8.8): frames drawn on the
device equal, bit for bit, the same frames drawn on the host with process_detection_ref's cv2 calls on float32 boxes and
angles, labels included."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))

pytestmark = pytest.mark.gpu


def _ref_draw(img, box, ang):
    """What process_detection_ref draws for one head on img with display="full" (in place), or nothing where the reference
    raises."""
    import cv2
    import overlay_oracle as O
    y_min, x_min, y_max, x_max = (np.float32(v) for v in box)
    y_min = max(0, y_min - abs(y_min - y_max) / 10)
    y_max = min(img.shape[0], y_max + abs(y_min - y_max) / 10)
    x_min = max(0, x_min - abs(x_min - x_max) / 5)
    x_max = min(img.shape[1], x_max + abs(x_min - x_max) / 5)
    x_max = min(x_max, img.shape[1])
    if not (int(y_min) < int(y_max) and int(x_min) < int(x_max)):
        return False
    tmp = img.copy()
    yaw, pitch, roll = np.float32(ang[0]), np.float32(ang[1]), np.float32(ang[2])
    try:
        with np.errstate(over="ignore", invalid="ignore"):
            cv2.rectangle(tmp, (int(x_min), int(y_min)), (int(x_max), int(y_max)), (0, 0, 0), 2)
            O.draw_axis_ref(tmp, yaw, pitch, roll, tdx=(x_min + x_max) / 2, tdy=(y_min + y_max) / 2, size=abs(x_max - x_min) // 2)
    except (ValueError, OverflowError):
        return False
    cv2.putText(tmp, "yaw: {}".format(np.round(yaw)), (int(x_min), int(y_min)), cv2.FONT_HERSHEY_SIMPLEX, 0.4, (100, 255, 0), 1)
    cv2.putText(tmp, "pitch: {}".format(np.round(pitch)), (int(x_min), int(y_min) - 15), cv2.FONT_HERSHEY_SIMPLEX, 0.4, (100, 255, 0), 1)
    cv2.putText(tmp, "roll: {}".format(np.round(roll)), (int(x_min), int(y_min) - 30), cv2.FONT_HERSHEY_SIMPLEX, 0.4, (100, 255, 0), 1)
    img[:] = tmp
    return True


def _host(frames, results):
    out = [f.copy() for f in frames]
    drawn = []
    for img, (b, _s, a) in zip(out, results):
        drawn.append(np.array([_ref_draw(img, b[i], a[i]) for i in range(len(b))], bool))
    return out, drawn


def _results(rng, shapes, k):
    from test_gpu_draw import _heads
    return [(b, np.ones(len(b), np.float32), a) for b, a in (_heads(rng, H, W, k) for H, W in shapes)]


@pytest.fixture(scope="module")
def wn():
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


def _diff(a, b):
    return np.argwhere((a != b).any(-1))[:5].tolist()


@pytest.mark.parametrize("H,W,n", [(1080, 1920, 8), (720, 1280, 1), (2160, 3840, 1), (417, 417, 64), (3, 5, 8), (1, 1, 8)])
def test_draw_heads_full_equals_host(wn, H, W, n):
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(H * 7 + W + n + 1)
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    res = _results(rng, [(H, W)] * n, 20 if H * W > 100 else 6)
    ref, ref_drawn = _host(list(frames), res)
    dev = torch.from_numpy(frames).cuda()
    drawn = overlay.draw_heads(wn, dev, res, display="full")
    got = dev.cpu().numpy()
    for f in range(n):
        assert np.array_equal(drawn[f], ref_drawn[f]), f
        assert np.array_equal(got[f], ref[f]), (f, _diff(got[f], ref[f]))
    for f in (0, n - 1):        # each frame drawn alone equals the same frame drawn in the batch
        one = torch.from_numpy(frames[f:f + 1]).cuda()
        overlay.draw_heads(wn, one, res[f:f + 1], display="full")
        assert np.array_equal(one.cpu().numpy()[0], got[f])


def test_draw_heads_full_ragged(wn):
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(4)
    shapes = [(1080, 1920), (417, 417), (3, 5), (720, 1280), (1, 1), (2160, 3840)]
    frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in shapes]
    res = _results(rng, shapes, 20)
    ref, ref_drawn = _host(frames, res)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    drawn = overlay.draw_heads(wn, dev, res, display="full")
    for f in range(len(shapes)):
        assert np.array_equal(drawn[f], ref_drawn[f]), f
        assert np.array_equal(dev[f].cpu().numpy(), ref[f]), (f, _diff(dev[f].cpu().numpy(), ref[f]))


def test_labels_off_the_top_overlap_and_skipped_heads(wn):
    """Heads at the top edge (labels leave the frame), identical boxes (head i's labels over head i-1's axes), and NaN, inf
    and huge angles (skipped heads, or huge labels where the radian stays finite)."""
    import torch
    from whenet_b200 import overlay
    H, W = 240, 320
    frame = np.full((1, H, W, 3), 77, np.uint8)
    b = np.array([[2, 60, 120, 200], [40, 60, 200, 260], [40, 60, 200, 260], [40, 60, 200, 260], [10, 5, 60, 80],
                  [30, 100, 90, 160], [30, 100, 90, 160], [0, 0, 240, 320]], np.float32)
    a = np.array([[10, 20, 30], [-40, 5, 80], [170.5, -60.5, -0.4], [np.nan, 1, 2], [np.inf, 0, 0], [3e38, 0, 0],
                  [1e30, -2.5e20, 123456789], [-179.5, 179.5, 0.5]], np.float32)
    res = [(b, np.ones(len(b), np.float32), a)]
    ref, ref_drawn = _host(list(frame), res)
    assert ref_drawn[0][:3].all() and not ref_drawn[0][3:5].any()
    dev = torch.from_numpy(frame).cuda()
    drawn = overlay.draw_heads(wn, dev, res, display="full")
    got = dev.cpu().numpy()[0]
    assert np.array_equal(drawn[0], ref_drawn[0])
    assert np.array_equal(got, ref[0]), _diff(got, ref[0])
    assert (got == (100, 255, 0)).all(-1).sum() > 200


def test_simple_is_unchanged(wn):
    """display="simple" through the new entry equals whenet_draw_heads_u8 on the same inputs."""
    import torch
    from whenet_b200 import overlay
    from whenet_b200._lib import check
    from whenet_b200.whenet import _ptr
    rng = np.random.default_rng(9)
    n, H, W = 4, 480, 640
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    res = _results(rng, [(H, W)] * n, 20)
    a = torch.from_numpy(frames).cuda()
    overlay.draw_heads(wn, a, res)
    boxes = np.ascontiguousarray(np.concatenate([r[0] for r in res]), np.float32)
    angles = np.ascontiguousarray(np.concatenate([r[2] for r in res]), np.float32)
    fo = np.repeat(np.arange(n, dtype=np.int32), [len(r[0]) for r in res])
    b = torch.from_numpy(frames).cuda()
    c = torch.from_numpy(frames).cuda()
    L = wn._L
    torch.cuda.synchronize()
    check(L.whenet_draw_heads_u8(wn._h, _ptr(b), n, H, W, _ptr(boxes), _ptr(angles), _ptr(fo), len(fo), None))
    check(L.whenet_draw_heads_ex_u8(wn._h, _ptr(c), n, H, W, _ptr(boxes), _ptr(angles), _ptr(fo), len(fo), 0, None))
    wn.synchronize()
    assert torch.equal(a, b) and torch.equal(b, c)
    ref, _ = __import__("test_gpu_draw")._host(list(frames), res)
    assert np.array_equal(a.cpu().numpy(), np.stack(ref))


def test_put_text_every_character(wn):
    import cv2
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(5)
    H, W = 300, 1400
    frames = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    items = []
    chars = "".join(chr(c) for c in range(32, 127))
    for f, scale in enumerate((0.4, 1.0, 2.5)):
        step = max(1, int(95 * 25 * scale) // W + 1)
        for k in range(0, 95, 95 // step + 1):
            items.append((f, chars[k:k + 95 // step + 1], (int(rng.integers(-20, 20)), int(30 * scale) + 40 * (k // (95 // step + 1))),
                          scale, tuple(int(v) for v in rng.integers(0, 256, 3))))
    for _ in range(60):         # random strings, origins partly and fully outside, over each other
        f = int(rng.integers(0, 3))
        text = "".join(chr(int(c)) for c in rng.integers(32, 127, int(rng.integers(1, 41))))
        items.append((f, text, (int(rng.integers(-400, W + 50)), int(rng.integers(-60, H + 60))), float(rng.uniform(0.1, 8)),
                      tuple(int(v) for v in rng.integers(0, 256, 3))))
    ref = frames.copy()
    for f, text, org, scale, col in items:
        cv2.putText(ref[f], text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, col, 1)
    dev = torch.from_numpy(frames).cuda()
    overlay.put_text(wn, dev, items)
    got = dev.cpu().numpy()
    for f in range(3):
        assert np.array_equal(got[f], ref[f]), (f, _diff(got[f], ref[f]))
    ragged = [torch.from_numpy(frames[0].copy()).cuda(), torch.from_numpy(frames[1, :77, :301].copy()).cuda()]
    rref = [frames[0].copy(), frames[1, :77, :301].copy()]
    its = [(1, "ragged: " + chars, (-3, 20), 0.5, (1, 2, 3)), (0, chars, (5, 250), 0.4, (100, 255, 0))]
    for f, text, org, scale, col in its:
        cv2.putText(rref[f], text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, col, 1)
    overlay.put_text(wn, ragged, its)
    for f in range(2):
        assert np.array_equal(ragged[f].cpu().numpy(), rref[f]), f
    with pytest.raises(ValueError):
        overlay.put_text(wn, dev, [(0, "bold", (0, 0), 1.0, (0, 0, 0), 2)])


@pytest.mark.parametrize("kind", ["yolov3", "tiny"])
def test_detect_then_draw_full_end_to_end(wn, kind):
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
    overlay.draw_heads(wn, dev, res, display="full")
    got = dev.cpu().numpy()
    for f in range(3):
        assert np.array_equal(got[f], ref[f]), (f, _diff(got[f], ref[f]))


def test_buffers_grow_in_any_order():
    """On a fresh context: display="full" with one head, then "simple" with many more segments (its segment table grows),
    then "full" and put_text again; every frame equals the host reference."""
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import overlay
    m = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=8)
    try:
        rng = np.random.default_rng(21)
        H, W = 360, 640
        base = rng.integers(0, 256, (4, H, W, 3), dtype=np.uint8)
        one = [(np.array([[40, 60, 200, 260]], np.float32), np.ones(1, np.float32), np.array([[10, -20, 30]], np.float32))]
        many = _results(rng, [(H, W)] * 4, 40)
        full2 = _results(rng, [(H, W)] * 4, 30)
        steps = [("full", base[:1], one), ("simple", base, many), ("full", base, full2)]
        for display, frames, res in steps:
            dev = torch.from_numpy(frames.copy()).cuda()
            overlay.draw_heads(m, dev, res, display=display)
            ref = (_host if display == "full" else __import__("test_gpu_draw")._host)(list(frames), res)[0]
            got = dev.cpu().numpy()
            for f in range(len(frames)):
                assert np.array_equal(got[f], ref[f]), (display, f, _diff(got[f], ref[f]))
        items = [(f, "put_text %d after growth" % f, (5, 20 + 30 * f), 0.5 + f, (1, 2, 3)) for f in range(4)]
        ref = base.copy()
        for f, text, org, scale, col in items:
            cv2.putText(ref[f], text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, col, 1)
        dev = torch.from_numpy(base.copy()).cuda()
        overlay.put_text(m, dev, items)
        assert np.array_equal(dev.cpu().numpy(), ref)
    finally:
        m.close()


def test_put_text_checks_every_item_before_drawing(wn):
    """A bad item in the second group of 64 frames raises before the first group is drawn."""
    import torch
    from whenet_b200 import overlay
    frames = torch.full((70, 8, 8, 3), 5, dtype=torch.uint8, device="cuda")
    good = (0, "a", (1, 7), 0.4, (255, 255, 255))
    for bad in [(69, "a", (1, 7), 0.0, (0, 0, 0)), (69, "a", (1 << 25, 7), 0.4, (0, 0, 0)), (69, "a", (1, 7), 0.4, (0, 0, 256)),
                (69, "a", (1, 7), 0.4, (0, 0, 0), 2), (69, "\t", (1, 7), 0.4, (0, 0, 0)), (69, "a" * 4097, (1, 7), 0.4, (0, 0, 0)),
                (70, "a", (1, 7), 0.4, (0, 0, 0)), (69, "a", (1, 7), float("nan"), (0, 0, 0))]:
        with pytest.raises(ValueError):
            overlay.put_text(wn, frames, [good, bad])
        assert bool((frames == 5).all())
