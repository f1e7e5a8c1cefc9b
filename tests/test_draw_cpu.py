"""Head overlay without a GPU (DESIGN.md section 8.7): oracle/draw_oracle.py equals cv2.line(..., 2) bit for bit, the C host
geometry (whenet_debug_overlay_segments) equals the reference-typed Python geometry, argument checks, and ptxas facts."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(__file__), "..")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
cv2 = pytest.importorskip("cv2")

import draw_oracle as D  # noqa: E402

EINVAL = -1         # WHENET_EINVAL

SIZES = [(1, 1, 12000), (2, 2, 12000), (3, 5, 12000), (40, 50, 14000), (417, 417, 2500), (1080, 1920, 400), (2160, 3840, 100),
         (16384, 24, 300), (24, 16384, 300)]


def _segment(rng, H, W):
    s = max(H, W)
    k = int(rng.integers(0, 5))
    lim = [3, s + 3, 2 * s, 5 * s, 3 * 16384][k]
    hi = lim + s * (k == 0)
    p0 = [int(v) for v in rng.integers(-lim, hi, 2)]
    p1 = [int(v) for v in rng.integers(-lim, hi, 2)]
    u = rng.random()
    if u < 0.05:
        p1 = list(p0)                                   # zero length: only the caps
    elif u < 0.1:
        p1[1] = p0[1]                                   # horizontal
    elif u < 0.15:
        p1[0] = p0[0]                                   # vertical
    elif u < 0.2:
        d = int(rng.integers(-s, s + 1))                # 45 degrees
        p1 = [p0[0] + d, p0[1] + d * int(rng.choice([-1, 1]))]
    elif u < 0.3:                                       # end points on the frame's edges and corners
        p0 = [int(rng.choice([0, W - 1, W, -1, W // 2])), int(rng.choice([0, H - 1, H, -1, H // 2]))]
    return p0, p1


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_equals_cv2_line(seed):
    """>= 100,000 random segments over both seeds, overlapping in order with random colours on one canvas per size."""
    rng = np.random.default_rng(seed)
    for H, W, n in SIZES:
        a = np.zeros((H, W, 3), np.uint8)
        b = a.copy()
        for t in range(n):
            p0, p1 = _segment(rng, H, W)
            c = tuple(int(v) for v in rng.integers(0, 256, 3))
            cv2.line(a, tuple(p0), tuple(p1), c, 2)
            D.draw_line2(b, p0, p1, c)
            if t % 100 == 99 or t == n - 1:
                assert np.array_equal(a, b), (H, W, t, p0, p1)


def test_rectangle_is_four_lines():
    rng = np.random.default_rng(7)
    for H, W in [(1, 1), (3, 5), (40, 50), (417, 417)]:
        for _ in range(500):
            x0, x1 = sorted(int(v) for v in rng.integers(-3, W + 4, 2))
            y0, y1 = sorted(int(v) for v in rng.integers(-3, H + 4, 2))
            a = np.full((H, W, 3), 9, np.uint8)
            b = a.copy()
            cv2.rectangle(a, (x0, y0), (x1, y1), (0, 0, 0), 2)
            for p, q in (((x0, y0), (x1, y0)), ((x1, y0), (x1, y1)), ((x1, y1), (x0, y1)), ((x0, y1), (x0, y0))):
                D.draw_line2(b, p, q, (0, 0, 0))
            assert np.array_equal(a, b), (H, W, x0, y0, x1, y1)


class _Recorder:
    """Stands in for cv2 inside overlay_oracle: records the segments instead of drawing them."""
    def __init__(self):
        self.segs = []

    def line(self, img, p, q, color, t):
        self.segs.append((p[0], p[1], q[0], q[1]))

    def rectangle(self, img, p, q, color, t):
        (x0, y0), (x1, y1) = p, q
        self.segs += [(x0, y0, x1, y0), (x1, y0, x1, y1), (x1, y1, x0, y1), (x0, y1, x0, y0)]


def _ref_segments(box, ang, H, W):
    """process_detection_ref's geometry with its numpy 2 scalar types, or None where it raises."""
    import overlay_oracle as O
    rec = _Recorder()
    img = np.zeros((H, W, 0), np.uint8)
    y_min, x_min, y_max, x_max = (np.float32(v) for v in box)
    y_min = max(0, y_min - abs(y_min - y_max) / 10)
    y_max = min(H, y_max + abs(y_min - y_max) / 10)
    x_min = max(0, x_min - abs(x_min - x_max) / 5)
    x_max = min(W, x_max + abs(x_min - x_max) / 5)
    x_max = min(x_max, W)
    if not (int(y_min) < int(y_max) and int(x_min) < int(x_max) and int(y_min) <= H and int(x_min) <= W):
        return None
    saved = O.cv2
    O.cv2 = rec
    try:
        rec.rectangle(img, (int(x_min), int(y_min)), (int(x_max), int(y_max)), None, 2)
        with np.errstate(over="ignore", invalid="ignore"):
            O.draw_axis_ref(img, np.float32(ang[0]), np.float32(ang[1]), np.float32(ang[2]), tdx=(x_min + x_max) / 2,
                            tdy=(y_min + y_max) / 2, size=abs(x_max - x_min) // 2)
    except (ValueError, OverflowError):
        return None
    finally:
        O.cv2 = saved
    return rec.segs


def test_host_geometry_equals_reference_types():
    from whenet_b200 import _lib
    L = _lib.load()
    rng = np.random.default_rng(11)
    sizes = [(1, 1), (2, 3), (417, 417), (1080, 1920), (2160, 3840), (16384, 16384), (16384, 7)]
    per = 15000
    kinds = set()
    drawn_total = 0
    for H, W in sizes:
        u = rng.random((per, 4))
        # boxes: inside, spilling over either or both sides (the clamp-type combinations), empty, far outside
        y0 = (u[:, 0] * 1.4 - 0.3) * H
        x0 = (u[:, 1] * 1.4 - 0.3) * W
        y1 = y0 + rng.uniform(-0.1, 1.6, per) * H
        x1 = x0 + rng.uniform(-0.1, 1.6, per) * W
        boxes = np.stack([y0, x0, y1, x1], 1).astype(np.float32)
        ang = rng.uniform(-200, 200, (per, 3)).astype(np.float32)
        ang[::97, 0] = np.nan
        ang[::89, 1] = np.inf
        ang[::83, 2] = -np.inf
        ang[::79, 0] = 3e38
        ang[::73, 1] = 1e30
        boxes[::71] = np.nan
        seg = np.zeros((per, 7, 4), np.int32)
        drawn = np.zeros(per, np.int32)
        assert L.whenet_debug_overlay_segments(boxes.ctypes.data, ang.ctypes.data, per, H, W, seg.ctypes.data, drawn.ctypes.data) == 0
        for i in range(per):
            ref = _ref_segments(boxes[i], ang[i], H, W)
            assert bool(drawn[i]) == (ref is not None), (H, W, i, boxes[i], ang[i])
            if ref is None:
                assert not seg[i].any()
                continue
            drawn_total += 1
            assert [tuple(s) for s in seg[i].tolist()] == [tuple(int(v) for v in s) for s in ref], (H, W, i, boxes[i], ang[i])
            vy0 = boxes[i, 0] - abs(boxes[i, 0] - boxes[i, 2]) / np.float32(10)
            vx0 = boxes[i, 1] - abs(boxes[i, 1] - boxes[i, 3]) / np.float32(5)
            kinds.add((bool(vx0 <= 0) and seg[i, 0, 2] == W, bool(vy0 <= 0) and seg[i, 1, 3] == H))
    assert len(sizes) * per >= 100000 and drawn_total > 50000
    assert kinds == {(False, False), (False, True), (True, False), (True, True)}


def test_argument_checks():
    from whenet_b200 import _lib
    L = _lib.load()
    b = np.zeros((1, 4), np.float32)
    a = np.zeros((1, 3), np.float32)
    fo = np.zeros(1, np.int32)
    buf = (C.c_uint8 * 3)()
    assert L.whenet_debug_overlay_segments(None, a.ctypes.data, 1, 10, 10, None, None) == EINVAL
    assert L.whenet_debug_overlay_segments(b.ctypes.data, a.ctypes.data, 1, 0, 10, None, None) == EINVAL
    assert L.whenet_debug_overlay_segments(b.ctypes.data, a.ctypes.data, 1, 10, 16385, None, None) == EINVAL
    d = C.addressof(buf)
    assert L.whenet_draw_heads_u8(None, None, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    assert L.whenet_draw_heads_u8(None, d, 0, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    assert L.whenet_draw_heads_u8(None, d, 65, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    assert L.whenet_draw_heads_u8(None, d, 1, 16385, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    assert L.whenet_draw_heads_u8(None, d, 1, 1, 1, None, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    bad_fo = np.array([1], np.int32)
    assert L.whenet_draw_heads_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, bad_fo.ctypes.data, 1, None) == EINVAL
    assert b"frame_of" in L.whenet_last_error()
    assert L.whenet_draw_heads_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, -1, None) == EINVAL
    assert L.whenet_draw_heads_u8(None, d, 1, 1, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1, None) == EINVAL
    assert b"context" in L.whenet_last_error()
    assert L.whenet_draw_heads_u8(None, d, 1, 1, 1, None, None, None, 0, None) == 0          # m = 0: nothing to do
    ptrs = (C.c_void_p * 1)(d)
    hw = np.array([[1, 0]], np.int32)
    assert L.whenet_draw_heads_ragged_u8(None, C.addressof(ptrs), hw.ctypes.data, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1,
                                         None) == EINVAL
    assert L.whenet_draw_heads_ragged_u8(None, None, hw.ctypes.data, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1,
                                         None) == EINVAL
    nul = (C.c_void_p * 1)()
    hw = np.array([[1, 1]], np.int32)
    assert L.whenet_draw_heads_ragged_u8(None, C.addressof(nul), hw.ctypes.data, 1, b.ctypes.data, a.ctypes.data, fo.ctypes.data, 1,
                                         None) == EINVAL


def test_draw_heads_refuses_bad_frames():
    from whenet_b200 import overlay

    class FakeWhenet:
        device = 0

    res = [(np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros((0, 3), np.float32))]
    with pytest.raises(ValueError):
        overlay.draw_heads(FakeWhenet(), np.zeros((1, 4, 4, 3), np.uint8), res)
    with pytest.raises(ValueError):
        overlay.draw_heads(FakeWhenet(), [np.zeros((4, 4, 3), np.uint8)], res)


def test_overlay_kernel_does_not_spill(tmp_path):
    src = tmp_path / "k.cu"
    src.write_text('#include "%s"\n' % os.path.abspath(os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc", "kernels_overlay.cuh")))
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas=-v", "-c", "-o",
                        str(tmp_path / "k.o"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "overlay_draw_kernel" in r.stderr
    assert "0 bytes spill stores, 0 bytes spill loads" in r.stderr, r.stderr
