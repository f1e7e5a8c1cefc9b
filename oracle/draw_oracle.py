"""CPU restatement of OpenCV's ``cv2.line(img, p0, p1, color, 2)`` (LINE_8, shift 0) on an H x W x 3 uint8 array
(TEST INFRASTRUCTURE ONLY, like overlay_oracle.py).  Pinned against the installed cv2 (4.13) as a black box, bit for bit;
tests/test_draw_cpu.py holds it there.  What cv2's output shows, in the order it is drawn:

1. The end points are clipped (Cohen-Sutherland, double arithmetic truncated to integers) against the frame grown by the
   thickness, 2, on every side.  A segment that misses that rectangle draws nothing.  This is why the pixels depend on
   the frame size and not only on the end points.
2. If the clipped end points differ, a convex quad around them in 16.16 fixed point:
   dp = (cvRound(dy * r), cvRound(dx * r)), r = 65536 / sqrt(dx^2 + dy^2) in double, dx = x0 - x1, dy = y1 - y0;
   vertices p0 + dp, p0 - dp, p1 - dp, p1 + dp.
   a. Its outline, four fixed-point line steppers (``_step_line``), each clipped against the frame in 16.16.
   b. Its scan-converted interior (``_fill_quad``), row by row with rounded per-edge x increments.
3. A plus-shaped radius-1 cap at each clipped end point (a zero-length segment is only the plus).

Every quantity is a Python integer except the two double expressions named above, so the restatement is exact."""
from __future__ import annotations

import math

ONE = 1 << 16
HALF = 1 << 15
THICKNESS = 2


def _tdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def clip_segment(w: int, h: int, x1: int, y1: int, x2: int, y2: int):
    """Cohen-Sutherland against [0, w-1] x [0, h-1] as OpenCV's clipLine does it (one pass per axis, double arithmetic
    truncated); None when the segment is rejected."""
    if w <= 0 or h <= 0:
        return None
    right, bottom = w - 1, h - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    if c1 | c2:
        return None
    return x1, y1, x2, y2


def _put(img, x: int, y: int, color) -> None:
    if 0 <= x < img.shape[1] and 0 <= y < img.shape[0]:
        img[y, x] = color


def _step_line(img, p, q, color) -> None:
    """One outline edge: a 16.16 line stepped one pixel per step along its major axis, clipped against the frame in 16.16."""
    H, W = img.shape[:2]
    r = clip_segment(W << 16, H << 16, p[0], p[1], q[0], q[1])
    if r is None:
        return
    x1, y1, x2, y2 = r
    dx, dy = x2 - x1, y2 - y1
    xmajor = abs(dx) > abs(dy)
    if (dx < 0) if xmajor else (dy < 0):
        x1, y1, x2, y2, dx, dy = x2, y2, x1, y1, -dx, -dy
    if xmajor:
        step, count = _tdiv(dy << 16, abs(dx) | 1), (x2 - x1) >> 16
    else:
        step, count = _tdiv(dx << 16, abs(dy) | 1), (y2 - y1) >> 16
    _put(img, (x2 + HALF) >> 16, (y2 + HALF) >> 16, color)
    x1 += HALF
    y1 += HALF
    if xmajor:
        x1 >>= 16
        for _ in range(count + 1):
            _put(img, x1, y1 >> 16, color)
            x1 += 1
            y1 += step
    else:
        y1 >>= 16
        for _ in range(count + 1):
            _put(img, x1 >> 16, y1, color)
            x1 += step
            y1 += 1


def _fill_quad(img, v, color) -> None:
    """Scan conversion of a convex polygon with 16.16 vertices: two edge chains walked down from the top vertex, each
    edge's x advanced by its rounded per-row increment; spans from round(left x) to round(right x), clipped."""
    H, W = img.shape[:2]
    n = len(v)
    imin = min(range(n), key=lambda i: (v[i][1], i))
    xmin = (min(p[0] for p in v) + HALF) >> 16
    xmax = (max(p[0] for p in v) + HALF) >> 16
    ymin = (v[imin][1] + HALF) >> 16
    ymax = (max(p[1] for p in v) + HALF) >> 16
    if xmax < 0 or ymax < 0 or xmin >= W or ymin >= H:
        return
    ymax = min(ymax, H - 1)
    idx, di = [imin, imin], [1, n - 1]
    ex, edx, ye = [-ONE, -ONE], [0, 0], [ymin, ymin]
    edges = n
    y = ymin
    while True:
        for i in range(2):
            if y < ye[i]:
                continue
            i0 = idx[i]
            i1 = (i0 + di[i]) % n
            while edges > 0:
                edges -= 1
                ty = (v[i1][1] + HALF) >> 16
                if ty > y:
                    ye[i] = ty
                    edx[i] = _tdiv((v[i1][0] - v[i0][0]) * 2 + (ty - y), 2 * (ty - y))
                    ex[i] = v[i0][0]
                    idx[i] = i1
                    break
                i0, i1 = i1, (i1 + di[i]) % n
            else:
                edges -= 1
        if edges < 0:
            return
        if y >= 0:
            lo, hi = sorted(ex)
            a, b = (lo + HALF) >> 16, (hi + HALF) >> 16
            if b >= 0 and a < W:
                img[y, max(a, 0):min(b, W - 1) + 1] = color
        ex[0] += edx[0]
        ex[1] += edx[1]
        y += 1
        if y > ymax:
            return


def _cap(img, x: int, y: int, color) -> None:
    for px, py in ((x - 1, y), (x, y), (x + 1, y), (x, y - 1), (x, y + 1)):
        _put(img, px, py, color)


def thick_line_geometry(H: int, W: int, p0, p1):
    """(clipped p0, clipped p1, quad vertices or None) of a thickness-2 segment on an H x W frame; None if nothing is drawn."""
    t = THICKNESS
    r = clip_segment(W + 2 * t, H + 2 * t, p0[0] + t, p0[1] + t, p1[0] + t, p1[1] + t)
    if r is None:
        return None
    q0, q1 = (r[0] - t, r[1] - t), (r[2] - t, r[3] - t)
    X0, Y0, X1, Y1 = q0[0] << 16, q0[1] << 16, q1[0] << 16, q1[1] << 16
    dx, dy = float(q0[0] - q1[0]), float(q1[1] - q0[1])
    rr = dx * dx + dy * dy
    quad = None
    if rr > 2.220446049250313e-16:
        rr = 65536.0 / math.sqrt(rr)
        dpx, dpy = round(dy * rr), round(dx * rr)          # Python's round is round-half-even, as cvRound
        quad = [(X0 + dpx, Y0 + dpy), (X0 - dpx, Y0 - dpy), (X1 - dpx, Y1 - dpy), (X1 + dpx, Y1 + dpy)]
    return q0, q1, quad


def draw_line2(img, p0, p1, color) -> None:
    """``cv2.line(img, p0, p1, color, 2)`` in place on an H x W x 3 uint8 array (integer end points)."""
    g = thick_line_geometry(img.shape[0], img.shape[1], (int(p0[0]), int(p0[1])), (int(p1[0]), int(p1[1])))
    if g is None:
        return
    q0, q1, quad = g
    if quad is not None:
        for k in range(4):
            _step_line(img, quad[k - 1], quad[k], color)
        _fill_quad(img, quad, color)
    _cap(img, q0[0], q0[1], color)
    _cap(img, q1[0], q1[1], color)
