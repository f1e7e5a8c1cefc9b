"""CPU restatement of OpenCV's ``cv2.putText(img, text, org, FONT_HERSHEY_SIMPLEX, scale, color, 1)`` (LINE_8,
bottomLeftOrigin=False) on an H x W x 3 uint8 array, and of the reference's label strings (TEST INFRASTRUCTURE ONLY, like
draw_oracle.py).  tests/test_text_cpu.py holds it bit for bit against the installed cv2.  What putText does:

1. hscale = vscale = cvRound(scale * 65536); the pen starts at (org.x << 16, (org.y << 16) + base_line * vscale).
2. For each character, its glyph (left bearing, right bearing, strokes of points, hershey_simplex.py): the pen moves left by
   the left bearing, each point (px, py) lands at (px * hscale + pen.x, py * vscale + pen.y) in 16.16, and the pen then
   moves right by the right bearing.
3. Every stroke of more than one point is a polyline of thickness 1 with shift 16.  cv2 4.13 draws each of its segments
   (``draw_line1``) by rounding both 16.16 end points to pixels ((v + 32768) >> 16), clipping them against the frame
   (draw_oracle.clip_segment, integer) and stepping OpenCV's 8-connected LineIterator from the left end point: pixel k
   along the major axis sits ceil((2Bk - A) / 2A) pixels along the minor one (A = major length, B = minor length), a
   tie going toward the left end point's row or column.  This is not draw_oracle._step_line's fixed-point stepper,
   which agrees only on horizontal, vertical and some diagonal segments.

Every quantity is a Python integer except cvRound's double product, so the restatement is exact."""
from __future__ import annotations

import numpy as np

import draw_oracle as D


def glyph_strokes(glyph: str, hscale: int, vscale: int, pen_x: int, pen_y: int):
    """The strokes of one glyph at pen (pen_x already moved by the left bearing), as lists of 16.16 points; OpenCV's own
    parse: a point is two characters, a space or the end closes a stroke."""
    strokes, pts, i = [], [], 2
    while True:
        if i >= len(glyph) or glyph[i] == " ":
            if len(pts) > 1:
                strokes.append(pts)
            if i >= len(glyph):
                return strokes
            i += 1
            pts = []
        else:
            pts.append(((ord(glyph[i]) - 82) * hscale + pen_x, (ord(glyph[i + 1]) - 82) * vscale + pen_y))
            i += 2


def text_segments(text: str, org, scale: float, glyphs=None, base_line=None):
    """The 16.16 segments (x1, y1, x2, y2) putText draws, in draw order (the committed table unless one is given)."""
    if glyphs is None:
        import hershey_simplex as HS
        glyphs, base_line = HS.GLYPHS, HS.BASE_LINE
    hscale = round(float(scale) * 65536)            # cvRound: round half to even, as Python's round
    vscale = hscale
    pen_x = int(org[0]) << 16
    pen_y = (int(org[1]) << 16) + base_line * vscale
    segs = []
    for ch in text:
        c = ord(ch)
        if not 32 <= c <= 126:
            raise ValueError("character %r is not printable ASCII" % ch)
        g = glyphs[c - 32]
        left, right = ord(g[0]) - 82, ord(g[1]) - 82
        advance = right * hscale
        pen_x -= left * hscale
        for pts in glyph_strokes(g, hscale, vscale, pen_x, pen_y):
            segs += [(p[0], p[1], q[0], q[1]) for p, q in zip(pts, pts[1:])]
        pen_x += advance
    return segs


def line_pixels(H: int, W: int, x1: int, y1: int, x2: int, y2: int):
    """The pixels (x, y) of one thickness-1 segment between 16.16 end points on an H x W frame, in LineIterator order."""
    r = D.clip_segment(W, H, (x1 + D.HALF) >> 16, (y1 + D.HALF) >> 16, (x2 + D.HALF) >> 16, (y2 + D.HALF) >> 16)
    if r is None:
        return []
    x1, y1, x2, y2 = r
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, abs(y2 - y1)
    sy = 1 if y2 >= y1 else -1
    A, B = max(dx, dy), min(dx, dy)
    out = []
    for k in range(A + 1):
        m = max(0, -((A - 2 * B * k) // (2 * A))) if A else 0
        out.append((x1 + m, y1 + sy * k) if dy > dx else (x1 + k, y1 + sy * m))
    return out


def draw_line1(img, x1: int, y1: int, x2: int, y2: int, color) -> None:
    """``cv2.line(img, (x1, y1), (x2, y2), color, 1, LINE_8, shift=16)`` in place."""
    for x, y in line_pixels(img.shape[0], img.shape[1], x1, y1, x2, y2):
        img[y, x] = color


def put_text(img, text: str, org, scale: float, color, glyphs=None, base_line=None):
    """``cv2.putText(img, text, org, FONT_HERSHEY_SIMPLEX, scale, color, 1)`` in place."""
    for x1, y1, x2, y2 in text_segments(text, org, scale, glyphs, base_line):
        draw_line1(img, x1, y1, x2, y2, color)
    return img


def label_text(a) -> str:
    """The number in the reference's labels (demo_video.py:31-34): ``"{}".format(np.round(a))`` of a float32 angle.  The empty
    format spec formats the float32 as a Python float ("1000000.0"), unlike ``str`` ("1e+06"); they agree within +-180."""
    return "{}".format(np.round(np.float32(a)))


def label_items(x_min: int, y_min: int, yaw, pitch, roll):
    """The three putText calls of display="full" for one head: (text, org), scale 0.4, colour (100, 255, 0)."""
    return [("yaw: " + label_text(yaw), (x_min, y_min)), ("pitch: " + label_text(pitch), (x_min, y_min - 15)),
            ("roll: " + label_text(roll), (x_min, y_min - 30))]
