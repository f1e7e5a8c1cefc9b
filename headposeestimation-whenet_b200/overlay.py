"""Host side of the stream path's output: the pose-axis overlay and frame annotation of the reference demos
(SURVEY.md section 8f-4).  Pure host code on top of OpenCV's drawing primitives, exactly the calls the reference makes,
so annotated frames are pixel-identical to the reference's for the same angles.

  ``axis_endpoints`` / ``draw_axis``   reference utils.py:13-43
  ``annotate_head``                    reference demo_video.py:25-34  (rectangle, axes, optional yaw/pitch/roll text)
  ``process_frame``                    reference demo_video.py:11-35,57-58 for all heads of one frame
  ``draw_heads``                       demo_video.py:26,29 (display="simple") for every head of a batch of DEVICE frames, on
                                       the GPU in place (``whenet_draw_heads_u8``, DESIGN.md section 8.7)

``process_frame(reference_order=True)`` reproduces the reference's order of operations bit for bit: it annotates the frame
after EACH head and cuts the next head's crop from the already annotated frame (demo_video.py:57-58 calls
process_detection head by head on the same array), one forward per head.  ``reference_order=False`` (the fast path) cuts
every crop from the CLEAN frame on the GPU in one batch (``WHENet.get_angle_from_frame``) and annotates afterwards; crops that
overlap an earlier head's rectangle / axes / text then differ from the reference's by those drawn pixels - a deliberate
deviation (the drawn overlay is not image content), documented in DESIGN.md.

``draw_heads`` draws on the clean frames what ``oracle/overlay_oracle.process_detection_ref`` draws for each head, pixel for
pixel, with the reference's float32 scalar types (``draw_axis`` below turns the angles into Python floats first, which moves an
axis end point for about 1 head in 100,000; DESIGN.md section 8.7).  ``display="full"`` adds the yaw, pitch and roll labels
of demo_video.py:31-34, and ``put_text`` draws any cv2.putText(FONT_HERSHEY_SIMPLEX, thickness 1) text, both on the GPU
(DESIGN.md section 8.8).
"""
from __future__ import annotations

from math import cos, sin

import numpy as np

from . import crops as _crops


def axis_endpoints(yaw, pitch, roll, tdx, tdy, size):
    """End points (x1,y1) red X axis, (x2,y2) green Y axis, (x3,y3) blue Z axis; angles in degrees (utils.py:15-38)."""
    pitch = pitch * np.pi / 180
    yaw = -(yaw * np.pi / 180)
    roll = roll * np.pi / 180
    x1 = size * (cos(yaw) * cos(roll)) + tdx
    y1 = size * (cos(pitch) * sin(roll) + cos(roll) * sin(pitch) * sin(yaw)) + tdy
    x2 = size * (-cos(yaw) * sin(roll)) + tdx
    y2 = size * (cos(pitch) * cos(roll) - sin(pitch) * sin(yaw) * sin(roll)) + tdy
    x3 = size * (sin(yaw)) + tdx
    y3 = size * (-cos(yaw) * sin(pitch)) + tdy
    return (x1, y1), (x2, y2), (x3, y3)


def draw_axis(img, yaw, pitch, roll, tdx=None, tdy=None, size=100):
    """reference utils.py:13-43: draws on ``img`` in place (BGR) and returns it."""
    import cv2
    if tdx is None or tdy is None:
        height, width = img.shape[:2]
        tdx, tdy = width / 2, height / 2
    (x1, y1), (x2, y2), (x3, y3) = axis_endpoints(float(yaw), float(pitch), float(roll), tdx, tdy, size)
    cv2.line(img, (int(tdx), int(tdy)), (int(x1), int(y1)), (0, 0, 255), 2)
    cv2.line(img, (int(tdx), int(tdy)), (int(x2), int(y2)), (0, 255, 0), 2)
    cv2.line(img, (int(tdx), int(tdy)), (int(x3), int(y3)), (255, 0, 0), 2)
    return img


def annotate_head(img, bounds, yaw, pitch, roll, display: str = "simple"):
    """What demo_video.py:25-34 draws for one head.  ``bounds`` = the margin-enlarged FLOAT bounds
    (y_min, y_max, x_min, x_max) of demo_video.py:15-19 (their fractional parts enter tdx/tdy/size before truncation)."""
    import cv2
    y_min, y_max, x_min, x_max = bounds
    cv2.rectangle(img, (int(x_min), int(y_min)), (int(x_max), int(y_max)), (0, 0, 0), 2)
    draw_axis(img, yaw, pitch, roll, tdx=(x_min + x_max) / 2, tdy=(y_min + y_max) / 2, size=abs(x_max - x_min) // 2)
    if display == "full":
        f, c = cv2.FONT_HERSHEY_SIMPLEX, (100, 255, 0)
        cv2.putText(img, "yaw: {}".format(np.round(yaw)), (int(x_min), int(y_min)), f, 0.4, c, 1)
        cv2.putText(img, "pitch: {}".format(np.round(pitch)), (int(x_min), int(y_min) - 15), f, 0.4, c, 1)
        cv2.putText(img, "roll: {}".format(np.round(roll)), (int(x_min), int(y_min) - 30), f, 0.4, c, 1)
    return img


def process_frame(model, frame, boxes, display: str = "simple", reference_order: bool = True):
    """All detections of one BGR frame: angles + annotation, in place.  Returns ``(frame, yaw, pitch, roll)``.
    ``model`` is anything with ``get_angle`` (and ``get_angle_from_frame`` for the batched path)."""
    import cv2
    n = len(boxes)
    yaw, pitch, roll = (np.zeros((n,), np.float32) for _ in range(3))
    if n == 0:
        return frame, yaw, pitch, roll
    bounds = [_crops.enlarge_bounds(b, frame.shape[0], frame.shape[1]) for b in boxes]
    if reference_order:
        for i, (y0, y1, x0, x1) in enumerate(bounds):
            crop = frame[int(y0):int(y1), int(x0):int(x1)]
            crop = cv2.resize(cv2.cvtColor(crop, cv2.COLOR_BGR2RGB), (224, 224))
            y, p, r = model.get_angle(np.expand_dims(crop, axis=0))
            yaw[i], pitch[i], roll[i] = np.squeeze([y, p, r])
            annotate_head(frame, bounds[i], yaw[i], pitch[i], roll[i], display)
    else:
        y, p, r = model.get_angle_from_frame(frame, boxes, margin=True)
        yaw[:], pitch[:], roll[:] = y, p, r
        for i in range(n):
            annotate_head(frame, bounds[i], yaw[i], pitch[i], roll[i], display)
    return frame, yaw, pitch, roll


DISPLAYS = {"simple": 0, "full": 1}
# put_text's limits, as the library checks them (include/whenet_b200.h)
TEXT_MAX_LEN, TEXT_MAX_CHARS, TEXT_MAX_ITEMS, TEXT_MAX_ORG, TEXT_MAX_SCALE = 4096, 1 << 22, 1 << 20, 1 << 24, 256.0


def _device_frames(whenet, frames, who):
    """(frame list?, items, n) of device BGR frames, or ValueError."""
    from .whenet import _is_device
    frame_list = isinstance(frames, (list, tuple))
    items = list(frames) if frame_list else [frames]
    for f in items:
        if not _is_device(f):
            raise ValueError("%s draws on CUDA tensors; use process_frame for host frames" % who)
        if str(f.dtype) != "torch.uint8" or not f.is_contiguous():
            raise ValueError("frames must be contiguous uint8 CUDA tensors")
        if f.device.index != whenet.device:
            raise ValueError("frames are on cuda:%s, WHENet on cuda:%d" % (f.device.index, whenet.device))
        if len(f.shape) != (3 if frame_list else 4) or f.shape[-1] != 3:
            raise ValueError("frames must be BGR (n, H, W, 3) or a list of (H, W, 3), not %s" % (tuple(f.shape),))
    return frame_list, items, (len(items) if frame_list else int(frames.shape[0]))


def draw_heads(whenet, frames, results, display: str = "simple"):
    """Draw every head of ``results`` into ``frames`` on the GPU, in place: a black thickness-2 rectangle around the
    margin-enlarged box, then the red, green and blue pose axes, bit-identical to the reference's cv2 calls
    (demo_video.py:26,29 with display="simple").  Heads are drawn in result order.  ``display="full"`` also draws, after each
    head's axes, its three labels (demo_video.py:31-34): "yaw: ", "pitch: " and "roll: " with the float32 angle rounded as
    ``np.round`` prints it, FONT_HERSHEY_SIMPLEX at scale 0.4 in (100, 255, 0), at (int(x_min), int(y_min)) and 15 and 30
    rows higher, bit-identical to cv2.putText.  Any other ``display`` raises ``ValueError``.

    ``frames``: a contiguous (n, H, W, 3) uint8 BGR CUDA tensor on ``whenet.device``, or a list or tuple of contiguous
    (H_i, W_i, 3) ones; ``results``: what ``pipeline.detect_and_estimate_frames`` returned for those frames.  A head is
    skipped where the reference would raise: its enlarged slice is empty or leaves the frame, or an angle's float32 radian
    is not finite (the NaN angles of invalid slices).  Returns the per-frame (k,) bool arrays of drawn heads after one
    synchronisation.  Host frames are refused (``process_frame`` is the host path)."""
    import ctypes as C
    import torch
    from ._lib import check
    from .whenet import _ptr
    if display not in DISPLAYS:
        raise ValueError("display must be one of %s, not %r" % (sorted(DISPLAYS), display))
    full = DISPLAYS[display]
    frame_list, items, n = _device_frames(whenet, frames, "draw_heads")
    if len(results) != n:
        raise ValueError("%d results for %d frames" % (len(results), n))
    if n == 0:
        return []
    counts = [len(r[0]) for r in results]
    m = sum(counts)
    if m == 0:
        return [np.zeros((0,), bool) for _ in range(n)]
    boxes = np.ascontiguousarray(np.concatenate([np.asarray(r[0], np.float32).reshape(-1, 4) for r in results]), np.float32)
    angles = np.ascontiguousarray(np.concatenate([np.asarray(r[2], np.float32).reshape(-1, 3) for r in results]), np.float32)
    frame_of = np.repeat(np.arange(n, dtype=np.int32), counts)
    drawn = np.zeros(m, np.int32)
    L = whenet._L
    with torch.cuda.device(whenet.device):
        torch.cuda.current_stream().synchronize()       # frames the caller wrote on torch's stream are complete
        for lo in range(0, n, 64):
            hi = min(n, lo + 64)
            a, b = int(np.searchsorted(frame_of, lo)), int(np.searchsorted(frame_of, hi))
            if a == b:
                continue
            fo = np.ascontiguousarray(frame_of[a:b] - lo)
            if frame_list:
                ptrs = (C.c_void_p * (hi - lo))(*[f.data_ptr() for f in items[lo:hi]])
                hw = np.array([f.shape[:2] for f in items[lo:hi]], np.int32)
                if full:
                    check(L.whenet_draw_heads_ex_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, _ptr(boxes[a:]),
                                                           _ptr(angles[a:]), _ptr(fo), b - a, full, _ptr(drawn[a:])))
                else:
                    check(L.whenet_draw_heads_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, _ptr(boxes[a:]), _ptr(angles[a:]),
                                                        _ptr(fo), b - a, _ptr(drawn[a:])))
            else:
                _, H, W, _c = frames.shape
                if full:
                    check(L.whenet_draw_heads_ex_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, _ptr(boxes[a:]), _ptr(angles[a:]),
                                                    _ptr(fo), b - a, full, _ptr(drawn[a:])))
                else:
                    check(L.whenet_draw_heads_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, _ptr(boxes[a:]), _ptr(angles[a:]),
                                                 _ptr(fo), b - a, _ptr(drawn[a:])))
        whenet.synchronize()
    out, off = [], 0
    for k in counts:
        out.append(drawn[off:off + k].astype(bool))
        off += k
    return out


def put_text(whenet, frames, items):
    """Draw text into device BGR ``frames`` on the GPU, in place, bit-identical to
    ``cv2.putText(frame, text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, color, thickness)`` (LINE_8).

    ``frames``: as ``draw_heads``.  ``items``: a sequence of ``(frame_index, text, (x, y), scale, (b, g, r))`` or
    ``(frame_index, text, (x, y), scale, (b, g, r), thickness)`` tuples, drawn in order.  ``text`` is printable ASCII of at
    most 4096 characters (2^22 in all per 64 frames); |x|, |y| <= 2^24; 0 < scale <= 256; colour channels are integers in
    [0, 255]; only thickness 1 is supported.  Every item and frame is checked here, before anything is drawn, and a bad one
    raises ``ValueError``.  The library can still refuse a group of 64 frames after earlier groups were drawn in one case
    only: text so large that its row-banded segment list would exceed 2^31 entries.  Synchronises once."""
    import ctypes as C
    import torch
    from ._lib import WhenetError, check
    from .whenet import _ptr
    import math
    frame_list, fitems, n = _device_frames(whenet, frames, "put_text")
    if n == 0 or len(items) == 0:
        return
    for k, f in enumerate(fitems if frame_list else [frames[0]]):
        H, W = int(f.shape[-3]), int(f.shape[-2])
        if not (1 <= H <= 16384 and 1 <= W <= 16384):
            raise ValueError("frame %d: size %dx%d outside [1, 16384]" % (k, W, H))
    rows = []
    for it in items:
        it = tuple(it)
        if len(it) not in (5, 6):
            raise ValueError("an item is (frame_index, text, (x, y), scale, (b, g, r)[, thickness]), not %r" % (it,))
        f, text, (x, y), scale, col = it[:5]
        thick = it[5] if len(it) == 6 else 1
        if int(f) != f or not 0 <= f < n:
            raise ValueError("frame index %r outside [0, %d)" % (f, n))
        if not isinstance(text, str) or len(text) > TEXT_MAX_LEN or not all(32 <= ord(ch) <= 126 for ch in text):
            raise ValueError("text must be printable ASCII of at most %d characters: %r" % (TEXT_MAX_LEN, text))
        if int(x) != x or int(y) != y or abs(x) > TEXT_MAX_ORG or abs(y) > TEXT_MAX_ORG:
            raise ValueError("origin %r must be integers within +-2^24" % ((x, y),))
        if not (math.isfinite(float(scale)) and 0 < float(scale) <= TEXT_MAX_SCALE):
            raise ValueError("scale %r outside (0, %g]" % (scale, TEXT_MAX_SCALE))
        col = tuple(col)
        if len(col) != 3 or any(int(v) != v or not 0 <= v <= 255 for v in col):
            raise ValueError("colour %r must be three integers in [0, 255]" % (col,))
        if thick != 1:
            raise ValueError("thickness %r: only 1 is supported" % (thick,))
        rows.append((int(f), text.encode("ascii"), int(x), int(y), float(scale), [int(v) for v in col]))
    fo = np.array([r[0] for r in rows], np.int32)
    for lo in range(0, n, 64):          # the library's per-call limits, one call per 64 frames
        chunk = [len(r[1]) for r in rows if lo <= r[0] < lo + 64]
        if len(chunk) > TEXT_MAX_ITEMS or sum(chunk) > TEXT_MAX_CHARS:
            raise ValueError("more than 2^20 items or 2^22 characters for frames %d..%d" % (lo, min(n, lo + 64) - 1))
    texts = [r[1] for r in rows]
    org = np.array([[r[2], r[3]] for r in rows], np.int32).reshape(-1, 2)
    scale = np.array([r[4] for r in rows], np.float64)
    bgr = np.array([r[5] for r in rows], np.uint8).reshape(-1, 3)
    thick = np.ones(len(rows), np.int32)
    L = whenet._L
    with torch.cuda.device(whenet.device):
        torch.cuda.current_stream().synchronize()
        for lo in range(0, n, 64):
            hi = min(n, lo + 64)
            sel = np.nonzero((fo >= lo) & (fo < hi))[0]
            if len(sel) == 0:
                continue
            tp = (C.c_char_p * len(sel))(*[texts[i] for i in sel])
            f_sel = np.ascontiguousarray(fo[sel] - lo)
            o_sel, s_sel = np.ascontiguousarray(org[sel]), np.ascontiguousarray(scale[sel])
            c_sel, t_sel = np.ascontiguousarray(bgr[sel]), np.ascontiguousarray(thick[sel])
            try:
                if frame_list:
                    ptrs = (C.c_void_p * (hi - lo))(*[f.data_ptr() for f in fitems[lo:hi]])
                    hw = np.array([f.shape[:2] for f in fitems[lo:hi]], np.int32)
                    check(L.whenet_put_text_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, _ptr(f_sel), C.addressof(tp),
                                                      _ptr(o_sel), _ptr(s_sel), _ptr(c_sel), _ptr(t_sel), len(sel)))
                else:
                    _, H, W, _c = frames.shape
                    check(L.whenet_put_text_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, _ptr(f_sel), C.addressof(tp),
                                               _ptr(o_sel), _ptr(s_sel), _ptr(c_sel), _ptr(t_sel), len(sel)))
            except WhenetError as e:
                if e.code == -1:
                    raise ValueError(str(e)) from e
                raise
        whenet.synchronize()
