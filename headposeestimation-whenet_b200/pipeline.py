"""Frames -> head poses on the GPU: reference demo_video.py:49-63 (detect, then margin, crop, resize and get_angle for every
head, demo_video.py:13-23 and 54-58) for the heads of many frames at once."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import crops as _crops
from ._lib import WhenetError, check
from .whenet import _is_device, _ptr
from .yolo import _entry_name, _frame_list, _frame_table, _image_size, _is_422, _pixel_layout, _yuv422_image_size, _yuv_image_size


def detect_and_estimate(yolo, whenet, frame_bgr, *, pixel_format="bgr"):
    """``frame_bgr``: H x W x 3 uint8 as cv2 delivers it -> (boxes (k,4) float32, scores (k,) float32, angles (k,3) float32
    yaw/pitch/roll in degrees).  The one-frame case of ``detect_and_estimate_frames``, except that a head whose slice is
    empty or outside the frame raises ``WhenetError`` (code -1, naming the box and its slice) as cv2.resize raises in the
    reference, instead of getting NaN angles.  ``pixel_format="nv12"`` / ``"i420"``: an (H * 3/2, W) YUV 4:2:0 frame in
    cv2's layout, ``"yuyv"`` / ``"uyvy"``: an (H, W, 2) packed YUV 4:2:2 frame (see ``detect_and_estimate_frames``)."""
    layout = _pixel_layout(pixel_format)
    frame = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
    if _is_422(layout):
        _yuv422_image_size(frame.shape, "frame")
    elif layout:
        _yuv_image_size(frame.shape, "frame")
    elif frame.ndim != 3 or frame.shape[2] != 3:
        raise ValueError("frame must be H x W x 3 uint8")
    return _run(yolo, whenet, frame[None], strict=True, pixel_format=pixel_format)[0]


def detect_and_estimate_frames(yolo, whenet, frames_bgr, *, pixel_format="bgr"):
    """``frames_bgr``: (n, H, W, 3) uint8 BGR frames of one size, a numpy array or a contiguous CUDA uint8 tensor on
    ``whenet.device`` -> n tuples (boxes (k,4) float32, scores (k,) float32, angles (k,3) float32), per frame bit-identical
    to ``detect_and_estimate`` on that frame alone.

    Frames go through the detector ``yolo.max_frames`` at a time (host frames are uploaded chunk by chunk into two reused
    device buffers); each chunk's boxes are enlarged, cut out of that chunk's device frames, resized and fed to WHENet in
    sub-batches of ``whenet.max_batch`` through one reused crop buffer, queued on WHENet's stream while the detector runs the
    next chunk on its own.  One synchronisation at the end.

    A head whose enlarged slice is empty or leaves the frame (where the reference's cv2.resize raises and ends the video
    loop) gets NaN angles; its box and score are returned as the detector gave them.

    ``frames_bgr`` may also be a list or tuple of (H_i, W_i, 3) uint8 BGR frames of any sizes (several cameras), all numpy
    arrays or all contiguous CUDA tensors on ``whenet.device``; frames of one size run as the batch above.  Frames of several
    sizes take the same path through the per-frame entries (``whenet_det_detect_ragged_u8``, ``whenet_crop_boxes_ragged_u8``),
    each frame's result bit-identical to ``detect_and_estimate`` on that frame alone.  An empty list gives [].

    ``pixel_format="nv12"`` or ``"i420"`` takes YUV 4:2:0 video frames in cv2's layout (what hardware and software video
    decoders hand out) instead of BGR: (n, H * 3/2, W) uint8, or a list or tuple of (H_i * 3/2, W_i) frames, H and W even.
    The letterbox and the crops convert each pixel as they read it, so host frames upload half the bytes of BGR frames, and
    the results are the bits ``detect_and_estimate_frames`` gives on ``cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12 / _I420)``.

    ``pixel_format="yuyv"`` or ``"uyvy"`` takes packed YUV 4:2:2 frames (what raw webcams, V4L2 and GStreamer pipelines and
    HDMI capture cards hand out): (n, H, W, 2) uint8, or a list or tuple of (H_i, W_i, 2) frames, W even, any H.  Host frames
    upload 2 bytes per pixel, and the results are the bits ``detect_and_estimate_frames`` gives on
    ``cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_YUYV / _UYVY)``.  ``video.to_bgr`` turns the same frames into BGR frames on the
    device for ``overlay.draw_heads`` and ``video.encode_jpeg``."""
    return _run(yolo, whenet, frames_bgr, strict=False, pixel_format=pixel_format)


def _checked_frames(yolo, whenet, frames, layout):
    if yolo.device != whenet.device:
        raise ValueError("the detector runs on device %d and WHENet on device %d" % (yolo.device, whenet.device))
    if isinstance(frames, (list, tuple)):
        frames, dev = _frame_list(frames, whenet.device, layout)
        if len({tuple(f.shape) for f in frames}) > 1:
            return frames
        if not frames:
            return np.zeros((0, 1, 1, 3), np.uint8)
        if not dev:
            return np.stack(frames)
        import torch
        with torch.cuda.device(whenet.device):
            return torch.stack(frames)
    if _is_device(frames):
        if str(frames.dtype) != "torch.uint8" or not frames.is_contiguous():
            raise ValueError("device frames must be a contiguous uint8 CUDA tensor")
        if frames.device.index != whenet.device:
            raise ValueError("frames are on cuda:%s, WHENet on cuda:%d" % (frames.device.index, whenet.device))
    else:
        frames = np.asarray(frames)
        if frames.dtype != np.uint8:
            raise ValueError("frames must be uint8, not %s" % frames.dtype)
    if _is_422(layout):
        if len(frames.shape) != 4:
            raise ValueError("frames must be (n, H, W, 2) uint8 for a 4:2:2 pixel format, not %s" % (tuple(frames.shape),))
        _yuv422_image_size(frames.shape[1:], "a frame")
    elif layout:
        if len(frames.shape) != 3:
            raise ValueError("frames must be (n, H * 3/2, W) uint8 for a 4:2:0 pixel format, not %s" % (tuple(frames.shape),))
        _yuv_image_size(frames.shape[1:], "a frame")
    elif len(frames.shape) != 4 or frames.shape[3] != 3:
        raise ValueError("frames must be (n, H, W, 3) uint8, not %s" % (tuple(frames.shape),))
    return frames


def _raise_first_invalid(L, boxes, H, W):
    """detect_and_estimate's error: the first box whose slice cv2.resize would refuse, as whenet_crop_resize_u8 names it."""
    valid = np.empty(len(boxes), np.int32)
    check(L.whenet_debug_enlarge_boxes(_ptr(boxes), len(boxes), H, W, None, _ptr(valid)))
    if valid.all():
        return
    i = int(np.flatnonzero(valid == 0)[0])
    y0, y1, x0, x1 = _crops.enlarge_box(boxes[i], H, W)
    raise WhenetError(-1, "box %d: slice [%d:%d, %d:%d] is empty or outside the %dx%d frame (cv2.resize would raise)"
                      % (i, y0, y1, x0, x1, H, W))


def _run(yolo, whenet, frames, strict, pixel_format="bgr"):
    layout = _pixel_layout(pixel_format)
    frames = _checked_frames(yolo, whenet, frames, layout)
    ragged = isinstance(frames, list)       # frames of several sizes; otherwise one (n, H, W, 3), (n, H * 3/2, W) or (n, H, W, 2) array or tensor
    n = len(frames) if ragged else int(frames.shape[0])
    if n == 0:
        return []
    if not ragged:
        H, W = _image_size(frames.shape[1:], layout)
    import torch
    L = whenet._L
    dev = _is_device(frames[0] if ragged else frames)
    step = yolo.max_frames
    n_chunks = -(-n // step)
    results = []            # per chunk: (detections, device angles or None, validity or None)
    keep = []               # device buffers WHENet's stream may still read or write: alive until the final synchronisation
    stage = [None, None]    # host frames: chunk k goes to stage[k % 2]
    crop_buf = None

    def stage_ragged(k, part):
        """Host frames of several sizes -> views of one device buffer, each frame at a 256-byte aligned offset."""
        offs = np.cumsum([0] + [-(-f.size // 256) * 256 for f in part])
        buf = stage[k % 2]
        if buf is None or buf.numel() < offs[-1]:
            cap = max(sum(-(-f.size // 256) * 256 for f in frames[j:j + step]) for j in range(0, n, step))
            buf = stage[k % 2] = torch.empty((cap,), dtype=torch.uint8, device="cuda")
        views = [buf[int(o):int(o) + f.size].view(f.shape) for f, o in zip(part, offs)]
        for v, f in zip(views, part):
            v.copy_(torch.from_numpy(f))
        torch.cuda.current_stream().synchronize()       # the detector reads them on its own stream
        return views

    def chunk(k):
        lo, hi = k * step, min(n, (k + 1) * step)
        if dev:
            return frames[lo:hi]
        if ragged:
            return stage_ragged(k, frames[lo:hi])
        buf = stage[k % 2]
        if buf is None:
            buf = stage[k % 2] = torch.empty((min(step, n),) + tuple(frames.shape[1:]), dtype=torch.uint8, device="cuda")
        buf[:hi - lo].copy_(torch.from_numpy(np.ascontiguousarray(frames[lo:hi])))
        torch.cuda.current_stream().synchronize()       # the detector reads it on its own stream
        return buf[:hi - lo]

    with torch.cuda.device(whenet.device):
        if dev:
            torch.cuda.current_stream().synchronize()   # frames the caller wrote on torch's stream are complete
        try:
            cur = chunk(0)
            for k in range(n_chunks):
                nb = len(cur)
                dets = yolo.detect_frames(cur, pixel_format=pixel_format)      # synchronous, on the detector's stream
                if k + 1 < n_chunks:
                    if not dev:
                        whenet.synchronize()            # chunk k-1's crops have read the buffer chunk k+1 goes to
                    nxt = chunk(k + 1)
                counts = [len(d[0]) for d in dets]
                m = sum(counts)
                if m == 0:
                    results.append((dets, None, None))
                else:
                    boxes = np.ascontiguousarray(np.concatenate([d[0] for d in dets]), np.float32)
                    frame_of = np.repeat(np.arange(nb, dtype=np.int32), counts)
                    if strict:
                        _raise_first_invalid(L, boxes, H, W)
                    valid = np.empty(m, np.int32)
                    d_ang = torch.empty((m, 3), dtype=torch.float32, device="cuda")
                    keep.append(d_ang)
                    if ragged:
                        ptrs, hw = _frame_table(cur, layout)
                    for s in range(0, m, whenet.max_batch):
                        mb = min(whenet.max_batch, m - s)
                        if crop_buf is None or crop_buf.shape[0] < mb:
                            crop_buf = torch.empty((mb, 224, 224, 3), dtype=torch.uint8, device="cuda")
                            keep.append(crop_buf)
                        # layout in place of swap_rb = 1: the YUV entries write RGB crops as the BGR ones do with it
                        if ragged:
                            crop = getattr(L, _entry_name("whenet_crop_boxes_ragged", layout))
                            check(crop(whenet._h, C.addressof(ptrs), _ptr(hw), nb, 1, _ptr(boxes[s:]), _ptr(frame_of[s:]), mb, layout or 1,
                                       _ptr(crop_buf), None, _ptr(valid[s:])))
                        else:
                            crop = getattr(L, _entry_name("whenet_crop_boxes", layout))
                            check(crop(whenet._h, _ptr(cur), nb, H, W, 1, _ptr(boxes[s:]), _ptr(frame_of[s:]), mb, layout or 1,
                                       _ptr(crop_buf), None, _ptr(valid[s:])))
                        check(L.whenet_forward_u8(whenet._h, _ptr(crop_buf), mb, 1, _ptr(d_ang[s:s + mb]), None, 1))
                    results.append((dets, d_ang, valid))
                if k + 1 < n_chunks:
                    keep.append(cur)
                    cur = nxt
        except BaseException:
            L.whenet_synchronize(whenet._h)             # unchecked: the buffers must outlive the queued work on the way out
            raise
        whenet.synchronize()
        out = []
        for dets, d_ang, valid in results:
            if d_ang is None:
                out.extend((b, s, np.zeros((0, 3), np.float32)) for b, s, _c in dets)
                continue
            ang = d_ang.cpu().numpy()
            ang[valid == 0] = np.nan
            off = 0
            for b, s, _c in dets:
                out.append((b, s, ang[off:off + len(b)].copy()))
                off += len(b)
        return out
