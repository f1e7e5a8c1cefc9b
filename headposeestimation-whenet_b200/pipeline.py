"""Frame -> head poses on the GPU (reference demo_video.py:54-58 steps 1-3 for every head of a frame at once)."""
from __future__ import annotations

import numpy as np

from . import crops as _crops
from ._lib import check
from .whenet import _ptr


def detect_and_estimate(yolo, whenet, frame_bgr):
    """``frame_bgr``: H x W x 3 uint8 as cv2 delivers it.  The frame is uploaded once; the detector reads it on the device
    (yolo.detect on its RGB view), only the small box arrays visit the host for the margin arithmetic
    (crops.rects_from_boxes, demo_video.py:13-21), and the crops are cut, resized and fed to WHENet without leaving the device.

    Returns (boxes (k,4) float32, scores (k,) float32, angles (k,3) float32 yaw/pitch/roll in degrees)."""
    import torch
    frame = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
    if frame.ndim != 3 or frame.shape[2] != 3:
        raise ValueError("frame must be H x W x 3 uint8")
    H, W = frame.shape[:2]
    with torch.cuda.device(whenet.device):
        d_frame = torch.from_numpy(frame).to("cuda")
        torch.cuda.current_stream().synchronize()
        boxes, scores, _classes = yolo.detect_frames(d_frame[None])[0]
        m = len(boxes)
        if m == 0:
            return boxes, scores, np.zeros((0, 3), np.float32)
        rects = _crops.rects_from_boxes(boxes, H, W, True)
        d_crops = torch.empty((m, 224, 224, 3), dtype=torch.uint8, device="cuda")
        d_ang = torch.empty((m, 3), dtype=torch.float32, device="cuda")
        L = whenet._L
        check(L.whenet_crop_resize_u8(whenet._h, _ptr(d_frame), H, W, 1, _ptr(rects), m, 1, _ptr(d_crops)))
        for off in range(0, m, whenet.max_batch):
            nb = min(whenet.max_batch, m - off)
            check(L.whenet_forward_u8(whenet._h, _ptr(d_crops[off:off + nb]), nb, 1, _ptr(d_ang[off:off + nb]), None, 1))
        whenet.synchronize()
        return boxes, scores, d_ang.cpu().numpy()
