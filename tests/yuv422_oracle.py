"""Integer numpy restatement of OpenCV's cv2.cvtColor(buf, cv2.COLOR_YUV2BGR_YUYV) / COLOR_YUV2BGR_UYVY, the conversion the
detector's letterbox, the crop kernel and the frame conversion kernel apply to each packed YUV 4:2:2 pixel they read
(csrc/yuv.cuh), and a scene maker for such frames.

``buf`` is an (H, W, 2) uint8 array, W even, any H.  Each row is W/2 pixel pairs of 4 bytes, Y0 U Y1 V (YUYV) or U Y0 V Y1
(UYVY); both pixels of a pair take its U and V.  The arithmetic is that of oracle/yuv_oracle.py (OpenCV's YUV422 to RGB8
converter: BT.601 limited range in 20-bit fixed point).
"""
import numpy as np

LAYOUTS_422 = ("yuyv", "uyvy")


def planes422(buf, layout):
    """(Y (H, W), U (H, W/2), V (H, W/2)) uint8 views of a packed 4:2:2 frame (H, W, 2)."""
    buf = np.asarray(buf)
    if buf.dtype != np.uint8 or buf.ndim != 3 or buf.shape[2] != 2 or buf.shape[0] < 1 or buf.shape[1] < 2 or buf.shape[1] % 2:
        raise ValueError("a 4:2:2 frame is (H, W, 2) uint8 with W even, not %s %s" % (buf.dtype, buf.shape))
    H, W = buf.shape[:2]
    q = buf.reshape(H, W // 2, 4)
    if layout == "yuyv":
        return buf[..., 0], q[..., 1], q[..., 3]
    if layout == "uyvy":
        return buf[..., 1], q[..., 0], q[..., 2]
    raise ValueError("layout must be one of %s, not %r" % (LAYOUTS_422, layout))


def yuv422_to_bgr(buf, layout):
    """cv2.cvtColor(buf, COLOR_YUV2BGR_YUYV / COLOR_YUV2BGR_UYVY) -> (H, W, 3) uint8 BGR, in int64 integer arithmetic."""
    y, u, v = planes422(buf, layout)
    u = np.repeat(u.astype(np.int64) - 128, 2, axis=1)
    v = np.repeat(v.astype(np.int64) - 128, 2, axis=1)
    c = np.maximum(y.astype(np.int64) - 16, 0) * 1220542 + (1 << 19)
    b = (c + 2116026 * u) >> 20
    g = (c - 409993 * u - 852492 * v) >> 20
    r = (c + 1673527 * v) >> 20
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def bgr_to_yuv422(bgr, layout):
    """A packed 4:2:2 frame (H, W, 2) whose Y is the BT.601 luma of ``bgr`` and whose chroma is the mean of each horizontal
    pixel pair, so the converted frame looks like ``bgr`` (test scenes with structure a detector responds to).  W must be
    even."""
    f = np.asarray(bgr, np.float64)
    H, W = f.shape[:2]
    b, g, r = f[..., 0], f[..., 1], f[..., 2]
    yy = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
    cb = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
    cr = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
    sub = lambda p: p.reshape(H, W // 2, 2).mean(axis=2)
    q = lambda p: np.clip(np.rint(p), 0, 255).astype(np.uint8)
    yq, uq, vq = q(yy).reshape(H, W // 2, 2), q(sub(cb)), q(sub(cr))
    if layout == "yuyv":
        quad = np.stack([yq[..., 0], uq, yq[..., 1], vq], axis=-1)
    elif layout == "uyvy":
        quad = np.stack([uq, yq[..., 0], vq, yq[..., 1]], axis=-1)
    else:
        raise ValueError("layout must be one of %s, not %r" % (LAYOUTS_422, layout))
    return np.ascontiguousarray(quad.reshape(H, W, 2))
