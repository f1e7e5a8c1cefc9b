"""Integer numpy restatement of OpenCV's cv2.cvtColor(buf, cv2.COLOR_YUV2BGR_NV12) / COLOR_YUV2BGR_I420, the conversion the
detector's letterbox and the crop kernel apply to each YUV 4:2:0 pixel they read (csrc/yuv.cuh).

``buf`` is cv2's layout: an (H * 3/2, W) uint8 array, H and W even.  Rows [0, H) are the Y plane.  NV12: rows [H, H * 3/2) are
(H/2) x W interleaved (U, V) pairs, U first.  I420: the bytes after the Y plane are the (H/2) x (W/2) U plane, then the
(H/2) x (W/2) V plane.  Pixel (y, x) takes Y at (y, x) and U, V at (y/2, x/2) of their planes.

BT.601 limited range in 20-bit fixed point (OpenCV's YUV420sp / YUV420p to RGB8 converters):

    u = U - 128, v = V - 128, c = max(0, Y - 16) * 1220542
    B = clip8((c + 2^19 + 2116026 u) >> 20)
    G = clip8((c + 2^19 - 409993 u - 852492 v) >> 20)
    R = clip8((c + 2^19 + 1673527 v) >> 20)
"""
import numpy as np

LAYOUTS = ("nv12", "i420")


def planes(buf, layout):
    """(Y (H, W), U (H/2, W/2), V (H/2, W/2)) uint8 views of a cv2-layout 4:2:0 frame."""
    buf = np.asarray(buf)
    if buf.dtype != np.uint8 or buf.ndim != 2 or buf.shape[0] % 3 or buf.shape[1] % 2:
        raise ValueError("a 4:2:0 frame is (H * 3/2, W) uint8 with H, W even, not %s %s" % (buf.dtype, buf.shape))
    H, W = buf.shape[0] // 3 * 2, buf.shape[1]
    y = buf[:H]
    if layout == "nv12":
        uv = buf[H:].reshape(H // 2, W // 2, 2)
        return y, uv[..., 0], uv[..., 1]
    if layout == "i420":
        c = buf[H:].reshape(-1)
        q = (H // 2) * (W // 2)
        return y, c[:q].reshape(H // 2, W // 2), c[q:].reshape(H // 2, W // 2)
    raise ValueError("layout must be one of %s, not %r" % (LAYOUTS, layout))


def yuv420_to_bgr(buf, layout):
    """cv2.cvtColor(buf, COLOR_YUV2BGR_NV12 / COLOR_YUV2BGR_I420) -> (H, W, 3) uint8 BGR, in int64 integer arithmetic."""
    y, u, v = planes(buf, layout)
    up = lambda p: np.repeat(np.repeat(p.astype(np.int64) - 128, 2, axis=0), 2, axis=1)
    u, v = up(u), up(v)
    c = np.maximum(y.astype(np.int64) - 16, 0) * 1220542 + (1 << 19)
    b = (c + 2116026 * u) >> 20
    g = (c - 409993 * u - 852492 * v) >> 20
    r = (c + 1673527 * v) >> 20
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def bgr_to_yuv420(bgr, layout):
    """A 4:2:0 frame in cv2's layout whose Y plane is the BT.601 luma of ``bgr`` and whose chroma is its 2x2 mean, so the
    converted frame looks like ``bgr`` (test scenes with structure a detector responds to).  H and W must be even."""
    f = np.asarray(bgr, np.float64)
    H, W = f.shape[:2]
    b, g, r = f[..., 0], f[..., 1], f[..., 2]
    yy = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
    cb = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
    cr = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
    sub = lambda p: p.reshape(H // 2, 2, W // 2, 2).mean(axis=(1, 3))
    q = lambda p: np.clip(np.rint(p), 0, 255).astype(np.uint8)
    yq, uq, vq = q(yy), q(sub(cb)), q(sub(cr))
    if layout == "nv12":
        chroma = np.stack([uq, vq], axis=-1).reshape(H // 2, W)
    elif layout == "i420":
        chroma = np.concatenate([uq.reshape(-1), vq.reshape(-1)]).reshape(H // 2, W)
    else:
        raise ValueError("layout must be one of %s, not %r" % (LAYOUTS, layout))
    return np.ascontiguousarray(np.concatenate([yq, chroma], axis=0))
