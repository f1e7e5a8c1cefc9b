"""CPU restatements of the YOLOv3 head detector (reference yolo_v3/), the yardsticks of the CUDA path.

* ``pil_resize_bicubic`` / ``letterbox``: numpy restatement of Pillow's uint8 BICUBIC resample (libImaging/Resample.c:
  precompute_coeffs, normalize_coeffs_8bpc, the horizontal then vertical 8-bit passes) and of ``letterbox_image``
  (reference utils.py:23-34).
* ``conv_layer`` / ``body_numpy``: the body (model.py:20-90) in float64 numpy, one layer at a time so a test can feed a
  layer the GPU's own input.  BatchNorm is applied as Keras does (unfolded) unless the layer carries folded (w, b).
* ``body_torch``: an independent torch-CPU restatement (F.pad + F.conv2d) to cross-check the numpy one.
* ``decode`` / ``nms_tf`` / ``yolo_eval``: float32 restatement of yolo_head, yolo_correct_boxes, the score mask and
  tf.image.non_max_suppression (model.py:125-232).
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from whenet_b200 import yolo_arch as Y  # noqa: E402

# ----------------------------------------------------------------------------------------------------------- letterbox
PRECISION_BITS = 22


def _bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _coeffs(in_size, out_size):
    scale = float(np.float32(in_size)) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        for x, w in enumerate(k):
            kk[xx, x] = int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _pass(img, bounds, kk, axis):
    """One 8-bit pass along ``axis`` (1: horizontal, 0: vertical) of an (H, W, 3) uint8 image."""
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((len(bounds),) + src.shape[1:], np.int64)
    for i, (xmin, cnt) in enumerate(bounds):
        s = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for j in range(cnt):
            s += src[xmin + j] * kk[i, j]
        out[i] = s
    out = np.clip(out >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out.astype(np.uint8), 0, axis)


def pil_resize_bicubic(img, nw, nh):
    """``PIL.Image.fromarray(img).resize((nw, nh), Image.BICUBIC)`` for an (H, W, 3) uint8 RGB array."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    if (nw, nh) == (W, H):
        return img.copy()
    bx, kx = _coeffs(W, nw)
    by, ky = _coeffs(H, nh)
    out = _pass(img, bx, kx, 1)
    return _pass(out, by, ky, 0)


def letterbox_geometry(iw, ih, w, h):
    """utils.py:25-29 and the paste offset of :33 (float64 scale, int() truncation)."""
    scale = min(w / iw, h / ih)
    nw, nh = int(iw * scale), int(ih * scale)
    return nw, nh, (w - nw) // 2, (h - nh) // 2


def letterbox(img, size):
    """``letterbox_image`` (utils.py:23-34) on an (H, W, 3) uint8 RGB array; ``size`` = (w, h).  Returns the uint8 canvas."""
    img = np.asarray(img, np.uint8)
    w, h = size
    nw, nh, ox, oy = letterbox_geometry(img.shape[1], img.shape[0], w, h)
    canvas = np.full((h, w, 3), 128, np.uint8)
    canvas[oy:oy + nh, ox:ox + nw] = pil_resize_bicubic(img, nw, nh)
    return canvas


# ----------------------------------------------------------------------------------------------------------- body
def _pad_top_left(x, k, stride):
    """SAME (stride 1) or ZeroPadding2D(((1,0),(1,0))) + VALID (stride 2): pad 1 at the top/left, and for stride 1 at the
    bottom/right too.  x: (n, H, W, C)."""
    if k == 1:
        return x
    after = 1 if stride == 1 else 0
    return np.pad(x, ((0, 0), (1, after), (1, after), (0, 0)))


def conv_layer(x, w, b=None, k=3, stride=1, leaky=True, resid=None, up=None, bn=None, dtype=np.float64):
    """One YOLOv3 conv in ``dtype``: x (n,H,W,C) (concat: the skip tensor, ``up`` (n,H/2,W/2,Cu) upsampled x2 and put first),
    w [k,k,Cin,Cout]; then ``b`` (folded bias) or ``bn`` = (gamma, beta, mean, var) applied as Keras does, LeakyReLU(0.1)
    unless ``leaky`` is False, then ``+ resid``."""
    x = np.asarray(x, dtype)
    if up is not None:
        u = np.asarray(up, dtype).repeat(2, axis=1).repeat(2, axis=2)
        x = np.concatenate([u, x], axis=3)
    n, H, W, _ = x.shape
    Ho, Wo = H // stride, W // stride
    xp = _pad_top_left(x, k, stride)
    w = np.asarray(w, dtype)
    out = np.zeros((n, Ho, Wo, w.shape[3]), dtype)
    for ky in range(k):
        for kx in range(k):
            patch = xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride, :]
            out += patch @ w[ky, kx]
    if bn is not None:
        g, be, m, v = (np.asarray(a, dtype) for a in bn)
        out = (out - m) / np.sqrt(v + dtype(Y.BN_EPS)) * g + be
    if b is not None:
        out = out + np.asarray(b, dtype)
    if leaky:
        out = np.where(out > 0, out, dtype(Y.LEAKY) * out)
    if resid is not None:
        out = out + np.asarray(resid, dtype)
    return out


def layer_inputs(i, outs, image):
    """(x, up, resid) of table layer i given the outputs so far."""
    L = Y.LAYERS[i]
    x = image if L.src < 0 else outs[L.src]
    return x, (outs[L.up] if L.up is not None else None), (outs[L.res] if L.res is not None else None)


def body_numpy(image, layers, folded=False, dtype=np.float64):
    """All 75 outputs for ``image`` (n,H,W,3) float in [0,1]; ``layers`` from yolo_arch.map_weights (folded=False: BN as Keras),
    or a list of (w, b) with BN already folded (folded=True)."""
    outs = []
    for i, L in enumerate(Y.LAYERS):
        x, up, res = layer_inputs(i, outs, image)
        if folded:
            w, b = layers[i]
            outs.append(conv_layer(x, w, b, L.k, L.stride, L.bn, res, up, dtype=dtype))
        else:
            d = layers[i]
            bn = (d["gamma"], d["beta"], d["moving_mean"], d["moving_variance"]) if L.bn else None
            outs.append(conv_layer(x, d["kernel"], d.get("bias"), L.k, L.stride, L.bn, res, up, bn=bn, dtype=dtype))
    return outs


def body_torch(image, layers):
    """Independent torch-CPU float64 restatement (F.pad + F.conv2d + batch_norm + leaky_relu, NCHW): the three head outputs,
    NHWC."""
    import torch
    import torch.nn.functional as F
    outs = []
    img = torch.from_numpy(np.asarray(image, np.float64)).permute(0, 3, 1, 2)
    for L, d in zip(Y.LAYERS, layers):
        x = img if L.src < 0 else outs[L.src]
        if L.up is not None:
            x = torch.cat([F.interpolate(outs[L.up], scale_factor=2, mode="nearest"), x], dim=1)
        if L.k == 3:
            x = F.pad(x, (1, 1, 1, 1) if L.stride == 1 else (1, 0, 1, 0))
        w = torch.from_numpy(np.asarray(d["kernel"], np.float64)).permute(3, 2, 0, 1)
        y = F.conv2d(x, w, torch.from_numpy(np.asarray(d["bias"], np.float64)) if not L.bn else None, stride=L.stride)
        if L.bn:
            t = [torch.from_numpy(np.asarray(d[k], np.float64)) for k in ("moving_mean", "moving_variance", "gamma", "beta")]
            y = F.batch_norm(y, t[0], t[1], t[2], t[3], training=False, eps=Y.BN_EPS)
            y = F.leaky_relu(y, Y.LEAKY)
        if L.res is not None:
            y = y + outs[L.res]
        outs.append(y)
    return [outs[i].permute(0, 2, 3, 1).numpy() for i in Y.HEADS]


# ----------------------------------------------------------------------------------------------------------- decode + NMS
f32 = np.float32


def _sigmoid(x):
    x = np.asarray(x, f32)
    return (f32(1) / (f32(1) + np.exp(-x))).astype(f32)


def correct_params(in_h, in_w, img_h, img_w):
    """yolo_correct_boxes' float32 letterbox size (K.round: half to even), offset and scale (model.py:157-161)."""
    inp = np.array([in_h, in_w], f32)
    img = np.array([img_h, img_w], f32)
    new = np.round(img * np.min(inp / img)).astype(f32)
    off = ((inp - new) / f32(2.0) / inp).astype(f32)
    scale = (inp / new).astype(f32)
    return off, scale


def decode(heads, anchors, num_classes, img_h, img_w):
    """yolo_boxes_and_scores for the three heads of ONE frame -> boxes (NC,4) float32 (y_min, x_min, y_max, x_max) and
    scores (NC, C), candidates ordered layer 0, 1, 2 then (y, x, anchor)."""
    gh0, gw0 = heads[0].shape[:2]
    in_h, in_w = gh0 * 32, gw0 * 32
    off, scale = correct_params(in_h, in_w, img_h, img_w)
    ch = 5 + num_classes
    all_b, all_s = [], []
    for l, h in enumerate(heads):
        gh, gw = h.shape[:2]
        t = np.asarray(h, f32).reshape(gh, gw, 3, ch)
        gx = np.arange(gw, dtype=f32)[None, :, None]
        gy = np.arange(gh, dtype=f32)[:, None, None]
        an = np.asarray(anchors, f32)[Y.ANCHOR_MASK[l]]
        bx = ((_sigmoid(t[..., 0]) + gx) / f32(gw)).astype(f32)
        by = ((_sigmoid(t[..., 1]) + gy) / f32(gh)).astype(f32)
        bw = (np.exp(t[..., 2]) * an[:, 0] / f32(in_w)).astype(f32)
        bh = (np.exp(t[..., 3]) * an[:, 1] / f32(in_h)).astype(f32)
        yc = ((by - off[0]) * scale[0]).astype(f32)
        xc = ((bx - off[1]) * scale[1]).astype(f32)
        hh = (bh * scale[0]).astype(f32)
        ww = (bw * scale[1]).astype(f32)
        hh2, ww2 = (hh / f32(2.0)).astype(f32), (ww / f32(2.0)).astype(f32)
        b = np.stack([(yc - hh2) * f32(img_h), (xc - ww2) * f32(img_w), (yc + hh2) * f32(img_h), (xc + ww2) * f32(img_w)], -1).astype(f32)
        s = (_sigmoid(t[..., 4:5]) * _sigmoid(t[..., 5:])).astype(f32)
        all_b.append(b.reshape(-1, 4))
        all_s.append(s.reshape(-1, num_classes))
    return np.concatenate(all_b), np.concatenate(all_s)


def iou_tf(a, b):
    """TF non_max_suppression IoU in float32: corners via min/max, 0 when either area <= 0."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    aymin, aymax = min(a[0], a[2]), max(a[0], a[2])
    axmin, axmax = min(a[1], a[3]), max(a[1], a[3])
    bymin, bymax = min(b[0], b[2]), max(b[0], b[2])
    bxmin, bxmax = min(b[1], b[3]), max(b[1], b[3])
    area_a = f32((aymax - aymin) * (axmax - axmin))
    area_b = f32((bymax - bymin) * (bxmax - bxmin))
    if area_a <= 0 or area_b <= 0:
        return f32(0)
    inter = f32(max(f32(min(aymax, bymax) - max(aymin, bymin)), f32(0)) * max(f32(min(axmax, bxmax) - max(axmin, bxmin)), f32(0)))
    return f32(inter / f32(f32(area_a + area_b) - inter))


def nms_tf(boxes, scores, max_output_size, iou_threshold):
    """tf.image.non_max_suppression: greedy in descending score (equal scores: lower index first), a box is suppressed when
    its IoU with a kept box is > the threshold (so a NaN IoU, of two boxes with infinite corners, suppresses nothing).
    Returns kept indices."""
    order = sorted(range(len(scores)), key=lambda i: (-float(scores[i]), i))
    keep = []
    for i in order:
        if len(keep) >= max_output_size:
            break
        if not any(iou_tf(boxes[i], boxes[j]) > f32(iou_threshold) for j in keep):
            keep.append(i)
    return keep


def yolo_eval(boxes, scores, score_threshold, iou_threshold, max_boxes=20):
    """model.py:211-232 for one frame: per class, mask score >= threshold, NMS, concatenate class by class.
    Returns (boxes, scores, classes, candidate indices)."""
    ob, os_, oc, oi = [], [], [], []
    for c in range(scores.shape[1]):
        idx = np.nonzero(scores[:, c] >= f32(score_threshold))[0]
        keep = nms_tf(boxes[idx], scores[idx, c], max_boxes, iou_threshold)
        sel = idx[keep]
        ob.append(boxes[sel]); os_.append(scores[sel, c]); oc.append(np.full(len(sel), c, np.int32)); oi.append(sel)
    return (np.concatenate(ob).reshape(-1, 4).astype(f32), np.concatenate(os_).astype(f32), np.concatenate(oc).astype(np.int32),
            np.concatenate(oi).astype(np.int64))
