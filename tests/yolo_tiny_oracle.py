"""CPU restatements of tiny YOLOv3 (reference yolo_v3/model.py:92-122, 199), built on oracle/yolo_oracle.py's conv, letterbox
and float32 decode + NMS:

* ``maxpool_same``: MaxPooling2D(pool_size=2, padding='same') in float64 numpy, the padding -inf so it never wins.
* ``body_numpy``: the 13 convs one layer at a time (``layer_inputs`` pools where a conv pools), so a test can feed a layer
  the GPU's own input; ``body_torch``: an independent torch-CPU restatement (F.pad(value=-inf) + F.max_pool2d, F.pad +
  F.conv2d, F.interpolate for the upsample).
* ``decode``: yolo_boxes_and_scores of the two heads with ``anchor_mask`` [[3,4,5],[1,2,3]] (model.py:199), through
  yolo_oracle.decode.
"""
import numpy as np

import yolo_oracle as O
from whenet_b200 import yolo_arch as Y


def maxpool_same(x, stride):
    """MaxPooling2D(pool_size=2, strides=stride, padding='same') of x (n,H,W,C) in float64: TF's SAME output size ceil(H/s),
    the padding (-inf) all at the bottom / right."""
    x = np.asarray(x, np.float64)
    n, H, W, C = x.shape
    Ho, Wo = -(-H // stride), -(-W // stride)
    xp = np.pad(x, ((0, 0), (0, (Ho - 1) * stride + 2 - H), (0, (Wo - 1) * stride + 2 - W), (0, 0)), constant_values=-np.inf)
    win = [xp[:, dy:dy + stride * (Ho - 1) + 1:stride, dx:dx + stride * (Wo - 1) + 1:stride] for dy in (0, 1) for dx in (0, 1)]
    return np.max(np.stack(win), axis=0)


def layer_inputs(i, outs, image):
    """(x, up) of tiny conv i given the outputs so far, x max-pooled where the conv pools."""
    L = Y.TINY_LAYERS[i]
    x = image if L.src < 0 else outs[L.src]
    if L.pool:
        x = maxpool_same(x, L.pool)
    return x, (outs[L.up] if L.up is not None else None)


def body_numpy(image, layers, dtype=np.float64):
    """All 13 outputs for ``image`` (n,H,W,3) float in [0,1]; ``layers`` from yolo_arch.map_weights(..., tiny=True), BN applied
    as Keras does."""
    outs = []
    for i, (L, d) in enumerate(zip(Y.TINY_LAYERS, layers)):
        x, up = layer_inputs(i, outs, image)
        bn = (d["gamma"], d["beta"], d["moving_mean"], d["moving_variance"]) if L.bn else None
        outs.append(O.conv_layer(x, d["kernel"], d.get("bias"), L.k, L.stride, L.bn, None, up, bn=bn, dtype=dtype))
    return outs


def body_torch(image, layers):
    """Independent torch-CPU float64 restatement (NCHW): the two head outputs, NHWC."""
    import torch
    import torch.nn.functional as F
    outs = []
    img = torch.from_numpy(np.asarray(image, np.float64)).permute(0, 3, 1, 2)
    for L, d in zip(Y.TINY_LAYERS, layers):
        x = img if L.src < 0 else outs[L.src]
        if L.pool:
            h, w = x.shape[2:]
            ph, pw = (-(-h // L.pool) - 1) * L.pool + 2 - h, (-(-w // L.pool) - 1) * L.pool + 2 - w
            x = F.max_pool2d(F.pad(x, (0, pw, 0, ph), value=-np.inf), 2, stride=L.pool)
        if L.up is not None:
            x = torch.cat([F.interpolate(outs[L.up], scale_factor=2, mode="nearest"), x], dim=1)
        if L.k == 3:
            x = F.pad(x, (1, 1, 1, 1))
        w = torch.from_numpy(np.asarray(d["kernel"], np.float64)).permute(3, 2, 0, 1)
        y = F.conv2d(x, w, torch.from_numpy(np.asarray(d["bias"], np.float64)) if not L.bn else None)
        if L.bn:
            t = [torch.from_numpy(np.asarray(d[k], np.float64)) for k in ("moving_mean", "moving_variance", "gamma", "beta")]
            y = F.batch_norm(y, t[0], t[1], t[2], t[3], training=False, eps=Y.BN_EPS)
            y = F.leaky_relu(y, Y.LEAKY)
        outs.append(y)
    return [outs[i].permute(0, 2, 3, 1).numpy() for i in Y.TINY_HEADS]


def decode(heads, anchors, num_classes, img_h, img_w):
    """yolo_boxes_and_scores for the two heads of ONE frame (candidates ordered layer 0, 1 then (y, x, anchor)): yolo_oracle's
    float32 decode with the anchors placed where its three-head mask reads them, so head l sees TINY_ANCHOR_MASK[l]."""
    assert len(heads) == 2
    a = np.asarray(anchors, np.float64).reshape(6, 2)
    slots = np.zeros((9, 2))
    for l in range(2):
        slots[Y.ANCHOR_MASK[l]] = a[Y.TINY_ANCHOR_MASK[l]]
    return O.decode(heads, slots, num_classes, img_h, img_w)
