"""YOLOv3 head-detector network description (reference ``yolo_v3/model.py:20-90``), shared by the weight loader, the
oracle, the bench and the tests.

The table lists the 75 convolutions in the order Keras ``load_weights`` consumes them: ``model.layers`` is sorted by
depth from the inputs, so the darknet chain and the three ``make_last_layers`` stacks come first and the three 3x3 convs
and three output convs of the heads last.  A conv reads the output of conv ``src`` (-1 = the letterboxed image); a concat
conv reads ``[upsample2x(out[up]), out[src]]`` (upsampled tensor first, model.py:81,87); ``res`` adds ``out[res]`` after
the LeakyReLU (resblock ``x + y``, model.py:46).  Stride-2 convs are ZeroPadding2D(((1,0),(1,0))) + VALID, every other
conv SAME: both are "pad 1 top/left" for a 3x3 kernel.

Tiny YOLOv3 (``tiny_yolo_body``, model.py:92-122; the reference builds it when the anchors file holds 6 anchors,
yolo_postprocess.py:71-79) is ``TINY_LAYERS``: 13 convs, all stride 1, six of them reading their source through a 2x2
max-pool (``pool``: 2 = stride 2, 1 = stride 1; MaxPooling2D padding 'same', so the stride-1 pool pads one row and column
at the bottom/right that never win the max).  Two heads, 13x13 and 26x26 at 416, decoded with ``TINY_ANCHOR_MASK``
(model.py:199; anchor 0 is never used).

Weight order of the tiny model.  Keras 2.1.6 ``load_weights`` walks ``model.layers``, which sorts the layers by decreasing
depth, the depth of a layer being its longest path to an output counting every layer (BatchNorm, LeakyReLU, pooling,
upsampling and concatenation included); layers at the same depth keep the order in which the walk back from
``outputs[0]``, then ``outputs[1]``, first met them.  The chain conv2d_1 .. conv2d_8 comes first.  Of the layers after
conv2d_8 (the 1x1 to 256), the 1x1 to 128 before the upsample is depth 8 (to ``y2``: BN, LeakyReLU, UpSampling2D,
Concatenate, conv, BN, LeakyReLU, output conv), the 3x3 to 512 of ``y1`` and the 3x3 concat conv of ``y2`` are both depth
3 (``y1``'s first), and the two output convs depth 0 (``y1``'s first).  Conv and BatchNorm names number in creation order
(the order tiny_yolo_body builds them): the 3x3 to 512 is conv2d_9, ``y1``'s output conv conv2d_10, the 1x1 to 128
conv2d_11, the concat conv conv2d_12 and ``y2``'s output conv conv2d_13, so the weight order is conv2d_1 .. conv2d_8,
conv2d_11, conv2d_9, conv2d_12, conv2d_10, conv2d_13 and batch_normalization_1 .. 8, 10, 9, 11.  This order is derived,
not checked against a file Keras wrote.  Within each tie (conv2d_9 / conv2d_12, conv2d_10 / conv2d_13, and their
BatchNorms) the shapes differ, so a file in the other order is refused with a "kernel shape" or BatchNorm-shape
ValueError, never loaded wrongly.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

BN_EPS = 1e-3           # keras BatchNormalization default epsilon
LEAKY = 0.1             # model.py:35
ANCHOR_MASK = [[6, 7, 8], [3, 4, 5], [0, 1, 2]]     # model.py:199
TINY_ANCHOR_MASK = [[3, 4, 5], [1, 2, 3]]          # model.py:199, two heads
# the nine YOLOv3 COCO anchor clusters (w, h) of the YOLOv3 paper (Redmon & Farhadi 2018, section 2.3)
DEFAULT_ANCHORS = np.array([[10, 13], [16, 30], [33, 23], [30, 61], [62, 45], [59, 119], [116, 90], [156, 198], [373, 326]],
                           dtype=np.float64)
DEFAULT_CLASSES = ["head"]
MIN_SIZE, MAX_SIZE = 32, 608
LARGE_MAX_SIZE = 4096      # whenet_det_create_large: sides above MAX_SIZE up to this (DESIGN.md 8.6)


@dataclass(frozen=True)
class Conv:
    idx: int              # position in the table (= Keras weight order)
    k: int                # 1 or 3
    stride: int           # 1 or 2
    cin: int              # total input channels (concat: c_up + skip channels)
    cout: int             # 0 = the head's 3 * (5 + num_classes)
    bn: bool              # bias-free + BatchNorm + LeakyReLU; False: bias, linear (output convs)
    src: int              # conv whose output is the input (-1: image)
    res: Optional[int] = None
    up: Optional[int] = None      # concat: conv whose output is upsampled x2 and put first
    keras_id: int = 0     # creation number: conv2d_<keras_id> in a freshly built model
    head: Optional[int] = None    # output conv of head l (0: 13x13 at 416, 1: 26x26, 2: 52x52)
    pool: int = 0         # tiny: the input is out[src] max-pooled 2x2 with this stride (0: no pool)
    tiny: bool = False    # a TINY_LAYERS row

    @property
    def c_up(self) -> int:
        return 0 if self.up is None else table(self.tiny)[self.up].cout


def _build() -> List[Conv]:
    rows = []            # dicts in table order, keras_id filled afterwards

    def add(k, s, cin, cout, src, bn=True, res=None, up=None, head=None):
        rows.append(dict(idx=len(rows), k=k, stride=s, cin=cin, cout=cout, bn=bn, src=src, res=res, up=up, head=head))
        return len(rows) - 1

    # darknet_body (model.py:49-57)
    x = add(3, 1, 3, 32, -1)
    c = 32
    skips = {}
    for nf, nb in ((64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)):
        x = add(3, 2, c, nf, x)
        for _ in range(nb):
            y = add(1, 1, nf, nf // 2, x)
            x = add(3, 1, nf // 2, nf, y, res=x)
        c = nf
        skips[nf] = x
    # make_last_layers x-part (five convs) of each head plus the 1x1 before each upsample, in depth order
    last5 = []

    def five(x, cin, nf, up=None):
        x = add(1, 1, cin, nf, x, up=up)
        for _ in range(2):
            x = add(3, 1, nf, 2 * nf, x)
            x = add(1, 1, 2 * nf, nf, x)
        last5.append(x)
        return x

    x = five(x, 1024, 512)
    u = add(1, 1, 512, 256, x)
    x = five(skips[512], 256 + 512, 256, up=u)
    u = add(1, 1, 256, 128, x)
    five(skips[256], 128 + 256, 128, up=u)
    y3 = [add(3, 1, nf, 2 * nf, last5[i]) for i, nf in enumerate((512, 256, 128))]
    for i, t in enumerate(y3):
        add(1, 1, rows[t]["cout"], 0, t, bn=False, head=i)
    # creation numbers (conv2d_N): darknet 1-52, then per head: five convs, 3x3, output, and (heads 0, 1) the 1x1 before upsampling
    order = list(range(52))
    t = 52
    for h in range(3):
        order += list(range(t, t + 5)) + [69 + h, 72 + h]
        t += 5
        if h < 2:
            order.append(t)
            t += 1
    keras_id = {table_idx: i + 1 for i, table_idx in enumerate(order)}
    return [Conv(keras_id=keras_id[r["idx"]], **r) for r in rows]


def _build_tiny() -> List[Conv]:
    rows = []
    # (k, cin, cout, src, pool, up, head, keras_id)
    for k, cin, cout_, src, pool, up, head, kid in (
            (3, 3, 16, -1, 0, None, None, 1), (3, 16, 32, 0, 2, None, None, 2), (3, 32, 64, 1, 2, None, None, 3),
            (3, 64, 128, 2, 2, None, None, 4), (3, 128, 256, 3, 2, None, None, 5), (3, 256, 512, 4, 2, None, None, 6),
            (3, 512, 1024, 5, 1, None, None, 7), (1, 1024, 256, 6, 0, None, None, 8), (1, 256, 128, 7, 0, None, None, 11),
            (3, 256, 512, 7, 0, None, None, 9), (3, 128 + 256, 256, 4, 0, 8, None, 12), (1, 512, 0, 9, 0, None, 0, 10),
            (1, 256, 0, 10, 0, None, 1, 13)):
        rows.append(Conv(idx=len(rows), k=k, stride=1, cin=cin, cout=cout_, bn=head is None, src=src, up=up, keras_id=kid, head=head,
                         pool=pool, tiny=True))
    return rows


LAYERS: List[Conv] = _build()
N_CONV = len(LAYERS)                 # 75
HEADS = [L.idx for L in LAYERS if L.head is not None]          # the three output convs, head 0..2
SKIP_LAYERS = sorted({L.src for L in LAYERS if L.up is not None})

TINY_LAYERS: List[Conv] = _build_tiny()
TINY_N_CONV = len(TINY_LAYERS)       # 13
TINY_HEADS = [L.idx for L in TINY_LAYERS if L.head is not None]    # the two output convs, head 0, 1
TINY_POOLED = [L.idx for L in TINY_LAYERS if L.pool]               # convs whose input is max-pooled


def table(tiny: bool = False) -> List[Conv]:
    return TINY_LAYERS if tiny else LAYERS


def heads(tiny: bool = False) -> List[int]:
    return TINY_HEADS if tiny else HEADS


def anchor_mask(tiny: bool = False) -> List[List[int]]:
    return TINY_ANCHOR_MASK if tiny else ANCHOR_MASK


def head_channels(num_classes: int) -> int:
    return 3 * (5 + num_classes)


def cout(L: Conv, num_classes: int) -> int:
    return head_channels(num_classes) if L.head is not None else L.cout


def in_hw(h: int, w: int, tiny: bool = False) -> List[Tuple[int, int]]:
    """Input (height, width) of every conv for a (h, w) model input, after the max-pool of a tiny conv (TF SAME: ceil)."""
    ins, outs = [], []
    for L in table(tiny):
        ih, iw = (h, w) if L.src < 0 else outs[L.src]
        if L.pool:
            ih, iw = -(-ih // L.pool), -(-iw // L.pool)
        ins.append((ih, iw))
        outs.append((ih // L.stride, iw // L.stride))
    return ins


def out_hw(h: int, w: int, tiny: bool = False) -> List[Tuple[int, int]]:
    """Output (height, width) of every conv for a (h, w) input."""
    return [(ih // L.stride, iw // L.stride) for L, (ih, iw) in zip(table(tiny), in_hw(h, w, tiny))]


def check_size(h: int, w: int, max_size: int = MAX_SIZE) -> None:
    """ValueError unless h and w are multiples of 32 in [MIN_SIZE, max_size] (MAX_SIZE, or LARGE_MAX_SIZE for a detector made
    by whenet_det_create_large)."""
    for v in (h, w):
        if v is None:
            raise ValueError("model_image_size (None, None) (image-sized input) is not supported")
        if v % 32 or not MIN_SIZE <= v <= max_size:
            raise ValueError("model_image_size must be multiples of 32 in [%d, %d], got (%r, %r)" % (MIN_SIZE, max_size, h, w))


def macs_per_frame(h: int, w: int, num_classes: int = 1, tiny: bool = False) -> int:
    """Multiply-accumulates of the 75 (tiny: 13) convs for one (h, w) frame (the algorithmic count: no padding, no tile
    rounding, no pools)."""
    hw = out_hw(h, w, tiny)
    return sum(hw[i][0] * hw[i][1] * L.k * L.k * L.cin * cout(L, num_classes) for i, L in enumerate(table(tiny)))


def num_candidates(h: int, w: int, tiny: bool = False) -> int:
    return sum(3 * (h // 32 << l) * (w // 32 << l) for l in range(2 if tiny else 3))


def keras_names(L: Conv, bn_id: int) -> List[str]:
    """Tensor names of one conv (+ its BatchNorm) in a freshly built keras-yolo3 model."""
    if not L.bn:
        return ["conv2d_%d/kernel:0" % L.keras_id, "conv2d_%d/bias:0" % L.keras_id]
    return ["conv2d_%d/kernel:0" % L.keras_id] + ["batch_normalization_%d/%s:0" % (bn_id, s)
                                                 for s in ("gamma", "beta", "moving_mean", "moving_variance")]


def random_weights(seed: int = 0, num_classes: int = 1, tiny: bool = False) -> Tuple[List[str], "OrderedDict[str, np.ndarray]"]:
    """Seeded weights with keras-yolo3 names and shapes, in file order (layer_names, {name: float32}).

    Kernels are N(0, 1/fan_in) and BatchNorm statistics are randomised (gamma, beta, mean, var all away from the identity) so
    that BN folding is exercised; with the 0.5 kernel gain of the residual branches the activations stay O(1) through all 75
    layers.  Output-conv kernels are small and their biases zero: head logits near 0, scores sigmoid * sigmoid near 0.25."""
    rng = np.random.default_rng(seed)
    bn_ids = _bn_ids(tiny)
    names: List[str] = []
    w: "OrderedDict[str, np.ndarray]" = OrderedDict()
    convs, bns = [], []
    for L in table(tiny):
        co = cout(L, num_classes)
        fan_in = L.k * L.k * L.cin
        gain = 0.5 if (L.res is not None) else 1.0
        std = (0.1 if not L.bn else gain) / np.sqrt(fan_in)
        kname, *rest = keras_names(L, bn_ids.get(L.idx, 0))
        kern = (rng.standard_normal((L.k, L.k, L.cin, co)) * std).astype(np.float32)
        convs.append((kname.split("/")[0], {kname: kern}))
        if L.bn:
            g = rng.uniform(0.8, 1.6, co)
            b = rng.uniform(-0.2, 0.2, co)
            m = rng.normal(0.0, 0.2, co)
            v = rng.uniform(0.5, 1.5, co)
            bns.append((rest[0].split("/")[0], dict(zip(rest, [a.astype(np.float32) for a in (g, b, m, v)]))))
        else:
            convs[-1][1][rest[0]] = np.zeros((co,), np.float32)
    # file order: every conv directly followed by its BatchNorm (the relative order of each kind is what matters, see _classify)
    bn_iter = iter(bns)
    for L, (cn, cw) in zip(table(tiny), convs):
        names.append(cn)
        w.update(cw)
        if L.bn:
            bn_name, bw = next(bn_iter)
            names.append(bn_name)
            w.update(bw)
    return names, w


def _bn_ids(tiny: bool = False) -> Dict[int, int]:
    """batch_normalization_<id> of every BN conv: BN layers are numbered in creation order like the convs."""
    by_creation = sorted((L for L in table(tiny) if L.bn), key=lambda L: L.keras_id)
    return {L.idx: i + 1 for i, L in enumerate(by_creation)}


_BN_KEYS = ("gamma", "beta", "moving_mean", "moving_variance")


def _classify(layer_names: List[str], weights: Dict[str, np.ndarray]):
    """Group tensors by layer (``<layer>/<weight>:0``) in file order; split the layers that carry weights into convs
    (kernel [+ bias]) and BatchNorms (gamma, beta, moving_mean, moving_variance)."""
    groups: "OrderedDict[str, Dict[str, np.ndarray]]" = OrderedDict()
    for name, a in weights.items():
        lname, _, wn = name.partition("/")
        groups.setdefault(lname, {})[wn.split(":")[0]] = a
    order = [n for n in layer_names if n in groups] if layer_names else list(groups)
    order += [n for n in groups if n not in order]
    convs, bns = [], []
    for lname in order:
        g = groups[lname]
        if set(g) <= {"kernel", "bias"} and "kernel" in g:
            convs.append((lname, g))
        elif set(g) == set(_BN_KEYS):
            bns.append((lname, g))
        else:
            raise ValueError("layer %s: unexpected weights %s for a YOLOv3 body" % (lname, sorted(g)))
    return convs, bns


def map_weights(layer_names: List[str], weights: Dict[str, np.ndarray], tiny: bool = False):
    """File tensors -> per-table-layer dicts {kernel, bias | gamma, beta, moving_mean, moving_variance, name}.

    Layers are matched by ORDER among the layers that carry weights (what Keras ``load_weights`` does), convs and
    BatchNorms each in their own sequence, never by name: the conv2d_<N> numbering depends on the session that built the
    model.  ``tiny``: the file is a tiny YOLOv3 (TINY_LAYERS).  Returns (layers, num_classes).  Anything that does not fit
    the table raises ValueError naming the layer or the count."""
    T = table(tiny)
    net = "tiny YOLOv3 (6 anchors)" if tiny else "YOLOv3 (9 anchors)"
    convs, bns = _classify(layer_names, weights)
    if len(convs) != len(T):
        raise ValueError("expected %d conv layers for %s, the file has %d" % (len(T), net, len(convs)))
    n_bn = sum(L.bn for L in T)
    if len(bns) != n_bn:
        raise ValueError("expected %d BatchNormalization layers for %s, the file has %d" % (n_bn, net, len(bns)))
    h0 = heads(tiny)[0]
    hc = convs[h0][1]["kernel"].shape[-1] if convs[h0][1]["kernel"].ndim == 4 else -1
    if hc < 18 or hc % 3 or (hc // 3 - 5) < 1:
        raise ValueError("layer %s: output conv has %d channels, not 3 * (5 + classes)" % (convs[h0][0], hc))
    num_classes = hc // 3 - 5
    out = []
    bn_iter = iter(bns)
    for L, (cname, g) in zip(T, convs):
        co = cout(L, num_classes)
        want = (L.k, L.k, L.cin, co)
        if tuple(g["kernel"].shape) != want:
            raise ValueError("layer %s (conv %d): kernel shape %s, expected %s" % (cname, L.idx, tuple(g["kernel"].shape), want))
        d = {"name": cname, "kernel": np.asarray(g["kernel"], np.float32)}
        if L.bn:
            if "bias" in g:
                raise ValueError("layer %s (conv %d): has a bias, expected a bias-free conv followed by BatchNorm" % (cname, L.idx))
            bname, bg = next(bn_iter)
            for key in _BN_KEYS:
                if tuple(bg[key].shape) != (co,):
                    raise ValueError("layer %s (BN of conv %d): %s has shape %s, expected (%d,)" % (bname, L.idx, key, tuple(bg[key].shape), co))
                d[key] = np.asarray(bg[key], np.float32)
        else:
            if "bias" not in g or tuple(g["bias"].shape) != (co,):
                raise ValueError("layer %s (output conv %d): needs a bias of shape (%d,)" % (cname, L.idx, co))
            d["bias"] = np.asarray(g["bias"], np.float32)
        out.append(d)
    return out, num_classes


def fold_bn(d: Dict[str, np.ndarray], bn: bool = True):
    """One mapped layer -> (kernel [k,k,cin,cout], bias [cout]) in float64 with BatchNorm folded in (eps 1e-3); the
    library folds the same way in double before its single rounding of the kernel to bf16."""
    k = np.asarray(d["kernel"], np.float64)
    if "gamma" not in d:
        return k, np.asarray(d["bias"], np.float64)
    s = np.asarray(d["gamma"], np.float64) / np.sqrt(np.asarray(d["moving_variance"], np.float64) + BN_EPS)
    return k * s, np.asarray(d["beta"], np.float64) - np.asarray(d["moving_mean"], np.float64) * s


def bf16_round(a) -> np.ndarray:
    """float -> float32 -> bf16 (round to nearest even), returned as float32 (the kernels' operand rounding)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def read_anchors(path) -> np.ndarray:
    """The reference's anchors file format (yolo_postprocess.py:59-64): one line of comma-separated numbers."""
    with open(path) as f:
        line = f.readline()
    return np.array([float(x) for x in line.split(",")]).reshape(-1, 2)


def read_classes(path) -> List[str]:
    """yolo_postprocess.py:52-57"""
    with open(path) as f:
        return [c.strip() for c in f.readlines()]
