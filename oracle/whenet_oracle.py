"""CPU oracle for the WHENet per-crop forward.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
legs may import this module; it is the checker, never the product path.

**Parity unpinned.**  The arithmetic of the reference's hot path lives in
third-party packages that are not under ``/root/reference`` and cannot be
installed here (``efficientnet==0.0.4``, ``keras==2.1.6``,
``tensorflow-gpu==1.12.0``; reference ``requirements.txt:3-5``), and the
reference stores no expected angles anywhere (SURVEY.md section 4, 8c).  This
file therefore *restates* that arithmetic from (a) the reference's own call
sites and (b) the published definition of those packages, and is anchored on
the one artefact the reference does ship: the tensor names / shapes / order of
``WHENet.h5``.  The golden angles in ``tests/golden/golden.json`` were produced
by this oracle in float64 (script: ``tools/make_golden.py``), not by Keras.

Restated pieces and where they come from
----------------------------------------
* graph order        - ``layer_names`` root attribute of WHENet.h5, walked
                       one layer at a time exactly as ``Model.load_weights``
                       binds them (reference ``whenet.py:8-16``)
* preprocessing      - reference ``whenet.py:23-26``  (``img/255``; ``(img-mean)/std`` in float64)
* predict            - reference ``whenet.py:27``     (three logit arrays)
* softmax            - reference ``utils.py:7-11``
* expectation decode - reference ``whenet.py:31-33``
* package constants  - efficientnet==0.0.4 (public): every conv ``padding='same'``
                       (TensorFlow asymmetric rule), ``use_bias=False`` except the
                       two SE convs, BatchNorm ``epsilon=1e-3`` with moving statistics,
                       ``swish(x)=x*sigmoid(x)``, SE = mean over H,W (keepdims) ->
                       conv+bias -> swish -> conv+bias -> sigmoid -> multiply,
                       DropConnect = identity at inference, residual add iff the
                       ``add_k`` layer is present.  Depthwise strides (2 for
                       depthwise_conv2d_2/4/6/12, else 1) and the stride-2 stem come
                       from the B0 table; they are the only structural facts not
                       recoverable from the file.

This interpreter deliberately does NOT import the product's ``arch.py``: it
re-derives the graph from the file's layer list so a wrong block table in the
product cannot cancel out in the comparison.
"""
from __future__ import annotations

import re
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

MEAN = (0.485, 0.456, 0.406)   # reference whenet.py:23
STD = (0.229, 0.224, 0.225)    # reference whenet.py:24
BN_EPS = 1e-3
DW_STRIDE2 = {2, 4, 6, 12}     # EfficientNet-B0: first block of stages 2,3,4,6


# ----------------------------------------------------------------------------- primitives
def _same_pad(n_in: int, k: int, s: int, symmetric: bool = False) -> Tuple[int, int, int]:
    """(n_out, pad_before, pad_after).  Default: TensorFlow 'SAME' (out = ceil(in/s), the odd pad element goes AFTER).
    ``symmetric`` = the PyTorch-style (k-1)//2 on both sides: the WRONG rule for this network, kept only so the tests
    can prove that the padding convention matters (SURVEY.md 8c: 16.6 deg on the Sample crops)."""
    if symmetric:
        p = (k - 1) // 2
        return (n_in + 2 * p - k) // s + 1, p, p
    n_out = -(-n_in // s)
    total = max((n_out - 1) * s + k - n_in, 0)
    return n_out, total // 2, total - total // 2


def _sigmoid(x):
    with np.errstate(over="ignore"):      # exp(+large) -> inf -> 1/inf = 0, the correct limit
        return 1.0 / (1.0 + np.exp(-x))


def swish(x):
    return x * _sigmoid(x)


def conv2d_same(x: np.ndarray, w: np.ndarray, stride: int, symmetric_pad: bool = False) -> np.ndarray:
    """NHWC conv with HWIO kernel, TF 'SAME' padding, no bias."""
    n, h, wd, cin = x.shape
    kh, kw, _ci, cout = w.shape
    if kh == 1 and kw == 1 and stride == 1:
        return (x.reshape(-1, cin) @ w.reshape(cin, cout)).reshape(n, h, wd, cout)
    ho, pt, pb = _same_pad(h, kh, stride, symmetric_pad)
    wo, pl, pr = _same_pad(wd, kw, stride, symmetric_pad)
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    out = np.zeros((n, ho, wo, cout), dtype=x.dtype)
    for i in range(kh):
        for j in range(kw):
            patch = xp[:, i:i + (ho - 1) * stride + 1:stride, j:j + (wo - 1) * stride + 1:stride, :]
            out += (patch.reshape(-1, cin) @ w[i, j]).reshape(n, ho, wo, cout)
    return out


def depthwise_same(x: np.ndarray, w: np.ndarray, stride: int, symmetric_pad: bool = False) -> np.ndarray:
    """NHWC depthwise conv, kernel [kh,kw,C,1], TF 'SAME' padding."""
    n, h, wd, c = x.shape
    kh, kw = w.shape[:2]
    ho, pt, pb = _same_pad(h, kh, stride, symmetric_pad)
    wo, pl, pr = _same_pad(wd, kw, stride, symmetric_pad)
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    out = np.zeros((n, ho, wo, c), dtype=x.dtype)
    for i in range(kh):
        for j in range(kw):
            out += xp[:, i:i + (ho - 1) * stride + 1:stride, j:j + (wo - 1) * stride + 1:stride, :] * w[i, j, :, 0]
    return out


def batchnorm(x, gamma, beta, mean, var, eps=BN_EPS):
    return (x - mean) / np.sqrt(var + eps) * gamma + beta


def softmax(x: np.ndarray) -> np.ndarray:
    """reference utils.py:7-11 (without mutating the caller's array)."""
    x = x - np.max(x, axis=1, keepdims=True)
    a = np.exp(x)
    b = np.sum(np.exp(x), axis=1, keepdims=True)
    return a / b


def preprocess(img: np.ndarray) -> np.ndarray:
    """reference whenet.py:23-26; numpy promotes to float64 exactly as there."""
    img = np.asarray(img)
    img = img / 255
    img = (img - np.array(MEAN)) / np.array(STD)
    return img


def decode(yaw_logits, pitch_logits, roll_logits):
    """reference whenet.py:17-20,28-33."""
    idx = np.arange(66, dtype=np.float32)
    idx_yaw = np.arange(120, dtype=np.float32)
    yaw = np.sum(softmax(yaw_logits) * idx_yaw, axis=1) * 3 - 180
    pitch = np.sum(softmax(pitch_logits) * idx, axis=1) * 3 - 99
    roll = np.sum(softmax(roll_logits) * idx, axis=1) * 3 - 99
    return yaw, pitch, roll


# ----------------------------------------------------------------------------- the graph walker
class Oracle:
    """Interprets WHENet.h5's layer list on the CPU.

    ``dtype`` selects the arithmetic type of the network body (``np.float64``
    for golden values, ``np.float32`` to mimic Keras/TF float32).
    ``bn_eps`` / ``symmetric_pad`` exist only so tests can prove the structural
    constants matter (wrong variants must move the angles, SURVEY.md 8c).
    """

    def __init__(self, layer_names: Sequence[str], weights: Dict[str, np.ndarray],
                 dtype=np.float64, bn_eps: float = BN_EPS, symmetric_pad: bool = False):
        self.layer_names = list(layer_names)
        self.dtype = np.dtype(dtype)
        self.bn_eps = bn_eps
        self.symmetric_pad = bool(symmetric_pad)
        self.w = {k: np.asarray(v, dtype=self.dtype) for k, v in weights.items()}

    # -- single layers -------------------------------------------------------
    def _bn(self, x, name):
        w = self.w
        return batchnorm(x, w[name + "/gamma:0"], w[name + "/beta:0"],
                         w[name + "/moving_mean:0"], w[name + "/moving_variance:0"], self.bn_eps)

    def forward_normalised(self, x: np.ndarray, taps: Optional[Dict[str, np.ndarray]] = None):
        """x: (N,224,224,3) already normalised -> [yaw(N,120), pitch(N,66), roll(N,66)] logits.

        This is ``self.model.predict`` of reference whenet.py:27.
        """
        x = np.asarray(x, dtype=self.dtype)
        if x.ndim != 4 or x.shape[1:] != (224, 224, 3):
            raise ValueError("expected input of shape (N,224,224,3), got %s" % (x.shape,))
        w = self.w
        block_in = None      # tensor a following add_k adds back
        se_src = None        # tensor the SE gate multiplies
        blk = 0
        pooled = None
        outs = {}
        names = self.layer_names
        for pos, name in enumerate(names):
            m = re.match(r"([a-z_0-9]+?)_(\d+)$", name)
            kind, num = (m.group(1), int(m.group(2))) if m else (name, 0)
            if kind == "input":
                continue
            if kind == "conv2d":
                k = w[name + "/kernel:0"]
                if se_src is not None:
                    # inside the SE branch: 1x1 conv with bias on the (N,1,1,C) pooled tensor
                    x = conv2d_same(x, k, 1) + w[name + "/bias:0"]
                else:
                    x = conv2d_same(x, k, 2 if num == 1 else 1, self.symmetric_pad)   # only the stem conv strides
            elif kind == "batch_normalization":
                x = self._bn(x, name)
            elif kind == "swish":
                x = swish(x)
                if taps is not None and num == 1:
                    taps["stem"] = x.copy()
            elif kind == "depthwise_conv2d":
                x = depthwise_same(x, w[name + "/depthwise_kernel:0"], 2 if num in DW_STRIDE2 else 1, self.symmetric_pad)
            elif kind == "lambda":
                blk += 1
                if taps is not None:
                    taps["dw%d" % blk] = x.copy()
                se_src = x
                x = x.mean(axis=(1, 2), keepdims=True)
            elif kind == "activation":
                x = _sigmoid(x)
            elif kind == "multiply":
                if taps is not None:
                    taps["gate%d" % blk] = x.reshape(x.shape[0], -1).copy()
                x = se_src * x
                se_src = None
            elif kind == "drop_connect":
                pass  # identity at inference
            elif kind == "add":
                x = x + block_in
            elif kind == "global_average_pooling2d":
                if taps is not None:
                    taps["head"] = x.copy()
                pooled = x.mean(axis=(1, 2))
                x = pooled
                if taps is not None:
                    taps["pooled"] = pooled.copy()
            elif name in ("yaw_new", "pitch_new", "roll_new"):
                outs[name] = pooled @ w[name + "/kernel:0"] + w[name + "/bias:0"]
            else:
                raise ValueError("unknown layer %r in layer_names" % name)

            # ---- block bookkeeping: record block outputs / inputs ----
            # A block's output is the project BN (followed by add if present).  The next
            # block's input is that output.  We detect "project BN" as a BN whose next
            # layer is not a swish.
            if kind == "batch_normalization":
                nxt = names[pos + 1] if pos + 1 < len(names) else ""
                if not nxt.startswith("swish"):
                    if nxt.startswith("drop_connect"):
                        pass          # wait for the add
                    else:
                        if taps is not None:
                            taps["block%d" % blk] = x.copy()
                        block_in = x
            elif kind == "add":
                if taps is not None:
                    taps["block%d" % blk] = x.copy()
                block_in = x
            elif kind == "swish" and num == 1:
                block_in = x   # stem output feeds block 1 (never added: Cin != Cout)
        return [outs["yaw_new"], outs["pitch_new"], outs["roll_new"]]

    # -- one stage at a time -------------------------------------------------
    def stage_layers(self) -> Dict[str, object]:
        """The layer names of every stage, from the same ``layer_names`` walk as the forward.

        Returns ``{"stem": (conv, bn), "blocks": [ {expand: (conv, bn) | None, dw, dw_bn, stride, se: [conv, conv],
        proj, proj_bn, skip}, ... ], "head": (conv, bn)}``."""
        stem = head = pend = None
        blocks: List[dict] = []
        cur: Optional[dict] = None
        pend_conv = None
        in_se = 0
        for name in self.layer_names:
            m = re.match(r"([a-z_0-9]+?)_(\d+)$", name)
            kind, num = (m.group(1), int(m.group(2))) if m else (name, 0)
            if kind == "conv2d":
                if in_se:
                    cur["se"].append(name)
                    in_se -= 1
                elif cur is not None and cur["proj"] is None:
                    cur["proj"] = name
                else:
                    pend_conv = name
            elif kind == "batch_normalization":
                if stem is None:
                    stem, pend_conv = (pend_conv, name), None
                elif cur is not None and cur["proj"] is not None and cur["proj_bn"] is None:
                    cur["proj_bn"] = name
                elif cur is not None and cur["dw_bn"] is None:
                    cur["dw_bn"] = name
                else:
                    pend, pend_conv = (pend_conv, name), None
            elif kind == "depthwise_conv2d":
                cur = {"expand": pend, "dw": name, "dw_bn": None, "stride": 2 if num in DW_STRIDE2 else 1,
                       "se": [], "proj": None, "proj_bn": None, "skip": False}
                blocks.append(cur)
                pend = None
            elif kind == "lambda":
                in_se = 2
            elif kind == "add":
                cur["skip"] = True
        head = pend
        return {"stem": stem, "blocks": blocks, "head": head}

    def _fold(self, conv: str, bn: str, kernel: str = "/kernel:0"):
        """BN folded into the preceding conv in float64: (kernel * scale, shift)."""
        w = self.w
        scale = w[bn + "/gamma:0"] / np.sqrt(w[bn + "/moving_variance:0"] + self.bn_eps)
        shift = w[bn + "/beta:0"] - w[bn + "/moving_mean:0"] * scale
        k = w[conv + kernel]
        return k * (scale if kernel == "/kernel:0" else scale[:, None]), shift

    def run_stage(self, stage: str, x: np.ndarray, block: int = 0, gate: Optional[np.ndarray] = None,
                  resid: Optional[np.ndarray] = None, symmetric_pad: Optional[bool] = None) -> Dict[str, np.ndarray]:
        """One stage of the network on a given input, every weight folded and applied in ``self.dtype``.

        Returns the stage's intermediate values and the matching sums of absolute terms (``S_*``), which an
        error bound of the same arithmetic in another precision needs.  NHWC throughout.

        * ``"stem"``:    x = normalised image (N,224,224,3) -> ``pre``, ``S``, ``out`` = swish(pre)
        * ``"dw"``:      x = block input (the stem output for block 1); ``block`` = 1..16 ->
                         [``pre_e``, ``S_e``, ``X_e`` (sum |x|), ``shift_e``, ``e``] for blocks with an expand conv, then
                         ``pre``, ``S`` (sum |e w|), ``X`` (sum |e| over the window), ``w`` (folded depthwise kernel,
                         (k,k,C)), ``shift``, ``out``
        * ``"gate"``:    x = depthwise output -> ``mean``, ``z1``, ``S_z1``, ``a``, ``z2``, ``S_z2``, ``w1``, ``w2``, ``out``
        * ``"project"``: x = depthwise output, ``gate`` (N,C), ``resid`` = block input or None -> ``pre``, ``S``,
                         ``X`` (sum |x g|), ``shift``, ``out``
        * ``"head"``:    x = block 16 output -> ``pre``, ``S``, ``X``, ``shift``, ``out``
        * ``"dense"``:   x = pooled features (N,1280) -> ``logits`` (three arrays), ``S`` (three arrays)
        """
        sym = self.symmetric_pad if symmetric_pad is None else bool(symmetric_pad)
        L = self.stage_layers()
        x = np.asarray(x, dtype=self.dtype)
        w = self.w
        r: Dict[str, np.ndarray] = {}
        if stage == "stem":
            conv, bn = L["stem"]
            k, sh = self._fold(conv, bn)
            r["pre"] = conv2d_same(x, k, 2, sym) + sh
            r["S"] = conv2d_same(np.abs(x), np.abs(k), 2, sym) + np.abs(sh)
            r["out"] = swish(r["pre"])
            return r
        if stage in ("dw", "gate", "project"):
            b = L["blocks"][block - 1]
        if stage == "dw":
            if b["expand"] is not None:
                k, sh = self._fold(*b["expand"])
                c = k.shape[-1]
                r["pre_e"] = x.reshape(-1, x.shape[-1]) @ k.reshape(-1, c) + sh
                r["S_e"] = np.abs(x).reshape(-1, x.shape[-1]) @ np.abs(k).reshape(-1, c)
                r["X_e"] = np.abs(x).sum(axis=-1).reshape(x.shape[:3] + (1,))
                r["pre_e"] = r["pre_e"].reshape(x.shape[:3] + (c,))
                r["S_e"] = r["S_e"].reshape(x.shape[:3] + (c,))
                r["shift_e"] = sh
                x = r["e"] = swish(r["pre_e"])
            k, sh = self._fold(b["dw"], b["dw_bn"], "/depthwise_kernel:0")
            r["w"] = k[:, :, :, 0]
            r["shift"] = sh
            r["pre"] = depthwise_same(x, k, b["stride"], sym) + sh
            r["S"] = depthwise_same(np.abs(x), np.abs(k), b["stride"], sym)
            r["X"] = depthwise_same(np.abs(x), np.ones_like(k), b["stride"], sym)
            r["out"] = swish(r["pre"])
            return r
        if stage == "gate":
            c1, c2 = b["se"]
            w1, b1 = w[c1 + "/kernel:0"][0, 0], w[c1 + "/bias:0"]
            w2, b2 = w[c2 + "/kernel:0"][0, 0], w[c2 + "/bias:0"]
            r["mean"] = x.mean(axis=(1, 2))
            r["z1"] = r["mean"] @ w1 + b1
            r["S_z1"] = np.abs(r["mean"]) @ np.abs(w1) + np.abs(b1)
            r["a"] = swish(r["z1"])
            r["z2"] = r["a"] @ w2 + b2
            r["S_z2"] = np.abs(r["a"]) @ np.abs(w2) + np.abs(b2)
            r["out"] = _sigmoid(r["z2"])
            r["w1"], r["w2"] = w1, w2
            return r
        if stage == "project":
            k, sh = self._fold(b["proj"], b["proj_bn"])
            k = k[0, 0]
            xg = x * gate[:, None, None, :]
            r["pre"] = (xg.reshape(-1, k.shape[0]) @ k).reshape(x.shape[:3] + (k.shape[1],)) + sh
            r["S"] = (np.abs(xg).reshape(-1, k.shape[0]) @ np.abs(k)).reshape(r["pre"].shape) + np.abs(sh)
            r["X"] = np.abs(xg).sum(axis=-1)[..., None]
            r["shift"] = sh
            r["out"] = r["pre"] + (resid if resid is not None else 0.0)
            return r
        if stage == "head":
            k, sh = self._fold(*L["head"])
            k = k[0, 0]
            r["pre"] = (x.reshape(-1, k.shape[0]) @ k).reshape(x.shape[:3] + (k.shape[1],)) + sh
            r["S"] = (np.abs(x).reshape(-1, k.shape[0]) @ np.abs(k)).reshape(r["pre"].shape)
            r["X"] = np.abs(x).sum(axis=-1)[..., None]
            r["shift"] = sh
            r["out"] = swish(r["pre"])
            return r
        if stage == "dense":
            names = ("yaw_new", "pitch_new", "roll_new")
            r["logits"] = [x @ w[n + "/kernel:0"] + w[n + "/bias:0"] for n in names]
            r["S"] = [np.abs(x) @ np.abs(w[n + "/kernel:0"]) + np.abs(w[n + "/bias:0"]) for n in names]
            return r
        raise ValueError("unknown stage %r" % stage)

    # -- the reference surface -----------------------------------------------
    def predict(self, img_normalised, taps=None):
        return self.forward_normalised(img_normalised, taps)

    def get_angle(self, img, taps=None, return_logits=False):
        """reference whenet.py:22-34 end to end (float64 preprocessing, then the net in ``dtype``)."""
        x = preprocess(img)
        if self.dtype == np.float32:
            x = x.astype(np.float32)     # Keras feeds float32 placeholders
        logits = self.forward_normalised(x, taps)
        yaw, pitch, roll = decode(*logits)
        out = (yaw.astype(np.float32), pitch.astype(np.float32), roll.astype(np.float32))
        if return_logits:
            return out, logits
        return out


def load_oracle(snapshot: str, dtype=np.float64, **kw) -> Oracle:
    """Build an oracle from a Keras ``.h5`` or a converted ``.npz`` (tools/convert_weights.py)."""
    import os, sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "..", "headposeestimation-whenet_b200"))
    try:
        import h5lite  # the weight *reader* is host plumbing shared with the product
    finally:
        sys.path.pop(0)
    if snapshot.endswith(".npz"):
        z = np.load(snapshot, allow_pickle=False)
        layer_names = [str(s) for s in z["__layer_names__"]]
        weights = {k: z[k] for k in z.files if not k.startswith("__")}
    else:
        layer_names, weights, _meta = h5lite.read_keras_weights(snapshot)
    return Oracle(layer_names, weights, dtype=dtype, **kw)


# ----------------------------------------------------------------------------- torch-CPU port (baseline timing only)
class TorchCpuPort:
    """The same graph on torch-CPU float32 (oneDNN convs, all host threads).

    Exists only so ``bench.py`` can time a *strong* CPU implementation next to
    the GPU numbers (``cpu_baseline.kind == "port"``): Keras/TF-1.12 cannot run
    here, and a numpy loop would flatter the GPU.  Drives the reference's own
    chunking, ``predict(batch_size=8)`` (reference whenet.py:27).
    """

    def __init__(self, layer_names, weights, threads: Optional[int] = None):
        import torch
        self.torch = torch
        if threads:
            torch.set_num_threads(threads)
        self.layer_names = list(layer_names)
        self.w = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)) for k, v in weights.items()}
        # pre-permute conv kernels HWIO -> OIHW once (not part of the timed path)
        self.k = {}
        for name, t in self.w.items():
            if name.endswith("/kernel:0") and t.dim() == 4:
                self.k[name] = t.permute(3, 2, 0, 1).contiguous()
            elif name.endswith("/depthwise_kernel:0"):
                self.k[name] = t.permute(2, 3, 0, 1).contiguous()   # [C,1,kh,kw]

    def _conv_same(self, x, wk, stride, groups=1):
        F = self.torch.nn.functional
        kh = wk.shape[2]
        h = x.shape[2]
        _o, pb, pa = _same_pad(h, kh, stride)
        if pb or pa:
            x = F.pad(x, (pb, pa, pb, pa))
        return F.conv2d(x, wk, None, stride, 0, 1, groups)

    def predict_chunk(self, x_nchw):
        torch = self.torch
        F = torch.nn.functional
        w, k = self.w, self.k
        x = x_nchw
        block_in = None
        se_src = None
        outs = {}
        names = self.layer_names
        for pos, name in enumerate(names):
            m = re.match(r"([a-z_0-9]+?)_(\d+)$", name)
            kind, num = (m.group(1), int(m.group(2))) if m else (name, 0)
            if kind == "input":
                continue
            if kind == "conv2d":
                if se_src is not None:
                    x = F.conv2d(x, k[name + "/kernel:0"], w[name + "/bias:0"])
                else:
                    x = self._conv_same(x, k[name + "/kernel:0"], 2 if num == 1 else 1)
            elif kind == "batch_normalization":
                x = F.batch_norm(x, w[name + "/moving_mean:0"], w[name + "/moving_variance:0"],
                                 w[name + "/gamma:0"], w[name + "/beta:0"], False, 0.0, BN_EPS)
                nxt = names[pos + 1]
                if not nxt.startswith("swish") and not nxt.startswith("drop_connect"):
                    block_in = x
            elif kind == "swish":
                x = x * torch.sigmoid(x)
                if num == 1:
                    block_in = x
            elif kind == "depthwise_conv2d":
                wk = k[name + "/depthwise_kernel:0"]
                x = self._conv_same(x, wk, 2 if num in DW_STRIDE2 else 1, groups=wk.shape[0])
            elif kind == "lambda":
                se_src = x
                x = x.mean(dim=(2, 3), keepdim=True)
            elif kind == "activation":
                x = torch.sigmoid(x)
            elif kind == "multiply":
                x = se_src * x
                se_src = None
            elif kind == "drop_connect":
                pass
            elif kind == "add":
                x = x + block_in
                block_in = x
            elif kind == "global_average_pooling2d":
                x = x.mean(dim=(2, 3))
            elif name in ("yaw_new", "pitch_new", "roll_new"):
                outs[name] = x @ w[name + "/kernel:0"] + w[name + "/bias:0"]
        return outs["yaw_new"], outs["pitch_new"], outs["roll_new"]

    def get_angle(self, img, batch_size: int = 8):
        torch = self.torch
        x = preprocess(img).astype(np.float32)                       # whenet.py:25-26
        ys, ps, rs = [], [], []
        with torch.no_grad():
            for i in range(0, x.shape[0], batch_size):                # whenet.py:27
                t = torch.from_numpy(x[i:i + batch_size]).permute(0, 3, 1, 2).contiguous()
                y, p, r = self.predict_chunk(t)
                ys.append(y.numpy()); ps.append(p.numpy()); rs.append(r.numpy())
        yaw, pitch, roll = decode(np.concatenate(ys), np.concatenate(ps), np.concatenate(rs))
        return yaw.astype(np.float32), pitch.astype(np.float32), roll.astype(np.float32)
