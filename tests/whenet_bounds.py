"""Per-element error bounds of the WHENet kernels, derived from their arithmetic (DESIGN §2.1).

Each stage is compared on its own GPU input (the previous tap, which is exact: a float32 copy of the storage type),
so a bound only covers the rounding of the stage itself.  First-order terms; the tests assert |got - ref| <= 2 B, the
factor 2 standing for the second-order terms (products of two roundings, the derivative of swish / sigmoid taken at the
reference point instead of the GPU's).

Units: u_bf16 = 2^-8, u_fp16 = 2^-11, u_fp32 = 2^-24 (unit roundoff of round-to-nearest).  ``r`` is the dict of
``Oracle.run_stage`` for the stage (float64 values and sums of absolute terms S = sum |x w|).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from whenet_oracle import depthwise_same

U = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "fp32": 2.0 ** -24}
U32 = U["fp32"]
# tanh.approx.f32 (the 16-bit modes' swish h + h tanh(h), h = x/2): PTX documents a maximum error of about 2^-11; the model
# takes twice that.  The error of h * t is then <= EPS_TANH |h| = EPS_TANH |x| / 2, absolute: for x < 0 the two terms cancel
# and the output can be far smaller than the error.
EPS_TANH = 2.0 ** -10
SWISH_SLOPE = 1.1        # max |swish'(x)| = 1.0998
# split-bf16 operands of the fp32 tensor-core mode (pw_tc32_kernel): hi = bf16(x), lo = bf16(x - hi), product
# Ahi*Whi + Ahi*Wlo + Alo*Whi.  With u = 2^-8: |x - hi| <= u|x|, so |lo| <= u|x| and the residual |x - hi - lo| <= u|x - hi|
# <= u^2 |x|.  Writing x = hi + lo + rx, w = ... + rw, the kernel misses lo_x lo_w + rx (w_hi + w_lo) + rw (x_hi + x_lo):
# at most 3 u^2 = 3 * 2^-16 of |x w| (random pairs reach about 1.8 * 2^-16).
SPLIT = 3 * 2.0 ** -16
# fp16 weights below 2^-14 are subnormal: spacing 2^-24, rounding error <= 2^-25 absolute.  K1 stores 0.5 w, so in units of
# w the floor is 2^-24; the HFMA2 depthwise stores 0.5 w / kDwScale = w / 8, floor 8 * 2^-25 = 2^-22 in units of w.
FP16_W_FLOOR = 2.0 ** -24
FP16_DW_FLOOR = 2.0 ** -22
KDW = 4.0                # kDwScale (kernels_fused.cuh)


@dataclass(frozen=True)
class Arith:
    """What a route's kernels round, per family."""
    store: str           # activation storage type: "bf16" | "fp16" | "fp32"
    stem_store: str      # storage type of the stem output (fp16 in bf16 mode when block 1's depthwise is KD)
    weights: str         # 1x1-conv weights on the tensor core: "bf16" | "fp16" | "fp32" (CUDA cores) | "split" (bf16 hi + lo)
    dw: str              # depthwise of the blocks with an expand conv: "hfma2" (fp16 sums) | "ffma" (fp32)
    dw1: str             # depthwise of block 1 (its E tile is the stem output)

    @property
    def sixteen(self) -> bool:
        return self.store != "fp32"


BF16 = Arith("bf16", "fp16", "bf16", "hfma2", "hfma2")
FP16 = Arith("fp16", "fp16", "fp16", "ffma", "ffma")
FP32_CUDA = Arith("fp32", "fp32", "fp32", "ffma", "ffma")
FP32_SPLIT = Arith("fp32", "fp32", "split", "ffma", "ffma")


def _u_w(a: Arith) -> float:
    return {"bf16": U["bf16"], "fp16": U["fp16"], "fp32": U32, "split": SPLIT + U32}[a.weights]


def _w_floor(a: Arith) -> float:
    return FP16_W_FLOOR if a.weights == "fp16" else 0.0


def swish_bound(pre, b_pre, a: Arith, fast: bool):
    """Error of swish(pre + err) for |err| <= b_pre: slope times b_pre plus the function's own error.
    fast: tanh form (eps |x|/2, plus the fma); otherwise x / (1 + expf(-x)) in fp32 (expf 2 ulp, add, divide)."""
    own = (EPS_TANH / 2 + 2 * U32) * np.abs(pre) if fast else 5 * U32 * np.abs(pre)
    return SWISH_SLOPE * b_pre + own


def stem(r, a: Arith):
    """stem_tile_kernel: fp32 FFMA over 27 taps of the float32 normalisation table (u32 per input), fp32 folded weights."""
    b_pre = (27 + 3) * U32 * r["S"]
    return swish_bound(r["pre"], b_pre, a, fast=a.sixteen) + U[a.stem_store] * np.abs(r["out"])


def expand(r, a: Arith, k: int):
    """Expand 1x1 conv + BN + swish, written to E (K1 / K1X / dwse_x on chip, the expand GEMM of the split KD route).

    Weights rounded once to the tensor-core type (BN scale folded first); fp32 accumulation over K; the BN shift either
    rides the MMA as a 16-bit hi + lo pair (K1, K1X: <= 2^-16 |shift|) or is added in fp32.  E is fp16 in the 16-bit
    modes (u_fp16 |e|), the storage type otherwise."""
    shift = np.abs(r["shift_e"])
    b_pre = (_u_w(a) + k * U32) * r["S_e"] + _w_floor(a) * r["X_e"] + (2.0 ** -16 if a.sixteen else U32) * shift
    u_e = U["fp16"] if a.sixteen else U32
    return swish_bound(r["pre_e"], b_pre, a, fast=a.sixteen) + u_e * np.abs(r["e"])


def depthwise(r, a: Arith, block: int, stride: int, b_e=None):
    """Depthwise k x k + BN shift + swish + store.

    hfma2 (bf16 storage, K1 / K1X / KD): fp16 weights w/8 (u_fp16 plus the subnormal floor), k^2 fused steps each rounding
    an fp16 running sum bounded by the sum of |terms| (k^2 u_fp16 S), the same floor on every step, then sum * 4 + shift in
    fp32.  ffma: fp32 weights, k^2 + 1 fp32 roundings.  The E error b_e propagates through |w|."""
    w = r["w"]
    kk = w.shape[0] * w.shape[1]
    mode = a.dw1 if block == 1 else a.dw
    if mode == "hfma2":
        b_pre = (kk + 1) * U["fp16"] * r["S"] + FP16_DW_FLOOR * (r["X"] + kk) + 2 * U32 * (np.abs(r["pre"]) + np.abs(r["shift"]))
    else:
        b_pre = (kk + 2) * U32 * (r["S"] + np.abs(r["shift"]))
    if b_e is not None:
        b_pre = b_pre + depthwise_same(b_e, np.abs(w)[:, :, :, None], stride)
    return swish_bound(r["pre"], b_pre, a, fast=a.sixteen) + U[a.store] * np.abs(r["out"])


def gate(r, a: Arith, d_abs_mean, hw: int, b_in_mean=None):
    """SE gate from the squeeze sums.  The sums are formed from the fp32 depthwise values BEFORE the 16-bit store
    (dw_strip_finish), while the reference starts from the stored tap: u_store mean|d|, plus hw fp32 additions.  Then two
    fp32 FCs (K+1 roundings each), swish and sigmoid through expf.  b_in_mean: the mean distance of the reference's input
    from the values the kernel summed, where it is not the stored tap (default u_store mean|d|)."""
    b_mean = (U[a.store] * d_abs_mean if b_in_mean is None else b_in_mean) + (hw + 1) * U32 * d_abs_mean
    cexp = r["w1"].shape[0]
    cse = r["w1"].shape[1]
    b_z1 = b_mean @ np.abs(r["w1"]) + (cexp + 1) * U32 * r["S_z1"]
    b_a = SWISH_SLOPE * b_z1 + 5 * U32 * np.abs(r["z1"])
    b_z2 = b_a @ np.abs(r["w2"]) + (cse + 1) * U32 * r["S_z2"]
    g = r["out"]
    return g * (1 - g) * b_z2 + 4 * U32 * g


def gated(b_dw, d, g, b_gate, a: Arith):
    """A depthwise output gated in place by the SE tail (scale_out, recorded as "dwg"): the stored d (within b_dw of the
    reference d) times the fp32 gate g (within b_gate), one fp32 product and one 16-bit store: |g| B_dw + |d| B_gate +
    u_store |d g|.  d: (n, h, w, c), g: (n, c)."""
    g4 = np.asarray(g)[:, None, None, :]
    b_g4 = np.asarray(b_gate)[:, None, None, :]
    return np.abs(g4) * b_dw + np.abs(d) * b_g4 + (U[a.store] + U32) * np.abs(d * g4)


def project(r, a: Arith, k: int):
    """Gated project 1x1 + BN (+ residual).  pw_tc2 / pw_tc3 round W * g to the 16-bit type, K2 rounds a * g: with the
    weight rounding, two roundings of every product (2 u S) either way; fp32 accumulation over K, shift and residual added
    in fp32, one store rounding."""
    if a.sixteen:
        u_p = 2 * U[a.weights] + k * U32
        floor = 2 * FP16_W_FLOOR * r["X"] if a.weights == "fp16" else 0.0
    else:
        u_p = _u_w(a) + (k + 1) * U32
        floor = 0.0
    return u_p * r["S"] + floor + 2 * U32 * np.abs(r["out"]) + U[a.store] * np.abs(r["out"])


def head(r, a: Arith):
    """Head 1x1 320 -> 1280 + BN + swish, the same GEMM epilogue as an ungated expand with the shift added in fp32."""
    b_pre = (_u_w(a) + 320 * U32) * r["S"] + _w_floor(a) * r["X"] + U32 * np.abs(r["shift"])
    return swish_bound(r["pre"], b_pre, a, fast=a.sixteen) + U[a.store] * np.abs(r["out"])


def pooled(head_abs):
    """Global average pool of the stored head tensor: 49 fp32 additions and the scale."""
    return (49 + 2) * U32 * np.abs(head_abs).mean(axis=(1, 2))


def angles(r, logits):
    """Dense (fp32, 1281 terms) + softmax expectation decode from the GPU's pooled features.

    A logit error b_l moves the expectation E = sum p_i v_i by at most sum p_i |v_i - E| b_l; the fp32 softmax and the
    weighted sum add (n + 10) u32 sum p_i v_i, and the final * 3 - offset one more rounding."""
    from whenet_oracle import softmax
    out = []
    for lg, s, off in zip(logits, r["S"], (180.0, 99.0, 99.0)):
        n = lg.shape[1]
        v = np.arange(n, dtype=np.float64)
        p = softmax(lg)
        e = (p * v).sum(axis=1)
        b_l = 1282 * U32 * s
        b = (p * np.abs(v[None, :] - e[:, None]) * b_l).sum(axis=1) + (n + 10) * U32 * e
        out.append(3 * b + U32 * (3 * e + off))
    return out


def ulp(x, kind: str):
    """Spacing of the storage type at |x| (normal range; the subnormal spacing below it)."""
    x = np.abs(np.asarray(x, dtype=np.float64))
    mant = {"bf16": 8, "fp16": 11, "fp32": 24}[kind]
    emin = {"bf16": -126, "fp16": -14, "fp32": -126}[kind]
    e = np.floor(np.log2(np.maximum(x, 2.0 ** emin)))
    return 2.0 ** (e - mant + 1)
