"""The per-element error model of tests/whenet_bounds.py, checked on the CPU before any GPU run.

Each kernel family's rounding steps are emulated in numpy / torch at every block's real shapes and weights (bf16
rounding through torch, fp16 through numpy, fused fp16 / fp32 FMAs as one rounding of the exact float64 result, tanh
perturbed by +-2^-11 relative, the fp32 tensor-core mode's operands split into bf16 hi + lo with the lo * lo product
dropped, the in-place gate of the SE tails as a 16-bit rounding of the fp32 product), on the oracle's activations of a
committed crop and of a uniform-random crop.  The
emulated error must stay inside B (the GPU test allows 2 B); the worst emulated / B per family is printed.
"""
import os

import numpy as np
import pytest
import torch

import whenet_bounds as wb
from conftest import GOLD, SNAP
from whenet_oracle import _same_pad, load_oracle, preprocess


def rnd(x, kind):
    x = np.asarray(x, dtype=np.float64)
    if kind == "bf16":
        return torch.from_numpy(x).to(torch.bfloat16).to(torch.float64).numpy()
    if kind == "fp16":
        return x.astype(np.float16).astype(np.float64)
    return x.astype(np.float32).astype(np.float64)


def f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def swish_half(h, sgn):
    """swish_from_half: h + h * tanh.approx(h), the tanh off by sgn * 2^-11 relative."""
    return f32(h + h * (np.tanh(h) * (1 + sgn * 2.0 ** -11)))


def swish_f32(x):
    """swish_f of the fp32 kernels: x / (1 + expf(-x)) in fp32."""
    x = np.asarray(x).astype(np.float32)
    with np.errstate(over="ignore"):          # expf(+large) = inf -> x / inf = -0, the kernel's limit too
        return (x / (np.float32(1) + np.exp(-x))).astype(np.float64)


def conv1x1(x, k, a):
    """x (rows, K) @ folded weights k (K, N) in the arithmetic of the route's 1x1 kernels, before the shift: 16-bit or fp32
    weights, or (pw_tc32) both operands split into bf16 hi + lo and Ahi Whi + Ahi Wlo + Alo Whi; fp32 result."""
    if a.weights == "split":
        wf = f32(k)
        xh, wh = rnd(x, "bf16"), rnd(wf, "bf16")
        xl, wl = rnd(x - xh, "bf16"), rnd(wf - wh, "bf16")
        return f32(xh @ wh + xh @ wl + xl @ wh)
    return f32(x @ (f32(k) if a.weights == "fp32" else rnd(k, a.weights)))


def dw_pad(x, k, s):
    _n, pt, pb = _same_pad(x.shape[1], k, s)
    return np.pad(x, ((0, 0), (pt, pb), (pt, pb), (0, 0))), (x.shape[1] + s - 1) // s


@pytest.fixture(scope="module")
def acts():
    """Oracle float64 taps of Sample crop 0 and a uniform-random crop (bench.py's input distribution)."""
    o = load_oracle(SNAP, np.float64)
    crops = np.concatenate([np.load(os.path.join(GOLD, "sample_crops.npy"))[:1],
                            np.random.default_rng(11).integers(0, 256, (1, 224, 224, 3), dtype=np.uint8)])
    taps = {}
    o.get_angle(crops, taps)
    return o, crops, taps


def test_stage_chain_reproduces_forward(acts):
    """run_stage on the previous stage's output gives the forward's own taps: the per-stage reference is the network."""
    o, crops, taps = acts
    L = o.stage_layers()
    assert len(L["blocks"]) == 16
    assert [b["stride"] for b in L["blocks"]].count(2) == 4
    assert [i + 1 for i, b in enumerate(L["blocks"]) if b["expand"] is None] == [1]
    assert [i + 1 for i, b in enumerate(L["blocks"]) if b["skip"]] == [3, 5, 7, 8, 10, 11, 13, 14, 15]
    x = preprocess(crops)

    def close(a, b):
        return np.abs(a - b).max() <= 1e-9 * (np.abs(b).max() + 1e-30)
    assert close(o.run_stage("stem", x)["out"], taps["stem"])
    prev = taps["stem"]
    for i in range(1, 17):
        d = o.run_stage("dw", prev, i)["out"]
        assert close(d, taps["dw%d" % i]), i
        g = o.run_stage("gate", taps["dw%d" % i], i)["out"]
        assert close(g, taps["gate%d" % i]), i
        y = o.run_stage("project", taps["dw%d" % i], i, gate=taps["gate%d" % i],
                        resid=prev if L["blocks"][i - 1]["skip"] else None)["out"]
        assert close(y, taps["block%d" % i]), i
        prev = taps["block%d" % i]
    assert close(o.run_stage("head", prev)["out"], taps["head"])
    lg = o.run_stage("dense", taps["pooled"])["logits"]
    ref = o.forward_normalised(x)
    assert all(close(a, b) for a, b in zip(lg, ref))


def emulate_block(o, blk, b, x, a, sgn, route_k2=False):
    """One block in the arithmetic of the route's kernels on the exact input x (storage-rounded); returns the emulated
    values and their bounds next to the float64 references."""
    out = {}
    ri = o.run_stage("dw", x, blk)
    if b["expand"] is not None:
        k, sh = o._fold(*b["expand"])
        k = k[0, 0]
        x2 = x.reshape(-1, k.shape[0])
        if a.sixteen:
            w16 = rnd(0.5 * k, a.weights)                      # K1: 0.5 * folded weights, one 16-bit rounding
            hi = rnd(0.5 * sh, a.weights)
            lo = rnd(0.5 * sh - hi, a.weights)                 # the BN shift as two extra K columns
            acc = f32(x2 @ w16 + hi + lo).reshape(x.shape[:3] + (k.shape[1],))
            e = rnd(swish_half(acc, sgn), "fp16")              # E: fp16 whatever the storage type
        else:
            pre = f32(conv1x1(x2, k, a) + f32(sh)).reshape(x.shape[:3] + (k.shape[1],))
            e = swish_f32(pre)
        b_e = wb.expand(ri, a, k.shape[0])
        out["expand"] = (e, ri["e"], b_e)
    else:
        e, b_e = x, None                                       # block 1: the E tile is the stem output
    w = ri["w"]
    ks = w.shape[0]
    ep, ho = dw_pad(e, ks, b["stride"])
    s = b["stride"]
    mode = a.dw1 if blk == 1 else a.dw
    if mode == "hfma2":
        wq = rnd(0.5 * w / wb.KDW, "fp16")
        acc = np.zeros(e.shape[:1] + (ho, ho, e.shape[3]))
        for ky in range(ks):
            for kx in range(ks):                                # fp16 running sum, one rounding per fused step
                acc = rnd(acc + ep[:, ky:ky + (ho - 1) * s + 1:s, kx:kx + (ho - 1) * s + 1:s, :] * wq[ky, kx], "fp16")
        d32 = swish_half(f32(acc * wb.KDW + f32(0.5 * ri["shift"])), sgn)
    else:
        half = 0.5 if a.sixteen else 1.0                       # K1 works on x/2 (swish_from_half), the fp32 kernels on x
        wq = f32(half * w)
        acc = np.broadcast_to(f32(half * ri["shift"]), e.shape[:1] + (ho, ho, e.shape[3])).copy()
        for ky in range(ks):
            for kx in range(ks):
                acc = f32(acc + ep[:, ky:ky + (ho - 1) * s + 1:s, kx:kx + (ho - 1) * s + 1:s, :] * wq[ky, kx])
        d32 = swish_half(acc, sgn) if a.sixteen else swish_f32(acc)
    d = rnd(d32, a.store)
    out["dw"] = (d, ri["out"], wb.depthwise(ri, a, blk, s, b_e))
    # SE gate: squeeze sums of the fp32 values before the store, fp32 FCs with expf
    rg = o.run_stage("gate", d, blk)
    m = f32(d32.astype(np.float32).sum(axis=(1, 2), dtype=np.float32) / np.float32(ho * ho))
    z1 = f32(m.astype(np.float32) @ rg["w1"].astype(np.float32) + o.w[b["se"][0] + "/bias:0"])
    a1 = f32(z1 / (1 + np.exp(-z1.astype(np.float32))))
    z2 = f32(a1.astype(np.float32) @ rg["w2"].astype(np.float32) + o.w[b["se"][1] + "/bias:0"])
    g = f32(1 / (1 + np.exp(-z2.astype(np.float32))))
    b_g = wb.gate(rg, a, np.abs(d).mean(axis=(1, 2)), ho * ho)
    out["gate"] = (g, rg["out"], b_g)
    if a.sixteen:
        # the SE tails' in-place gate (scale_out): round16(float32(d) * float32(g)), against the float64 d * g
        dg = rnd(f32(d * g[:, None, None, :]), a.store)
        out["gated"] = (dg, ri["out"] * rg["out"][:, None, None, :], wb.gated(out["dw"][2], ri["out"], rg["out"], b_g, a))
    # project: pw_tc2 / pw_tc3 round bf16(w) * g, K2 rounds d * g; the fp32 kernels gate A in fp32
    k, sh = o._fold(b["proj"], b["proj_bn"])
    k = k[0, 0]
    n, c = d.shape[0], d.shape[3]
    if not a.sixteen:
        acc = conv1x1(f32(d * g[:, None, None, :]).reshape(-1, c), k, a)
    elif route_k2:
        acc = rnd(d * g[:, None, None, :], a.store).reshape(n, -1, c) @ rnd(k, a.weights)
    else:
        acc = np.einsum("npk,nkj->npj", d.reshape(n, -1, c), rnd(rnd(k, a.weights)[None] * g[:, :, None], a.weights))
    y = f32(f32(acc.reshape(d.shape[:3] + (k.shape[1],))) + f32(sh))
    res = x if b["skip"] else None
    if res is not None:
        y = f32(y + res)
    y = rnd(y, a.store)
    rp = o.run_stage("project", d, blk, gate=g, resid=res)
    out["project"] = (y, rp["out"], wb.project(rp, a, c))
    return out


@pytest.mark.parametrize("a", [wb.BF16, wb.FP16, wb.FP32_SPLIT, wb.FP32_CUDA], ids=["bf16", "fp16", "fp32_split", "fp32_cuda"])
def test_emulated_error_within_bound(a, acts):
    o, crops, taps = acts
    L = o.stage_layers()
    worst = {}

    def note(fam, got, ref, b, blk):
        r = np.abs(got - ref) / b
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        if r[i] > worst.get(fam, (0.0,))[0]:
            worst[fam] = (float(r[i]), blk, i)
    for sgn in ((1, -1) if a.sixteen else (1,)):
        # stem: fp32 conv of the table-normalised input, tanh swish (16-bit modes) and store
        x = f32(preprocess(crops))
        rs = o.run_stage("stem", x)
        pre = f32(rs["pre"])                                   # the fp32 FFMA chain: one rounding of the exact sum
        st = swish_half(0.5 * pre, sgn) if a.sixteen else swish_f32(pre)
        note("stem", rnd(st, a.stem_store), rs["out"], wb.stem(rs, a), 0)
        prev = rnd(taps["stem"], a.stem_store)
        for blk in range(1, 17):
            b = L["blocks"][blk - 1]
            for fam, (got, ref, bound) in emulate_block(o, blk, b, prev, a, sgn, route_k2=(sgn < 0)).items():
                note(fam if fam != "dw" else ("dw_" + (a.dw1 if blk == 1 else a.dw)), got, ref, bound, blk)
            prev = rnd(taps["block%d" % blk], a.store)
        rh = o.run_stage("head", prev)
        k, sh = o._fold(*L["head"])
        hp = f32(conv1x1(prev.reshape(-1, 320), k[0, 0], a).reshape(rh["pre"].shape) + f32(sh))
        hs = swish_half(0.5 * hp, sgn) if a.sixteen else swish_f32(hp)
        note("head", rnd(hs, a.store), rh["out"], wb.head(rh, a), 17)
    for fam, (r, blk, i) in sorted(worst.items()):
        print("%s %-10s worst emulated/B = %.3f (block %d, element %s)" % (a.weights, fam, r, blk, i))
    for fam, (r, blk, i) in worst.items():
        assert r <= 1.0, (a.weights, fam, r, blk, i)
    assert set(worst) >= {"stem", "expand", "dw_" + a.dw, "dw_" + a.dw1, "gate", "project", "head"} | ({"gated"} if a.sixteen else set())
