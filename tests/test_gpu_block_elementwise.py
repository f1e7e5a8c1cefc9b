"""Every WHENet stage on the GPU, element by element, against float64 on its own GPU input (DESIGN §2.1).

A stage's input is the previous tap (an exact float32 copy of the storage type), so |got - ref| <= 2 B must hold for every
element, B being the first-order bound of tests/whenet_bounds.py (validated on the CPU by test_whenet_bounds_cpu.py); the
checker is tests/elementwise_check.py.  The routes below reach every 16-bit block kernel of the product; the profile's layer names pin which one ran.

Negative controls run on the reference side only, on the default bf16 route's data: a transposed depthwise kernel, an E
tile read one pixel off, symmetric padding on the stride-2 stages, a squeeze that loses the map's last row and a project
without its residual must each leave the bound somewhere, or the bound would be too loose to catch them.
"""
import os

import numpy as np
import pytest

import elementwise_check as ec
import whenet_bounds as wb
from conftest import GOLD, SNAP
from whenet_oracle import depthwise_same, load_oracle, preprocess, swish

pytestmark = pytest.mark.gpu

K1_NB2 = {2: (8, 7, 4, 48, 256, 1), 3: (7, 7, 4, 48, 256, 1), 5: (7, 7, 4, 48, 256, 1), 9: (14, 14, 7, 32, 256, 1),
          10: (7, 7, 4, 48, 256, 1), 12: (7, 7, 4, 32, 256, 1), 13: (7, 7, 4, 64, 512, 2), 14: (7, 7, 7, 64, 512, 2),
          15: (7, 7, 4, 48, 512, 2), 16: (7, 7, 7, 64, 512, 2)}     # plan set "nb2" of test_gpu_parity.py

# route: (precision, options, K1 plans, crops, arithmetic, expected profile layer kind per block)
LATE_SPLIT = {i: ("expand", "kd") for i in range(7, 17)}
LATE_KD = {i: ("kd",) for i in range(7, 17)}
ROUTES = {
    "bf16": ("bf16", {}, None, 8, wb.BF16, {1: ("dw",), **{i: ("k1",) for i in range(2, 7)}, **LATE_SPLIT}),
    "bf16_k1x": ("bf16", {"k1_split_ctas": 0}, None, 8, wb.BF16, {1: ("dw",), **{i: ("k1",) for i in range(2, 7)}, **LATE_KD}),
    "bf16_kd_tail": ("bf16", {"k1_split_ctas": 0, "kd_tail": 1}, None, 8, wb.BF16, {1: ("dw",), **LATE_KD}),
    "bf16_k2": ("bf16", {"pw_variant": 3}, None, 8, wb.BF16, {i: ("project",) for i in range(1, 17)}),
    "fp16": ("fp16", {}, None, 8, wb.FP16, {1: ("dw",), **{i: ("k1",) for i in range(2, 17)}}),
    "fp16_no_split": ("fp16", {"k1_split_ctas": 0}, None, 8, wb.FP16, {1: ("dw",), **{i: ("k1",) for i in range(2, 17)}}),
    "bf16_k1_nb2": ("bf16", {"kd_from": 0}, K1_NB2, 5, wb.BF16, {i: ("k1",) for i in range(2, 17)}),
    "fp32_cuda": ("fp32", {"tensor_cores": 0}, None, 8, wb.FP32_CUDA, {i: ("dw",) for i in range(1, 17)}),
    "fp32_split": ("fp32", {"tensor_cores": 1}, None, 8, wb.FP32_SPLIT, {i: ("dw",) for i in range(1, 17)}),
}

RATIOS = {}

# Which rounding the gated projects of blocks 1-5 (maps >= 28x28) must show: pw_tc2's per-crop route and pw_tc3 round
# bf16(bf16(w) * g), K2 (and pw_tc2 on smaller maps, which is why blocks 6-16 cannot tell the two apart) rounds
# bf16(a * g).  The profile names every project "bNN.project", so the rounding is what pins K2 on bf16_k2.
PROJECT_FORM = {"bf16": "w*g", "bf16_k2": "a*g"}
# blocks on whose (one-tile) K1 the SE gate comes out of the kernel tail when chunks are not split (no "bNN.se" launch)
SE_TAIL_BLOCKS = range(7, 17)
# blocks where a squeeze that loses the map's last row must leave 2 B (measured; see _controls)
GATE_ROW_CAUGHT = {3, 5, *range(7, 17)}


@pytest.fixture(scope="module")
def crops():
    """2 Sample crops, 2 jitter crops, a uniform-random crop (bench.py's distribution), all-0, all-255, and a one-pixel
    0/255 checkerboard: the constant crops make every interior pixel identical, so a tile-edge or padding error stands
    out; the saturated ones push activations towards the fp16 range kDwScale guards."""
    s = np.load(os.path.join(GOLD, "sample_crops.npy"))
    j = np.load(os.path.join(GOLD, "jitter_crops.npy"))[:2]
    rnd = np.random.default_rng(2024).integers(0, 256, (1, 224, 224, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:224, 0:224]
    cb = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], 3, axis=3)
    return np.concatenate([s, j, rnd, np.zeros_like(rnd), np.full_like(rnd, 255), cb])


@pytest.fixture(scope="module")
def oracle():
    return load_oracle(SNAP, np.float64)


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield RATIOS
    ec.print_table(RATIOS, "worst |got - ref| / B per route and tap kind (assertion: <= 2); share within one ulp of the storage type")


def _run_route(m, x, nb, a, route, oracle, blocks, expect, keep_refs=False):
    """Forward with taps, then every stage against float64 on its GPU input.  Returns the references of every block
    when keep_refs (the negative controls need them; they are several GB at 8 crops)."""
    m.enable_profile(True)
    m.get_angle(x)
    names = {p["name"] for p in m.read_profile()}
    m.enable_profile(False)
    for blk, kinds in expect.items():
        for k in kinds:
            assert "b%02d.%s" % (blk, k) in names, (route, blk, k, sorted(names))
    if route in ("bf16_k1x", "bf16_kd_tail"):
        assert not any("b%02d.expand" % i in names for i in range(7, 17)), route
    if route in ("bf16_kd_tail", "fp16_no_split"):
        assert not any("b%02d.se" % i in names for i in SE_TAIL_BLOCKS), route
    m.enable_taps(True)
    ang = np.stack(m.get_angle(x), axis=1).astype(np.float64)
    m.enable_taps(False)
    keep = {} if keep_refs else None
    RATIOS[route] = ec.check_stages(route, ec.tap_reader(m), x, ang, a, oracle, blocks, {}, keep=keep,
                                    project_form=PROJECT_FORM.get(route))
    return keep


def _exceeds(got, ref, b):
    return bool((np.abs(got - ref) > 2 * b).any())


def _controls(oracle, x, keep, blocks):
    """Reference-side mutations that the bound must catch, on the GPU's data of the default bf16 route."""
    failed, gate_inside = [], []
    stem, rs = keep["stem"]
    sym = oracle.run_stage("stem", preprocess(x), symmetric_pad=True)["out"]
    if not _exceeds(stem, sym, wb.stem(rs, wb.BF16)):
        failed.append("stem symmetric padding")
    for i in range(1, 17):
        b = blocks[i - 1]
        prev, rd, bd, d, rg, g, rp, y = keep[i]
        e = rd["e"] if "e" in rd else prev
        w = rd["w"][:, :, :, None]
        s = b["stride"]
        muts = {"transposed kernel": depthwise_same(e, w.transpose(1, 0, 2, 3), s)}
        sh = np.zeros_like(e)
        sh[:, :, 1:] = e[:, :, :-1]
        muts["E one pixel off"] = depthwise_same(sh, w, s)
        if s == 2:
            muts["symmetric padding"] = depthwise_same(e, w, s, symmetric_pad=True)
        for what, pre in muts.items():
            if not _exceeds(d, swish(pre + rd["shift"]), bd):
                failed.append("block %d dw: %s" % (i, what))
        # squeeze sums that lose the map's last row (a tile row dropped at the edge)
        hw = d.shape[1] * d.shape[2]
        m = d[:, :-1].sum(axis=(1, 2)) / hw
        gd = 1 / (1 + np.exp(-(swish(m @ rg["w1"] + (rg["z1"] - rg["mean"] @ rg["w1"])) @ rg["w2"] + (rg["z2"] - rg["a"] @ rg["w2"]))))
        if not _exceeds(g, gd, wb.gate(rg, wb.BF16, np.abs(d).mean(axis=(1, 2)), hw)):
            if i in GATE_ROW_CAUGHT:
                failed.append("block %d gate: last row dropped" % i)
            else:
                gate_inside.append(i)
        if b["skip"] and not _exceeds(y, rp["pre"], wb.project(rp, wb.BF16, d.shape[-1])):
            failed.append("block %d project: residual dropped" % i)
    # The squeeze bound (u_store mean|d| through sum |W1|, as if the rounding errors of 10^2-10^4 pixels had one sign) is
    # rigorous but wider than a lost row on blocks 1, 2, 4 and 6: reported there, asserted on the others.
    print("gate control (last row of the squeeze dropped) stays inside 2 B on blocks %s" % gate_inside)
    return failed


@pytest.mark.parametrize("route", list(ROUTES))
def test_stage_elementwise(route, crops, oracle):
    import whenet_b200
    prec, opts, plans, n, a, expect = ROUTES[route]
    x = crops[:n] if n == 8 else np.concatenate([crops[:4], crops[5:6]])
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    try:
        for k, v in opts.items():
            m.set_option(k, v)
        for blk, plan in (plans or {}).items():
            assert m.set_k1_plan(blk, *plan), (blk, plan)
        blocks = oracle.stage_layers()["blocks"]
        keep = _run_route(m, x, len(x), a, route, oracle, blocks, expect, keep_refs=(route == "bf16"))
    finally:
        m.close()
    if route == "bf16":
        failed = _controls(oracle, x, keep, blocks)
        assert not failed, "negative controls inside the bound: %s" % failed
