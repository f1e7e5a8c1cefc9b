"""Parity of the CUDA path (through the C ABI / WHENet class) against the CPU oracle.

Tolerances (stated per north_star):
  fp32 parity mode : |angle - oracle64| <= 0.01 deg on the Sample/ crops; every block-boundary
                     tensor within 2e-4 relative (max-norm) of the float32 oracle.
  bf16 mode        : |angle - oracle64| <= 1.5 deg (measured ~0.1-0.5, SURVEY.md 8c sensitivity
                     table: bf16 activation storage alone costs 0.33 deg on these crops).
  fp16 mode        : |angle - oracle64| <= 0.15 deg.
"""
import numpy as np
import pytest

from conftest import SNAP

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def net32():
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="fp32", max_batch=64)
    yield m
    m.close()


@pytest.fixture(scope="module")
def net16():
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=64)
    yield m
    m.close()


def _relerr(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_sample_angles_fp32(net32, sample_crops, golden):
    yaw, pitch, roll = net32.get_angle(sample_crops)
    assert yaw.dtype == np.float32 and yaw.shape == (2,)
    for i, s in enumerate(golden["samples"]):
        assert abs(yaw[i] - s["yaw"]) <= 0.01
        assert abs(pitch[i] - s["pitch"]) <= 0.01
        assert abs(roll[i] - s["roll"]) <= 0.01


def test_block_taps_fp32(net32, oracle32, sample_crops):
    taps = {}
    oracle32.get_angle(sample_crops, taps)
    net32.enable_taps(True)
    net32.get_angle(sample_crops)
    net32.enable_taps(False)
    names = ["stem"] + ["%s%d" % (k, i) for i in range(1, 17) for k in ("dw", "gate", "block")] + ["head", "pooled"]
    worst = 0.0
    for nm in names:
        ref = taps[nm].astype(np.float64).reshape(-1)
        got = net32.tap(nm).astype(np.float64)
        assert got.size == ref.size, nm
        e = _relerr(got, ref)
        worst = max(worst, e)
        assert e < 2e-4, (nm, e)
    print("worst relative tap error fp32: %.3g" % worst)


def test_logits_predict_fp32(net32, oracle64, sample_crops):
    from whenet_oracle import preprocess
    x = preprocess(sample_crops).astype(np.float32)
    got = net32.model.predict(x, batch_size=8)
    ref = oracle64.forward_normalised(x)
    assert [g.shape for g in got] == [(2, 120), (2, 66), (2, 66)]
    for g, r in zip(got, ref):
        assert g.dtype == np.float32
        assert np.abs(g - r).max() < 2e-3


def test_float_input_path(net32, sample_crops):
    a = net32.get_angle(sample_crops)
    b = net32.get_angle(sample_crops.astype(np.float64))
    for u, v in zip(a, b):
        assert np.abs(u - v).max() < 1e-3


def test_jitter_batch_fp32(net32, jitter_crops, golden):
    yaw, pitch, roll = net32.get_angle(jitter_crops)
    g = golden["jitter"]
    assert np.abs(yaw - np.array(g["yaw"])).max() <= 0.01
    assert np.abs(pitch - np.array(g["pitch"])).max() <= 0.01
    assert np.abs(roll - np.array(g["roll"])).max() <= 0.01


@pytest.mark.parametrize("prec,tol", [("bf16", 1.5), ("fp16", 0.15)])
def test_sample_angles_16bit(prec, tol, sample_crops, jitter_crops, golden):
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=16)
    crops = np.concatenate([sample_crops, jitter_crops])
    got = np.stack(m.get_angle(crops), axis=1)
    ref = np.array([[s["yaw"], s["pitch"], s["roll"]] for s in golden["samples"]] +
                   list(zip(golden["jitter"]["yaw"], golden["jitter"]["pitch"], golden["jitter"]["roll"])))
    err = np.abs(got - ref).max()
    print("%s max |angle - oracle64| = %.4f deg" % (prec, err))
    assert err <= tol
    m.close()


@pytest.mark.parametrize("tc", [0, 1])
def test_bf16_taps_vs_oracle(tc, oracle32, sample_crops):
    """Every block boundary of the bf16 path stays within bf16-rounding distance of the oracle."""
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
    m.set_option("tensor_cores", tc)
    m.set_option("fused", 0)
    taps = {}
    oracle32.get_angle(sample_crops, taps)
    m.enable_taps(True)
    m.get_angle(sample_crops)
    worst = ("", 0.0)
    for nm in ["stem"] + ["block%d" % i for i in range(1, 17)] + ["head", "pooled"]:
        ref = taps[nm].astype(np.float64).reshape(-1)
        got = m.tap(nm).astype(np.float64)
        e = float(np.sqrt(((got - ref) ** 2).mean()) / (np.sqrt((ref ** 2).mean()) + 1e-30))
        if e > worst[1]:
            worst = (nm, e)
        assert e < 0.05, (nm, e)       # rms-relative; bf16 has 8 mantissa bits (2^-9 = 0.2% per rounding)
    print("tc=%d worst rms-relative tap error: %s %.4f" % (tc, *worst))
    m.close()


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_fused_k1_taps(prec, oracle32, sample_crops):
    """K1 (expand + depthwise fused, expanded tensor kept in shared memory) for every block that has an
    expand conv: depthwise outputs, SE gates and block outputs against the oracle."""
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    m.set_option("fused", 1)
    m.set_option("fused_max_block", 16)
    m.set_option("kd_from", 0)               # K1 on the late blocks too (the default bf16 route there is KD: test_kd_route)
    taps = {}
    oracle32.get_angle(sample_crops, taps)
    m.enable_taps(True)
    got = np.stack(m.get_angle(sample_crops), axis=1)
    lim = 0.12 if prec == "bf16" else 0.02   # rms-relative; bf16 noise compounds through cancelling project outputs
    for i in range(1, 17):
        for kind in ("dw", "gate", "block"):
            nm = "%s%d" % (kind, i)
            ref = taps[nm].astype(np.float64).reshape(-1)
            g = m.tap(nm).astype(np.float64)
            e = float(np.sqrt(((g - ref) ** 2).mean()) / (np.sqrt((ref ** 2).mean()) + 1e-30))
            assert e < lim, (nm, e)
    ref_ang = np.stack(oracle32.get_angle(sample_crops), axis=1)
    assert np.abs(got - ref_ang).max() < (1.5 if prec == "bf16" else 0.15)
    m.close()


K1_PLAN_SETS = {
    # 512-thread CTAs (one per SM) on the late blocks
    "nt512": {7: (14, 14, 7, 96, 512, 1), 8: (14, 14, 7, 96, 512, 1), 9: (14, 14, 7, 96, 512, 1), 10: (14, 14, 7, 96, 512, 1),
              11: (14, 14, 7, 112, 512, 1), 12: (7, 7, 4, 96, 512, 1), 13: (7, 7, 4, 96, 512, 1), 14: (7, 7, 4, 64, 512, 1),
              15: (7, 7, 7, 96, 512, 1), 16: (7, 7, 4, 96, 512, 1)},
    # two crops per CTA on the 7x7 stages; small two-per-SM plans elsewhere (edge tiles with fewer GEMM rows than interior ones)
    "nb2": {2: (8, 7, 4, 48, 256, 1), 3: (7, 7, 4, 48, 256, 1), 5: (7, 7, 4, 48, 256, 1), 9: (14, 14, 7, 32, 256, 1),
            10: (7, 7, 4, 48, 256, 1), 12: (7, 7, 4, 32, 256, 1), 13: (7, 7, 4, 64, 512, 2), 14: (7, 7, 7, 64, 512, 2),
            15: (7, 7, 4, 48, 512, 2), 16: (7, 7, 7, 64, 512, 2)},
    "nb2_nt256": {13: (7, 7, 4, 64, 256, 2), 14: (7, 7, 4, 48, 256, 2), 16: (7, 7, 4, 64, 256, 2), 6: (7, 7, 4, 48, 256, 1),
                  4: (7, 7, 7, 48, 256, 1)},
}


@pytest.mark.parametrize("plan_set", sorted(K1_PLAN_SETS))
@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_fused_k1_plan_variants(prec, plan_set, oracle32, sample_crops, jitter_crops):
    """Every K1 tile-plan family (512-thread CTAs, two crops per CTA, small edge-tile plans) against the oracle taps on an
    odd crop count (the last two-crop CTA is half empty), and bitwise batch invariance under those plans."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops[:1]])
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    m.set_option("kd_from", 0)
    for blk, plan in K1_PLAN_SETS[plan_set].items():
        assert m.set_k1_plan(blk, *plan), (blk, plan)
    taps = {}
    ref_ang = np.stack(oracle32.get_angle(crops, taps), axis=1)
    m.enable_taps(True)
    got = np.stack(m.get_angle(crops), axis=1)
    lim = 0.12 if prec == "bf16" else 0.02
    for i in range(1, 17):
        for kind in ("dw", "gate", "block"):
            nm = "%s%d" % (kind, i)
            ref = taps[nm].astype(np.float64).reshape(-1)
            g = m.tap(nm).astype(np.float64)
            e = float(np.sqrt(((g - ref) ** 2).mean()) / (np.sqrt((ref ** 2).mean()) + 1e-30))
            assert e < lim, (plan_set, nm, e)
    assert np.abs(got - ref_ang).max() < (1.5 if prec == "bf16" else 0.15)
    m.enable_taps(False)
    for i in range(3):
        one = np.stack(m.get_angle(crops[i:i + 1]), axis=1)
        assert np.array_equal(one[0], got[i]), (plan_set, i)
    pair = np.stack(m.get_angle(crops[1:3]), axis=1)
    assert np.array_equal(pair, got[1:3])
    m.close()


def test_kd_route(oracle32, sample_crops, jitter_crops):
    """Late blocks (7-16) in bf16: expand as a tensor-core GEMM writing fp16 E + KD (depthwise + squeeze-excite + gating in one
    kernel, kernels_dwse.cuh).  Depthwise outputs, gates and block outputs against the oracle; agreement with the K1 route
    (same arithmetic up to the rounding of the expand accumulators); bitwise equality of the chunk-split route (small
    batches: several CTAs per crop, gate from se_gate_kernel, gated project conv) and the one-CTA-per-crop route (gate and
    gating in the kernel tail); bitwise batch invariance."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops[:3]])
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
    m.set_option("kd_from", 0)
    launches0 = m.launch_count()
    k1 = np.stack(m.get_angle(crops), axis=1)
    n_k1 = m.launch_count() - launches0
    m.set_option("kd_from", 7)
    launches0 = m.launch_count()
    split = np.stack(m.get_angle(crops), axis=1)          # 5 crops: chunks split over CTAs
    n_kd = m.launch_count() - launches0
    assert n_kd == n_k1 + 10                               # expand + KD instead of K1 on ten blocks
    assert np.abs(split - k1).max() < 0.25
    m.set_option("k1_split_ctas", 0)                       # one CTA per crop, gate still from se_gate + gated project (the default)
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), split)
    m.set_option("kd_tail", 1)                             # ... SE tail (+ in-place gating) inside KD
    for so in (0, 1):
        m.set_option("se_scale_out", so)
        tail = np.stack(m.get_angle(crops), axis=1)
        assert np.array_equal(tail, split), so
    m.set_option("kd_tail", 0)
    for i in (0, 4):
        one = np.stack(m.get_angle(crops[i:i + 1]), axis=1)
        assert np.array_equal(one[0], split[i])
    taps = {}
    ref_ang = np.stack(oracle32.get_angle(crops, taps), axis=1)
    m.enable_taps(True)
    got = np.stack(m.get_angle(crops), axis=1)
    for i in range(1, 17):
        for kind in ("dw", "gate", "block"):
            nm = "%s%d" % (kind, i)
            r = taps[nm].astype(np.float64).reshape(-1)
            g = m.tap(nm).astype(np.float64)
            e = float(np.sqrt(((g - r) ** 2).mean()) / (np.sqrt((r ** 2).mean()) + 1e-30))
            assert e < 0.12, (nm, e)
    assert np.abs(got - ref_ang).max() < 0.6
    m.close()


def test_pageable_input_staging(sample_crops, jitter_crops):
    """get_angle(numpy array) = a PAGEABLE host buffer (the reference's call shape): batches of 8 MB and more are copied into the
    context's pinned staging buffer by several host threads, piece by piece, each piece starting its DMA as soon as it is staged.
    Same bits as the plain cudaMemcpyAsync route, for repeated calls, changing sizes and a float32 input."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 20)[:150]
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=256)
    m.set_option("stage_threads", 0)
    ref = np.stack(m.get_angle(crops), axis=1)
    for nt in (8, 1, 3):
        m.set_option("stage_threads", nt)
        for n in (150, 70, 150):
            got = np.stack(m.get_angle(crops[:n]), axis=1)
            assert np.array_equal(got, ref[:n]), (nt, n)
    m.set_option("streams", 1)
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), ref)
    m.close()
    m32 = whenet_b200.WHENet(SNAP, device=0, precision="fp32", max_batch=64)
    x = crops[:40].astype(np.float32)
    m32.set_option("stage_threads", 0)
    a = np.stack(m32.get_angle(x), axis=1)
    m32.set_option("stage_threads", 4)
    assert np.array_equal(np.stack(m32.get_angle(x), axis=1), a)
    m32.close()


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_se_batch_and_k2_routes_bitwise(prec, sample_crops, jitter_crops):
    """Throughput-sized batches switch three kernels: the SE gates come from se_gate_batch_kernel (four crops per CTA share
    the FC weight loads), the ungated / small-map 1x1 convs run on the persistent K2 kernel, the head runs as GAP kernel +
    Dense/decode for eight crops per CTA.  All must give the bits of the small-batch routes (se_gate_kernel, pw_tc2,
    head_pool_fc_decode_kernel)."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 9)[:70]
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=128)
    m.set_option("streams", 1)
    ref = np.stack(m.get_angle(crops), axis=1)
    small = np.concatenate([np.stack(m.get_angle(crops[i:i + 8]), axis=1) for i in range(0, 70, 8)])
    assert np.array_equal(ref, small)
    m.set_option("se_batch", 0)
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), ref)
    m.set_option("se_batch", 1)
    m.set_option("head_batch", 0)                          # one CTA per crop for GAP + Dense + decode
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), ref)
    m.set_option("head_batch", 1)
    m.set_option("pw3", 0)                                 # gated projects of the large maps: one tile per CTA (pw_tc2) instead of pw_tc3
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), ref)
    m.set_option("pw3", 1)
    m.set_option("pw_variant", 2)                          # pw_tc2 everywhere
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), ref)
    m.set_option("pw_variant", 3)                          # K2 everywhere: the gated projects of blocks 1-6 then scale A rows
    all_k2 = np.stack(m.get_angle(crops), axis=1)          # (bf16(a*g)) instead of W rows (bf16(w*g)) - same maths, other rounding
    assert np.abs(all_k2 - ref).max() < (1.0 if prec == "bf16" else 0.1)      # two valid roundings, each within 0.5 / 0.05 deg of the oracle
    m.close()


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_se_tail_paths_bitwise(prec, oracle32, sample_crops, jitter_crops):
    """Blocks whose K1 CTA holds whole crops compute the SE gate in the kernel tail and gate their depthwise output in
    place.  Both steps must reproduce the stand-alone route (se_gate_kernel + gate pass inside the project conv) bit for
    bit, because small batches (chunk split) still take that route; gates are also checked against the oracle."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops[:3]])          # 5 crops: the last two-crop CTA is half empty
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    m.set_option("kd_from", 0)                 # K1 on the late blocks (the KD route has its own test)
    m.set_option("se_tail", 0)
    ref = np.stack(m.get_angle(crops), axis=1)
    m.set_option("se_tail", 1)
    m.set_option("k1_split_ctas", 0)           # no chunk split even at 5 crops -> the tail path runs
    m.set_option("se_scale_out", 0)
    launches0 = m.launch_count()
    a = np.stack(m.get_angle(crops), axis=1)
    n_tail = m.launch_count() - launches0
    assert np.array_equal(a, ref)
    m.set_option("se_scale_out", 1)
    b = np.stack(m.get_angle(crops), axis=1)
    assert np.array_equal(b, ref)
    m.set_option("se_tail", 0)
    launches0 = m.launch_count()
    m.get_angle(crops)
    assert m.launch_count() - launches0 == n_tail + 10      # blocks 7..16 lose their se_gate launch under se_tail
    m.set_option("se_tail", 1)
    taps = {}
    oracle32.get_angle(crops, taps)
    m.enable_taps(True)
    m.get_angle(crops)
    lim = 0.12 if prec == "bf16" else 0.02
    for i in range(1, 17):
        for kind in ("dw", "gate", "block"):
            nm = "%s%d" % (kind, i)
            r = taps[nm].astype(np.float64).reshape(-1)
            g = m.tap(nm).astype(np.float64)
            e = float(np.sqrt(((g - r) ** 2).mean()) / (np.sqrt((r ** 2).mean()) + 1e-30))
            assert e < lim, (nm, e)
    m.close()


@pytest.mark.parametrize("kd_from", [0, 7])
def test_fused_k1_batch_invariance(kd_from, sample_crops, jitter_crops):
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 3)[:19]
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=32)
    m.set_option("fused", 1)
    m.set_option("fused_max_block", 16)
    m.set_option("kd_from", kd_from)
    full = np.stack(m.get_angle(crops), axis=1)
    for i in (0, 7, 18):
        one = np.stack(m.get_angle(crops[i:i + 1]), axis=1)
        assert np.array_equal(one[0], full[i])
    m.close()


def test_tensor_core_path_matches_simt(sample_crops, jitter_crops):
    """Same storage type, two kernel families: results agree to bf16 rounding noise."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops])
    out = []
    for tc in (0, 1):
        m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
        m.set_option("tensor_cores", tc)
        m.set_option("fused", 0)
        out.append(np.stack(m.get_angle(crops), axis=1))
        m.close()
    assert np.abs(out[0] - out[1]).max() < 1.5


def test_batch_invariance(net32, net16, sample_crops, jitter_crops):
    """A crop's result does not depend on its batch neighbours or position (N=1 vs N=37): bitwise."""
    crops = np.concatenate([sample_crops, jitter_crops] * 5)[:37]
    for m in (net32, net16):
        full = np.stack(m.get_angle(crops), axis=1)
        for i in (0, 1, 17, 36):
            one = np.stack(m.get_angle(crops[i:i + 1]), axis=1)
            assert np.array_equal(one[0], full[i]), (m.precision, i)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_dw_variants_agree(prec, sample_crops, jitter_crops):
    """One-output-per-thread and register-blocked depthwise kernels: same taps in the same order -> same sums
    (fp32: bitwise; 16-bit: the strip kernel uses the tanh-form swish, so only to rounding noise)."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops])
    out = []
    for v in (0, 1):
        m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
        m.set_option("dw_variant", v)
        m.set_option("tensor_cores", 0)
        m.set_option("fused", 0)
        out.append(np.stack(m.get_angle(crops), axis=1))
        m.close()
    if prec == "fp32":
        assert np.abs(out[0] - out[1]).max() < 1e-3
    else:
        assert np.abs(out[0] - out[1]).max() < 1.0


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_repeatability_stress(prec, sample_crops, jitter_crops):
    """Race detector of last resort: the same inputs, many forwards, several batch sizes, with per-tap profiling on
    and off (different kernel timing) - every result must be bitwise identical.  (Round 1 had a missing barrier in
    pw_tc2 between the cp.async of the SE gate rows and their first use; it only showed up intermittently.)"""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 8)[:61]
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=64)
    for n in (2, 8, 61):
        ref = np.stack(m.get_angle(crops[:n]), axis=1)
        for it in range(12):
            if it == 6:
                m.enable_profile(True)
            got = np.stack(m.get_angle(crops[:n]), axis=1)
            assert np.array_equal(got, ref), (prec, n, it)
        m.enable_profile(False)
        m.read_profile()
    m.close()


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_full_size_batch_properties(prec, sample_crops, jitter_crops):
    """BASELINE.json's full single-GPU size (512 crops) through the default configuration (two streams, fused kernels):
    the oracle is too slow for 512 crops, so use size-independent properties - a batch tiled from 8 distinct crops
    must be periodic and bitwise equal to the 8-crop result, whatever the position of a crop in the batch."""
    import whenet_b200
    base = np.concatenate([sample_crops, jitter_crops])
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=512)
    small = np.stack(m.get_angle(base), axis=1)
    rng = np.random.default_rng(7)
    order = rng.integers(0, 8, 512)
    big = np.stack(m.get_angle(base[order]), axis=1)
    assert big.shape == (512, 3)
    assert np.array_equal(big, small[order])
    m.close()


def test_two_stream_mode_bitwise(sample_crops, jitter_crops):
    """streams=2 runs the two half batches concurrently on two streams: same bits as the single-stream pass."""
    import torch
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 17)[:131]
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=160)
    ref = np.stack(m.get_angle(crops), axis=1)
    m.set_option("streams", 2)
    x = torch.from_numpy(crops).cuda()
    y = torch.empty((131, 3), dtype=torch.float32, device="cuda")
    for _ in range(4):
        y.zero_()
        torch.cuda.synchronize()
        m.forward_device(x, y)
        m.synchronize()
        assert np.array_equal(y.cpu().numpy(), ref)
    m.close()


def test_chunking_invariance(sample_crops, jitter_crops):
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops] * 3)   # 24
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=32)
    a = np.stack(m.get_angle(crops), axis=1)
    m.set_option("chunk", 5)     # ragged: 5,5,5,5,4
    b = np.stack(m.get_angle(crops), axis=1)
    assert np.array_equal(a, b)
    m.close()


def test_more_than_max_batch(net32, sample_crops):
    crops = np.tile(sample_crops, (40, 1, 1, 1))   # 80 > max_batch 64, alternating crop 0 / crop 1
    yaw, _p, _r = net32.get_angle(crops)
    assert yaw.shape == (80,)
    assert np.array_equal(yaw[0::2], np.full(40, yaw[0], dtype=np.float32))
    assert np.array_equal(yaw[1::2], np.full(40, yaw[1], dtype=np.float32))


def test_random_init_parity():
    """snapshot=None (reference whenet.py:15): random weights; CUDA path == oracle on the same tensors."""
    import whenet_b200
    from whenet_b200 import arch
    from whenet_oracle import Oracle
    w = arch.random_weights(0)
    names = whenet_b200.weights.load_snapshot(SNAP)[0]
    o = Oracle(names, w, np.float64)
    rng = np.random.default_rng(3)
    x = rng.integers(0, 256, (3, 224, 224, 3), dtype=np.uint8)
    ref = np.stack(o.get_angle(x), axis=1)
    m = whenet_b200.WHENet(None, device=0, precision="fp32", max_batch=4)
    got = np.stack(m.get_angle(x), axis=1)
    assert np.abs(got - ref).max() < 0.02
    m.close()


def test_errors(net32):
    import whenet_b200
    with pytest.raises(ValueError):
        net32.get_angle(np.zeros((1, 200, 224, 3), np.uint8))
    with pytest.raises(ValueError):
        net32.model.predict(np.zeros((224, 224, 3), np.float32))
    with pytest.raises(OSError):
        whenet_b200.WHENet("/nonexistent/WHENet.h5", device=0)
    import ctypes as C
    from whenet_b200 import _lib
    L = _lib.load()
    buf = np.zeros((1, 224, 224, 3), np.uint8)
    out = np.zeros((1, 3), np.float32)
    rc = L.whenet_forward_u8(net32._h, buf.ctypes.data, 65, 0, out.ctypes.data, None, 0)
    assert rc == -1 and b"max_batch" in L.whenet_last_error()
    h = C.c_void_p()
    assert L.whenet_create(C.byref(h), 0, 4, 0) == 0
    assert L.whenet_forward_u8(h, buf.ctypes.data, 1, 0, out.ctypes.data, None, 0) == -3   # no weights
    L.whenet_destroy(h)
    assert L.whenet_create(C.byref(h), 99, 4, 0) == -1


def test_empty_batch(net32):
    y, p, r = net32.get_angle(np.zeros((0, 224, 224, 3), np.uint8))
    assert y.shape == (0,) and y.dtype == np.float32


def test_cuda_graph_replay(sample_crops, jitter_crops):
    """Device-resident forwards replayed from a captured CUDA graph give bit-identical results, also after the
    input buffer CONTENT changes (same addresses), and new shapes capture new graphs."""
    import torch
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
    crops = np.concatenate([sample_crops, jitter_crops])
    ref = np.stack(m.get_angle(crops), axis=1)
    s = torch.cuda.Stream()
    torch.cuda.set_stream(s)
    m.set_stream(s.cuda_stream)
    m.set_option("graph", 1)
    x = torch.from_numpy(crops).cuda()
    y = torch.empty((8, 3), dtype=torch.float32, device="cuda")
    for _ in range(3):
        m.forward_device(x, y)
    torch.cuda.synchronize()
    assert np.array_equal(y.cpu().numpy(), ref)
    x.copy_(torch.from_numpy(crops[::-1].copy()).cuda())
    m.forward_device(x, y)
    torch.cuda.synchronize()
    assert np.array_equal(y.cpu().numpy(), ref[::-1])
    m.forward_device(x[:3], y[:3])
    torch.cuda.synchronize()
    assert np.array_equal(y.cpu().numpy()[:3], ref[::-1][:3])
    torch.cuda.set_stream(torch.cuda.default_stream())
    m.close()


def test_async_host_double_buffering(sample_crops, jitter_crops):
    """whenet_forward_u8_async: two host batches in flight, results identical to the synchronous call."""
    import torch
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
    a = torch.from_numpy(np.concatenate([sample_crops, jitter_crops])).pin_memory()
    b = torch.from_numpy(np.concatenate([jitter_crops, sample_crops])).pin_memory()
    ra = np.stack(m.get_angle(a.numpy()), axis=1)
    rb = np.stack(m.get_angle(b.numpy()), axis=1)
    oa = torch.empty((8, 3), dtype=torch.float32).pin_memory()
    ob = torch.empty((8, 3), dtype=torch.float32).pin_memory()
    for _ in range(3):
        m.forward_host_async(a, oa)
        m.forward_host_async(b, ob)
        m.synchronize()
        assert np.array_equal(oa.numpy(), ra) and np.array_equal(ob.numpy(), rb)
    m.close()


def test_device_resident_async(sample_crops):
    import torch
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="fp32", max_batch=8)
    ref = np.stack(m.get_angle(sample_crops), axis=1)
    x = torch.from_numpy(sample_crops).cuda()
    out = torch.empty((2, 3), dtype=torch.float32, device="cuda")
    m.set_stream(torch.cuda.current_stream().cuda_stream)
    m.forward_device(x, out)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)
    m.close()
