"""Parity at the sizes and on the input distribution bench.py measures (BASELINE configs[1] and [2]), the decode unit
hook, the timeout plumbing, and oracle taps for the persistent K1 variant.

Tolerances:
  fp32 parity mode, 512 / 32 uniform-random uint8 crops vs the torch-CPU float32 port of the oracle: 0.01 deg
      (north_star's tolerance; two float32 evaluations with different summation orders)
  bf16 (the benched mode) on the same crops: 0.6 deg;  fp16: 0.08 deg
"""
import numpy as np
import pytest

import whenet_oracle as wo
from conftest import SNAP

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def port():
    from whenet_b200 import weights
    names, w = weights.load_snapshot(SNAP)
    return wo.TorchCpuPort(names, w)


@pytest.fixture(scope="module")
def bench_crops():
    # bench.py's synthetic input distribution: independent uniform bytes
    return np.random.default_rng(0).integers(0, 256, (512, 224, 224, 3), dtype=np.uint8)


@pytest.fixture(scope="module")
def bench_ref(port, bench_crops):
    return np.stack(port.get_angle(bench_crops), axis=1)


@pytest.mark.parametrize("prec,tol", [("fp32", 0.01), ("bf16", 0.6), ("fp16", 0.08)])
def test_batch512_random_uint8_vs_cpu_port(prec, tol, bench_crops, bench_ref):
    """configs[2]: one 512-crop call in the default configuration (two half-batch streams, fused tensor-core kernels)."""
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=512)
    got = np.stack(m.get_angle(bench_crops), axis=1)
    err = np.abs(got - bench_ref)
    print("%s N=512 random uint8: max |angle - cpu port| = %.5f deg (mean %.5f)" % (prec, err.max(), err.mean()))
    assert err.max() <= tol
    # the same crops through the persistent K1 variant and as one stream
    if prec != "fp32":
        m.set_option("streams", 1)
        one = np.stack(m.get_angle(bench_crops), axis=1)
        assert np.array_equal(one, got)
    m.close()


@pytest.mark.parametrize("prec,tol", [("fp32", 0.01), ("bf16", 0.6)])
def test_batch32_random_uint8_vs_cpu_port(prec, tol, bench_crops, bench_ref):
    """configs[1]: batch 32."""
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=32)
    got = np.stack(m.get_angle(bench_crops[100:132]), axis=1)
    err = np.abs(got - bench_ref[100:132]).max()
    print("%s N=32: max |angle - cpu port| = %.5f deg" % (prec, err))
    assert err <= tol
    m.close()


@pytest.mark.parametrize("prec,tol", [("bf16", 0.8), ("fp16", 0.05)])
def test_sample_angles_16bit_tight(prec, tol, sample_crops, jitter_crops, golden):
    """Sample/ + jitter crops.  bf16: the eight crops' worst angle moved between 0.30 and 0.62 deg over the kernel routes of
    round 2 while every block-boundary tap got closer to the oracle (the angle error is rounding noise of ~50 bf16 tensors
    pushed through three softmax expectations, not a bias) - bound 0.8; fp16: 0.018-0.03 deg - bound 0.05."""
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


def test_decode_hook_extreme_logits():
    """The device softmax/expectation (the head kernel's own device function) against reference utils.py:7-11 +
    whenet.py:31-33 on logits a float32 exp() overflows on without the max subtraction."""
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="fp32", max_batch=8)
    rng = np.random.default_rng(5)
    rows = []
    rows.append(np.full(252, 1e4, np.float32))                    # all huge and equal -> uniform
    rows.append(np.full(252, -1e4, np.float32))
    r = np.full(252, -1e4, np.float32); r[[7, 120 + 65, 186 + 0]] = 1e4; rows.append(r)      # one-hot at the extremes
    r = rng.uniform(-1e4, 1e4, 252).astype(np.float32); rows.append(r)
    r = rng.normal(0, 3, 252).astype(np.float32); rows.append(r)
    r = (rng.normal(0, 3, 252) + 9e3).astype(np.float32); rows.append(r)                     # large common offset
    r = np.zeros(252, np.float32); r[50] = 88.0; r[51] = 88.5; rows.append(r)                # exp(88.x) ~ FLT_MAX
    logits = np.stack(rows)
    got = m.debug_decode(logits)
    ref = np.stack(wo.decode(logits[:, :120].copy(), logits[:, 120:186].copy(), logits[:, 186:].copy()), axis=1)
    assert np.isfinite(got).all()
    assert np.abs(got - ref).max() < 2e-3, (got, ref)
    assert abs(got[0, 0] - (59.5 * 3 - 180)) < 1e-3 and abs(got[2, 0] - (7 * 3 - 180)) < 1e-3
    assert abs(got[2, 1] - (65 * 3 - 99)) < 1e-3 and abs(got[2, 2] - (-99)) < 1e-3
    m.close()


@pytest.mark.parametrize("n", [8, 96])
def test_timeout_flag_reaches_every_sync_path(n, sample_crops, jitter_crops):
    """A raised mbarrier-timeout flag must fail the call that synchronises - on the single-stream path (n < 64) and on the
    two-stream path (n >= 64, the default for the benched batch), and through whenet_synchronize for device outputs."""
    import torch
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=128)
    crops = np.concatenate([sample_crops, jitter_crops] * 12)[:n]
    ok = np.stack(m.get_angle(crops), axis=1)
    m.debug_raise_timeout()
    with pytest.raises(whenet_b200.WhenetError, match="timed out"):
        m.get_angle(crops)
    again = np.stack(m.get_angle(crops), axis=1)                   # the flag was consumed: the context stays usable
    assert np.array_equal(ok, again)
    x = torch.from_numpy(crops).cuda()
    y = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    m.debug_raise_timeout()
    m.forward_device(x, y)
    with pytest.raises(whenet_b200.WhenetError, match="timed out"):
        m.synchronize()
    m.synchronize()
    m.close()


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_packed_artefact_round_trip(prec, tmp_path, sample_crops, jitter_crops):
    """SURVEY.md 8f-2: export the packed device image (BN-folded, tiled, storage-typed), construct a model from it, get
    bit-identical angles; the artefact is precision-specific and a damaged index is refused."""
    import time
    import whenet_b200
    from whenet_b200 import stlite
    crops = np.concatenate([sample_crops, jitter_crops])
    t0 = time.perf_counter()
    a = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    t_raw = time.perf_counter() - t0
    ref = np.stack(a.get_angle(crops), axis=1)
    path = str(tmp_path / ("whenet_%s.packed.safetensors" % prec))
    a.export_packed(path)
    a.close()
    t0 = time.perf_counter()
    b = whenet_b200.WHENet(path, device=0, precision=prec, max_batch=8)
    t_packed = time.perf_counter() - t0
    print("%s constructor: raw npz %.3f s, packed artefact %.3f s" % (prec, t_raw, t_packed))
    got = np.stack(b.get_angle(crops), axis=1)
    assert np.array_equal(got, ref)
    b.close()
    other = "fp32" if prec == "bf16" else "bf16"
    with pytest.raises((ValueError, whenet_b200.WhenetError)):
        whenet_b200.WHENet(path, device=0, precision=other, max_batch=8)
    z, meta = stlite.load(path)
    idx = z["index"].copy()
    idx[20] = 1 << 40
    bad = str(tmp_path / "bad.safetensors")
    stlite.save(bad, {"arena_f32": z["arena_f32"], "arena_16": z["arena_16"], "index": idx}, meta)
    with pytest.raises(whenet_b200.WhenetError):
        whenet_b200.WHENet(bad, device=0, precision=prec, max_batch=8)


def test_fp32_tensor_core_parity_mode(oracle64, oracle32, sample_crops, jitter_crops, golden):
    """fp32 storage, 1x1 convolutions on the tensor core through the bf16 hi/lo split (3 MMAs per product): the north_star tolerance
    (0.01 deg vs the float64 oracle) on tensor cores, every block boundary within 2e-4 relative of the float32 oracle,
    and agreement with the CUDA-core fp32 kernels far below that."""
    import whenet_b200
    crops = np.concatenate([sample_crops, jitter_crops])
    ref = np.array([[s["yaw"], s["pitch"], s["roll"]] for s in golden["samples"]] +
                   list(zip(golden["jitter"]["yaw"], golden["jitter"]["pitch"], golden["jitter"]["roll"])))
    m = whenet_b200.WHENet(SNAP, device=0, precision="fp32", max_batch=64)
    simt = np.stack(m.get_angle(crops), axis=1)
    n0 = m.launch_count()
    m.set_option("tensor_cores", 1)
    taps = {}
    oracle32.get_angle(crops[:2], taps)
    m.enable_taps(True)
    m.get_angle(crops[:2])
    m.enable_taps(False)
    for nm in ["stem"] + ["block%d" % i for i in range(1, 17)] + ["head", "pooled"]:
        r = taps[nm].astype(np.float64).reshape(-1)
        g = m.tap(nm).astype(np.float64)
        e = float(np.abs(g - r).max() / (np.abs(r).max() + 1e-30))
        assert e < 2e-4, (nm, e)
    got = np.stack(m.get_angle(crops), axis=1)
    err = np.abs(got - ref).max()
    print("fp32 tensor-core (split-bf16) mode: max |angle - oracle64| = %.5f deg, vs CUDA-core fp32 kernels %.5f deg" % (err, np.abs(got - simt).max()))
    assert err <= 0.01
    assert np.abs(got - simt).max() <= 5e-3
    big = np.concatenate([crops] * 8)
    many = np.stack(m.get_angle(big), axis=1)
    assert np.array_equal(many[:8], got)            # batch invariant as well
    m.close()
