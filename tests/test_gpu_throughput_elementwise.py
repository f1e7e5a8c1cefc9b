"""The throughput forward (bench.py's configuration: max_batch = chunk = n, fused kernels, two streams, device-resident
uint8 input) checked element by element on selected crops, through faithful taps (mode 2: the launches and kernel
parameters of the untapped call).

(a) taps change nothing: angles, logits, launch count and profile layer names are those of the untapped call;
(b) every stage of every selected crop is within 2 B of float64 on its own GPU input (tests/elementwise_check.py);
(c) every tap of a selected crop is bit-identical to the same crop run in a batch of 8 on the small-batch route;
(d) crop selection and staleness of taps.

The crops are picked where the schedule has its edges (first and last crop of each half, the last group of four of the
batched SE and head kernels, K2 tiles shared by two crops, K1X's persistent round boundaries), computed from the SM count.
The float-input forward is checked bitwise against the uint8 forward at the end.
"""
import os

import numpy as np
import pytest

import elementwise_check as ec
import whenet_bounds as wb
from conftest import GOLD, SNAP

pytestmark = pytest.mark.gpu

# config: (precision, options, n, arithmetic)
CONFIGS = {
    "bf16_512": ("bf16", {}, 512, wb.BF16),
    "bf16_509": ("bf16", {}, 509, wb.BF16),
    "fp16_512": ("fp16", {}, 512, wb.FP16),
    "fp32_cuda_512": ("fp32", {"tensor_cores": 0}, 512, wb.FP32_CUDA),
    "fp32_split_512": ("fp32", {"tensor_cores": 1}, 512, wb.FP32_SPLIT),
    "bf16_kd_tail_512": ("bf16", {"kd_tail": 1}, 512, wb.BF16),
}
RATIOS = {}
_RUNS = {}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _specials():
    s = np.load(os.path.join(GOLD, "sample_crops.npy"))
    j = np.load(os.path.join(GOLD, "jitter_crops.npy"))[:2]
    yy, xx = np.mgrid[0:224, 0:224]
    cb = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], 3, axis=3)
    z = np.zeros((1, 224, 224, 3), np.uint8)
    return np.concatenate([s, j, z, z + 255, cb])


def _batch(n, sel, seed):
    """Uniform random crops (bench.py's distribution) with the Sample, jitter, all-0, all-255 and checkerboard crops at
    the first selected positions."""
    x = np.random.default_rng(seed).integers(0, 256, (n, 224, 224, 3), dtype=np.uint8)
    sp = _specials()
    for c, v in zip(sel, sp):
        x[c] = v
    return x


def _model(prec, opts, n, streams=2):
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=n)
    m.set_option("chunk", n)
    m.set_option("fused", 1)
    m.set_option("streams", streams)
    for k, v in opts.items():
        m.set_option(k, v)
    return m


def _forward(m, xd, n):
    """Device-resident forward: angles, logits, launch count delta, profile layer names (a separate profiled call)."""
    import torch
    ang = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    lg = torch.empty((n, 252), dtype=torch.float32, device="cuda")
    l0 = m.launch_count()
    m.forward_device(xd, ang, lg)
    m.synchronize()
    launches = m.launch_count() - l0
    out = (ang.cpu().numpy(), lg.cpu().numpy(), launches)
    m.enable_profile(True)
    m.forward_device(xd, ang, lg)
    m.synchronize()
    names = sorted(p["name"] for p in m.read_profile())
    m.enable_profile(False)
    return out + (names,)


def _run(config):
    """One GPU pass per configuration, shared by (a), (b) and (c)."""
    if config in _RUNS:
        return _RUNS[config]
    import torch
    prec, opts, n, _a = CONFIGS[config]
    sel = ec.select_crops(n, _sms(), prec == "bf16")
    x = _batch(n, sel, 1000 + n)
    xd = torch.from_numpy(x).cuda()
    m = _model(prec, opts, n)
    try:
        plain = _forward(m, xd, n)
        m.enable_taps(True, faithful=True, crops=sel)
        tapped = _forward(m, xd, n)
        taps = ec.read_taps(m, len(sel))
    finally:
        m.close()
    _RUNS[config] = dict(sel=sel, x=x[sel], plain=plain, tapped=tapped, taps=taps)
    return _RUNS[config]


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield RATIOS
    ec.print_table(RATIOS, "throughput batches, selected crops: worst |got - ref| / B per tap kind (assertion: <= 2)")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_taps_change_nothing(config):
    r = _run(config)
    (a0, l0, n0, names0), (a1, l1, n1, names1) = r["plain"], r["tapped"]
    print("%s: selected crops %s, %d launches per call" % (config, r["sel"], n0))
    assert np.isfinite(a0).all() and np.isfinite(l0).all()
    assert np.array_equal(a0, a1) and np.array_equal(l0, l1), config
    assert n0 == n1, (config, n0, n1)
    assert names0 == names1, config
    if config == "bf16_512":
        assert n0 == 2 * 52, n0                              # DESIGN §4: two concurrent passes of 52 launches
    sizes = {k: v.shape[0] for k, v in r["taps"].items()}
    assert set(sizes.values()) == {len(r["sel"])}, sizes
    assert sum(k.startswith("dw") for k in r["taps"]) == 16


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_stage_within_bound(config, oracle64):
    r = _run(config)
    prec, _opts, _n, a = CONFIGS[config]
    taps = r["taps"]
    ang = r["tapped"][0][r["sel"]]

    def get(name):
        v = taps.get(name)
        return None if v is None else v.reshape(-1)
    RATIOS[config] = ec.check_stages(config, get, r["x"], ang, a, oracle64, oracle64.stage_layers()["blocks"], {})
    if config == "fp16_512" or config == "bf16_kd_tail_512":
        assert any(k.startswith("dwg") for k in taps), config     # the in-place gated tails ran and were checked


def _small_batch_taps(config, x):
    """The crops x in batches of 8 on the small-batch route (same precision and options, default chunking)."""
    prec, opts, _n, _a = CONFIGS[config]
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=8)
    for k, v in opts.items():
        m.set_option(k, v)
    m.enable_taps(True, faithful=True)
    out = {}
    try:
        for i in range(0, len(x), 8):
            m.get_angle(x[i:i + 8])
            for k, v in ec.read_taps(m, len(x[i:i + 8])).items():
                out.setdefault(k, []).append(v)
    finally:
        m.close()
    return {k: np.concatenate(v) for k, v in out.items()}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_taps_batch_invariant(config):
    """Bit for bit against the same crops at a batch of 8.  A block whose depthwise output is gated in place on one side
    only is compared through round16(float32(d) * float32(g)), which is what the in-place gate computes."""
    r = _run(config)
    a = CONFIGS[config][3]
    big = r["taps"]
    small = _small_batch_taps(config, r["x"])
    bad = ec.taps_mismatch(big, small, a.store)
    assert not bad, (config, bad)


def test_tap_selection_and_staleness():
    import torch
    from whenet_b200 import WhenetError
    n = 70
    x = _batch(n, [], 7)
    xd = torch.from_numpy(x).cuda()
    m = _model("bf16", {}, n)
    try:
        ang = torch.empty((n, 3), dtype=torch.float32, device="cuda")
        m.enable_taps(True, faithful=True)
        m.forward_device(xd, ang)
        m.synchronize()
        full = ec.read_taps(m, n)
        assert all(v.shape[0] == n for v in full.values())
        sel = [69, 3, 35, 34, 0]                              # both halves (35 + 35), out of order
        m.enable_taps(True, faithful=True, crops=sel)
        m.forward_device(xd, ang)
        m.synchronize()
        part = ec.read_taps(m, len(sel))
        assert sorted(part) == sorted(full)
        for k, v in part.items():
            assert np.array_equal(v, full[k][sel]), k
        # an index outside the call: refused before the first launch
        m.enable_taps(True, faithful=True, crops=[1, n])
        l0 = m.launch_count()
        with pytest.raises(WhenetError):
            m.forward_device(xd, ang)
        assert m.launch_count() == l0
        with pytest.raises(WhenetError):                       # the refused call invalidated the earlier taps
            m.tap("stem")
        # taps off: the next forward leaves no tap to read
        m.enable_taps(True, faithful=True, crops=[2])
        m.forward_device(xd, ang)
        m.synchronize()
        assert m.tap("stem").size == 112 * 112 * 32
        m.enable_taps(False)
        m.forward_device(xd, ang)
        m.synchronize()
        with pytest.raises(WhenetError):
            m.tap("stem")
        # mode 1 records at most 8 crops: a 70-crop call leaves nothing
        m.enable_taps(True)
        m.forward_device(xd, ang)
        m.synchronize()
        with pytest.raises(WhenetError):
            m.tap("block3")
        m.forward_device(xd[:5], ang)
        m.synchronize()
        from whenet_b200 import arch
        b3 = arch.blocks()[2]
        assert m.tap("block3").size == 5 * b3.hout * b3.hout * b3.cout
    finally:
        m.close()


FLOAT_MODES = {"fp32_cuda": ("fp32", {"tensor_cores": 0}), "fp32_split": ("fp32", {"tensor_cores": 1}),
               "bf16": ("bf16", {}), "fp16": ("fp16", {})}


@pytest.mark.parametrize("mode", list(FLOAT_MODES))
def test_float_input_bitwise(mode):
    """The device LUT and get_angle's host normalisation are the same float64 recipe cast to float32, so the float-input
    forward (whenet_forward_f32, the stem's float branch) must give the uint8 forward's bits: at 2 crops, at 70 (two
    streams, staged 4-byte upload) with and without staging threads, past max_batch, and through model.predict."""
    import whenet_b200
    from whenet_oracle import preprocess
    prec, opts = FLOAT_MODES[mode]
    x = _batch(90, [0, 1, 2, 3, 4, 5, 6], 5)
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=80)
    try:
        for k, v in opts.items():
            m.set_option(k, v)
        for threads in (0, 8):
            m.set_option("stage_threads", threads)
            for n in (2, 70, 90):
                u8 = np.stack(m.get_angle(x[:n]), axis=1)
                fl = np.stack(m.get_angle(x[:n].astype(np.float64)), axis=1)
                assert np.isfinite(u8).all()
                assert np.array_equal(u8, fl), (mode, threads, n)
        _ang, lg = m._forward(np.ascontiguousarray(x[:70]), want_logits=True)
        pr = np.concatenate(m.model.predict(preprocess(x[:70])), axis=1)
        assert np.array_equal(lg, pr), mode
    finally:
        m.close()
