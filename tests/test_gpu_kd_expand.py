"""KD with the expand conv on chip (dwse_x_kernel, blocks 7-16 in bf16 at throughput batches) against the split route that
small batches take (expand GEMM writing fp16 E + KD reading it).  Both compute every E element with the expand GEMM's
arithmetic, so depthwise outputs, gates, block outputs and angles must agree bit for bit."""
import numpy as np
import pytest

from conftest import SNAP

pytestmark = pytest.mark.gpu

LATE = range(7, 17)


def _crops(sample_crops, jitter_crops, n):
    rng = np.random.default_rng(7)
    base = np.concatenate([sample_crops, jitter_crops]).astype(np.float32)
    reps = -(-n // len(base))
    crops = np.concatenate([base] * reps)[:n]
    # per-crop brightness / noise so that no two crops of the batch are equal
    crops = crops * rng.uniform(0.6, 1.2, (n, 1, 1, 1)) + rng.normal(0, 6, crops.shape)
    return np.clip(crops, 0, 255).astype(np.uint8)


def _taps(m):
    return {"%s%d" % (k, i): m.tap("%s%d" % (k, i)) for i in LATE for k in ("dw", "gate", "block")}


@pytest.mark.parametrize("kd_tail", [0, 1])
def test_on_chip_expand_matches_split_route(sample_crops, jitter_crops, kd_tail):
    """256 crops in one pass (one CTA per crop, E on chip) against 8-crop passes (chunks split over CTAs, E through memory);
    the dw / gate / block taps (recorded for passes of at most 8 crops) with the on-chip route forced at 8 crops."""
    import whenet_b200
    n, part = 256, 8
    crops = _crops(sample_crops, jitter_crops, n)
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=n)
    m.set_option("streams", 1)
    m.set_option("chunk", n)
    m.set_option("kd_tail", kd_tail)
    whole = np.stack(m.get_angle(crops), axis=1)
    parts = np.concatenate([np.stack(m.get_angle(crops[i:i + part]), axis=1) for i in range(0, n, part)])
    assert np.array_equal(whole, parts)
    m.enable_taps(True)
    for i in (0, 120, 248):
        sub = crops[i:i + part]
        m.set_option("k1_split_ctas", 120)                   # 8 crops: chunks split over CTAs -> expand GEMM + KD
        split = np.stack(m.get_angle(sub), axis=1)
        split_taps = _taps(m)
        m.set_option("k1_split_ctas", 0)                     # one CTA per crop -> expand on chip
        fused = np.stack(m.get_angle(sub), axis=1)
        fused_taps = _taps(m)
        assert np.array_equal(fused, split) and np.array_equal(fused, whole[i:i + part])
        for k, v in fused_taps.items():
            assert np.array_equal(v, split_taps[k]), (i, k)
    m.close()


def _late_launches(m, crops):
    m.enable_profile(True)
    ang = np.stack(m.get_angle(crops), axis=1)
    st = m.read_profile()
    m.enable_profile(False)
    late = {s["name"]: s["launches"] for s in st if s["name"][:1] == "b" and int(s["name"][1:3]) in LATE}
    return ang, late


def test_on_chip_expand_launches(sample_crops, jitter_crops):
    """A pass of 128 crops: blocks 7-16 launch ten kernels fewer than the same pass with the expand GEMMs (chunk split forced:
    KD + se_gate + project per block instead of expand + KD + se_gate + project); same angles."""
    import whenet_b200
    n = 128
    crops = _crops(sample_crops, jitter_crops, n)
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=n)
    m.set_option("streams", 1)
    m.set_option("chunk", n)
    fused, late_fused = _late_launches(m, crops)
    m.set_option("k1_split_ctas", 1 << 20)                   # every late block splits its chunks -> expand GEMM + KD
    split, late_split = _late_launches(m, crops)
    m.close()
    assert not any(k.endswith(".expand") for k in late_fused)
    assert sum(late_split.values()) - sum(late_fused.values()) == 10
    assert np.array_equal(fused, split)
