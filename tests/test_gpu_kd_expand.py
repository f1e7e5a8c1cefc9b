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


def _taps(m, n):
    """dw (dwg where the depthwise output was gated in place) / gate / block taps of blocks 7-16, (n, elements) each."""
    from whenet_b200 import WhenetError
    out = {}
    for i in LATE:
        for k in ("dw", "gate", "block"):
            try:
                v = m.tap("%s%d" % (k, i))
            except WhenetError:
                if k != "dw":
                    raise
                k, v = "dwg", m.tap("dwg%d" % i)
            out["%s%d" % (k, i)] = v.reshape(n, -1)
    return out


def _gate16(d, g):
    """round16(float32(d) * float32(g)) in bf16: what the in-place gate of the SE tail stores."""
    import torch
    dg = d.reshape(d.shape[0], -1, g.shape[1]).astype(np.float32) * g.astype(np.float32)[:, None, :]
    return torch.from_numpy(dg).to(torch.bfloat16).float().numpy().reshape(d.shape)


@pytest.mark.parametrize("kd_tail", [0, 1])
def test_on_chip_expand_matches_split_route(sample_crops, jitter_crops, kd_tail):
    """256 crops in one pass (one CTA per crop, E on chip) against 8-crop passes (chunks split over CTAs, E through memory).
    The 256-crop pass's own dw / gate / block taps (faithful taps: the launches of the untapped pass) against those of the
    8-crop split passes.  With kd_tail=1 the 256-crop pass gates its depthwise output in place (dwg%d); the split route's
    ungated d then has to give it exactly as round16(float32(d) * float32(g))."""
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
    m.enable_taps(True, faithful=True)
    assert np.array_equal(np.stack(m.get_angle(crops), axis=1), whole)
    whole_taps = _taps(m, n)
    assert sum(k.startswith("dwg") for k in whole_taps) == (len(LATE) if kd_tail else 0), sorted(whole_taps)
    m.set_option("k1_split_ctas", 120)                       # 8 crops: chunks split over CTAs -> expand GEMM + KD
    for i in (0, 120, 248):
        split = np.stack(m.get_angle(crops[i:i + part]), axis=1)
        split_taps = _taps(m, part)
        assert np.array_equal(split, whole[i:i + part])
        for k, v in whole_taps.items():
            if k.startswith("dwg") and k not in split_taps:
                blk = int(k[3:])
                ref = _gate16(split_taps["dw%d" % blk], split_taps["gate%d" % blk])
            else:
                ref = split_taps[k]
            assert np.array_equal(v[i:i + part], ref), (i, k)
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
