"""K1X (k1x_kernel: blocks 2, 3, 4 and 6 in bf16 at throughput batches, operands by TMA) against K1 (option k1x=0).  The two
kernels share their tile plans and the device functions that hold the arithmetic, so depthwise outputs, gates, block outputs
and angles must agree bit for bit."""
import numpy as np
import pytest

from conftest import SNAP

pytestmark = pytest.mark.gpu

EARLY = range(2, 7)


def _model(n, streams=1, graph=0):
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=n)
    m.set_option("streams", streams)
    m.set_option("chunk", n)
    m.set_option("graph", graph)
    return m


def _both(m, crops):
    out = []
    for route in (0, 1):
        m.set_option("k1x", route)
        out.append(np.stack(m.get_angle(crops), axis=1))
    return out


def _taps(m):
    return {"%s%d" % (k, i): m.tap("%s%d" % (k, i)) for i in EARLY for k in ("dw", "gate", "block")}


def test_taps_bit_identical(sample_crops, jitter_crops):
    """The committed crops, with K1X forced at this small batch (no chunk split): every tap of blocks 2-6 and the angles."""
    crops = np.concatenate([sample_crops, jitter_crops])
    m = _model(len(crops))
    m.set_option("k1_split_ctas", 0)                   # one CTA per tile with all its chunks, whatever the batch
    m.enable_taps(True)
    got = {}
    for route in (0, 1):
        m.set_option("k1x", route)
        got[route] = (np.stack(m.get_angle(crops), axis=1), _taps(m))
    m.close()
    assert np.array_equal(got[0][0], got[1][0])
    for k, v in got[0][1].items():
        assert np.isfinite(v).all(), k
        assert np.array_equal(v, got[1][1][k]), k


@pytest.mark.parametrize("streams,graph", [(1, 0), (2, 0), (1, 1)])
def test_random_crops_bit_identical(streams, graph):
    crops = np.random.default_rng(11).integers(0, 256, (64, 224, 224, 3), dtype=np.uint8)
    m = _model(64, streams, graph)
    m.set_option("k1_split_ctas", 0)
    a, b = _both(m, crops)
    m.close()
    assert np.isfinite(a).all() and np.array_equal(a, b)


def test_batch_512_bit_identical_and_launches(sample_crops, jitter_crops):
    """The benchmark's batch on two streams (256-crop halves, which take K1X): same angles and the same number of
    launches as with K1; an 8-crop pass, whose chunks are split over CTAs, stays on K1 whatever the option says."""
    rng = np.random.default_rng(5)
    base = np.concatenate([sample_crops, jitter_crops]).astype(np.float32)
    crops = np.concatenate([base] * (512 // len(base) + 1))[:512]
    crops = np.clip(crops * rng.uniform(0.6, 1.2, (512, 1, 1, 1)) + rng.normal(0, 6, crops.shape), 0, 255).astype(np.uint8)
    m = _model(512, streams=2)
    counts, angles = [], []
    for route in (0, 1):
        m.set_option("k1x", route)
        m.get_angle(crops[:8])
        l0 = m.launch_count()
        angles.append(np.stack(m.get_angle(crops), axis=1))
        l1 = m.launch_count()
        m.get_angle(crops[:8])
        counts.append((l1 - l0, m.launch_count() - l1))
    m.close()
    assert np.array_equal(angles[0], angles[1])
    assert counts[0] == counts[1]
