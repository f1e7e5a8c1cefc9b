"""Persistent K1X (k1x_kernel: a grid of at most CTAs-per-SM x SMs CTAs, each walking (tile, crop) items b, b + grid, ...)
against K1 (option k1x=0), bit for bit, at batch sizes around the grid of each early block: fewer items than CTAs, one
full round, one item more or less than a round where the crop count allows it, a ragged last round, and a single crop.
The CTA's chunk counter carries the W / constants ring and the halo barrier's phase across items, so every item count
must give the same bits as one CTA per item."""
import numpy as np
import pytest

from conftest import SNAP

pytestmark = pytest.mark.gpu

EARLY = range(2, 7)
# the K1X instances: output tiles per crop and resident CTAs per SM (tests/test_k1x_occupancy_cpu.py checks the latter)
TILES = {2: 49, 3: 16, 4: 16, 6: 4}
CTAS_PER_SM = {2: 3, 3: 3, 4: 3, 6: 2}


def _batches():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {1}
    for b, t in TILES.items():
        grid = CTAS_PER_SM[b] * sms
        lo, hi = grid // t, -(-grid // t)              # items <= grid, items >= grid (equal when t divides the grid)
        out |= {lo - 1, lo, hi, hi + 1}                  # one crop less / more: items = grid -+ t (-+ 1 when t == 1)
        out.add((2 * grid) // t + 1)                     # two rounds and a ragged third
    return sorted(x for x in out if x >= 1)


def _crops(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 224, 224, 3), dtype=np.uint8)


def _model(n, streams=1, graph=0):
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=n)
    m.set_option("streams", streams)
    m.set_option("chunk", n)
    m.set_option("graph", graph)
    m.set_option("k1_split_ctas", 0)                   # one CTA holds all chunks of its tile at every batch: K1X is taken
    return m


def _per_crop():
    """Elements per crop of the dw / gate / block taps of blocks 2-6."""
    from whenet_b200 import arch
    out = {}
    for b in arch.blocks():
        if b.idx in EARLY:
            out.update({"dw%d" % b.idx: b.hout * b.hout * b.cexp, "gate%d" % b.idx: b.cexp, "block%d" % b.idx: b.hout * b.hout * b.cout})
    return out


def test_faithful_taps_bit_identical_around_the_grid():
    """One stream with faithful taps (the untapped route, every crop): the dw / gate / block taps of blocks 2-6 and the
    angles, at every batch of _batches().  Each tap must hold exactly n crops, so no tap of an earlier call can pass."""
    batches = _batches()
    per = _per_crop()
    m = _model(max(batches))
    m.enable_taps(True, faithful=True)
    for n in batches:
        crops = _crops(n, 100 + n)
        got = {}
        for route in (0, 1):
            m.set_option("k1x", route)
            ang = np.stack(m.get_angle(crops), axis=1)
            got[route] = (ang, {k: m.tap(k) for k in per})
            for k, v in got[route][1].items():
                assert v.size == n * per[k], (n, route, k, v.size)
        assert np.isfinite(got[0][0]).all() and np.array_equal(got[0][0], got[1][0]), n
        for k, v in got[0][1].items():
            assert np.array_equal(v, got[1][1][k]), (n, k)
    m.close()


def test_two_streams_bit_identical():
    """Two streams (half batches, each its own persistent grid, both resident at once): halves of n + 1 and n crops."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = sorted({2 * (CTAS_PER_SM[b] * sms // t) + 1 for b, t in TILES.items()} | {129})
    m = _model(max(ns), streams=2)
    for n in ns:
        crops = _crops(n, 200 + n)
        a = []
        for route in (0, 1):
            m.set_option("k1x", route)
            a.append(np.stack(m.get_angle(crops), axis=1))
        assert np.isfinite(a[0]).all() and np.array_equal(a[0], a[1]), n
    m.close()


def test_graph_replay_bit_identical():
    """Device-resident input and output with graphs on: the first call captures (grid sized at capture), the second replays;
    both give K1's bits."""
    import torch
    batches = [1, max(_batches())]
    m = _model(max(batches), graph=1)
    for n in batches:
        crops = torch.from_numpy(_crops(n, 300 + n)).cuda()
        a = []
        for route in (0, 1):
            m.set_option("k1x", route)
            outs = []
            ang = torch.empty((n, 3), dtype=torch.float32, device="cuda")     # the same pointers: the second call replays
            for _ in range(2):
                ang.fill_(float("nan"))
                m.forward_device(crops, ang)
                m.synchronize()
                outs.append(ang.cpu().numpy())
            assert np.array_equal(outs[0], outs[1]), (n, route)
            a.append(outs[0])
        assert np.isfinite(a[0]).all() and np.array_equal(a[0], a[1]), n
    m.close()
