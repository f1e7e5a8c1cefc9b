"""Tiny YOLOv3 head detector, everything that runs without a GPU: the layer table and its counts, the two float64 body
restatements against each other, the max-pool's SAME padding, weight mapping and the two-head decode restatement."""
import ctypes as C

import numpy as np
import pytest

import yolo_oracle as O
import yolo_tiny_cases as TC
import yolo_tiny_oracle as TO
from whenet_b200 import yolo_arch as Y

SIDES = range(32, 609, 32)


def test_tiny_table_and_counts():
    T = Y.TINY_LAYERS
    assert Y.TINY_N_CONV == 13 and sum(L.bn for L in T) == 11
    assert Y.TINY_HEADS == [11, 12] and Y.TINY_ANCHOR_MASK == [[3, 4, 5], [1, 2, 3]]
    assert [L.pool for L in T] == [0, 2, 2, 2, 2, 2, 1, 0, 0, 0, 0, 0, 0]
    assert [L.keras_id for L in T] == [1, 2, 3, 4, 5, 6, 7, 8, 11, 9, 12, 10, 13]
    assert T[10].up == 8 and T[10].src == 4 and T[10].c_up == 128 and T[10].k == 3 and T[10].cin == 384
    assert Y.macs_per_frame(416, 416, tiny=True) == 2_720_959_488
    assert abs(2 * Y.macs_per_frame(608, 608, tiny=True) / 1e9 - 11.62) < 0.005
    assert Y.num_candidates(416, 416, tiny=True) == 2535 and Y.num_candidates(32, 32, tiny=True) == 15
    assert Y.num_candidates(608, 608, tiny=True) == 5415
    # the full model's defaults are untouched
    assert Y.macs_per_frame(416, 416) == Y.macs_per_frame(416, 416, tiny=False) and Y.num_candidates(416, 416) == 10647


@pytest.mark.parametrize("h", SIDES)
def test_tiny_out_hw_at_every_size(h):
    for w in SIDES:
        gh, gw = h // 32, w // 32
        want = [(h >> i, w >> i) for i in range(6)] + [(gh, gw)] * 4 + [(2 * gh, 2 * gw), (gh, gw), (2 * gh, 2 * gw)]
        assert Y.out_hw(h, w, tiny=True) == want, (h, w)
        ins = Y.in_hw(h, w, tiny=True)
        assert ins[6] == (gh, gw) and ins[1] == (h // 2, w // 2)


def test_numpy_tiny_body_equals_torch_tiny_body():
    names, w = Y.random_weights(3, tiny=True)
    layers, _ = Y.map_weights(names, w, tiny=True)
    for shape in ((1, 64, 96, 3), (2, 32, 32, 3)):
        x = np.random.default_rng(1).random(shape)
        outs = TO.body_numpy(x, layers)
        heads_t = TO.body_torch(x, layers)
        assert len(heads_t) == 2
        for i, t in zip(Y.TINY_HEADS, heads_t):
            assert outs[i].shape == t.shape
            assert np.abs(outs[i] - t).max() <= 1e-9 * np.abs(t).max(), i
            assert 0.01 < np.abs(t).max() < 50          # the output convs are small by design (random_weights)


def _pool_loop(x, s):
    n, H, W, C = x.shape
    Ho, Wo = -(-H // s), -(-W // s)
    out = np.empty((n, Ho, Wo, C))
    for y in range(Ho):
        for xx in range(Wo):
            out[:, y, xx] = x[:, y * s:min(y * s + 2, H), xx * s:min(xx * s + 2, W)].max(axis=(1, 2))
    return out


@pytest.mark.parametrize("hw", [(13, 13), (6, 8), (7, 12), (1, 1)])
@pytest.mark.parametrize("stride", [1, 2])
def test_maxpool_same_equals_a_loop(hw, stride):
    x = np.random.default_rng(hw[0] * 31 + hw[1]).standard_normal((2,) + hw + (8,))
    assert np.array_equal(TO.maxpool_same(x, stride), _pool_loop(x, stride))


def test_stride1_pool_padding_never_wins():
    """On an all-negative input the last row and column of the stride-1 pool are the max of the real cells, not 0 (a zero
    pad) - in the numpy pool and in the torch body's F.pad(value=-inf) + F.max_pool2d."""
    import torch
    import torch.nn.functional as F
    x = -1.0 - np.random.default_rng(0).random((1, 13, 13, 16))
    p = TO.maxpool_same(x, 1)
    assert p.shape == x.shape and (p < 0).all()
    assert np.array_equal(p[:, 12, :12], np.maximum(x[:, 12, :12], x[:, 12, 1:]))
    assert np.array_equal(p[:, :12, 12], np.maximum(x[:, :12, 12], x[:, 1:, 12]))
    assert np.array_equal(p[:, 12, 12], x[:, 12, 12])
    t = torch.from_numpy(x).permute(0, 3, 1, 2)
    tp = F.max_pool2d(F.pad(t, (0, 1, 0, 1), value=-np.inf), 2, stride=1).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(tp, p)


# ----------------------------------------------------------------------------------------------- weight mapping
def test_tiny_weights_round_trip_and_offset_numbering():
    names, w = Y.random_weights(5, tiny=True)
    assert len(names) == 13 + 11
    assert [n for n in names if n.startswith("batch")] == ["batch_normalization_%d" % i for i in (1, 2, 3, 4, 5, 6, 7, 8, 10, 9, 11)]
    ref, C = Y.map_weights(names, w, tiny=True)
    assert C == 1 and len(ref) == 13
    for L, d in zip(Y.TINY_LAYERS, ref):
        assert d["name"] == "conv2d_%d" % L.keras_id
        assert np.array_equal(d["kernel"], w["conv2d_%d/kernel:0" % L.keras_id])

    def shift(n):
        base, _, rest = n.partition("/")
        kind, _, num = base.rpartition("_")
        return "%s_%d%s%s" % (kind, int(num) + 100, "/" if rest else "", rest)
    got, _ = Y.map_weights([shift(n) for n in names], {shift(k): v for k, v in w.items()}, tiny=True)
    for a, b in zip(ref, got):
        for k in a:
            if k != "name":
                assert np.array_equal(a[k], b[k])


def test_tiny_weight_mapping_refuses_bad_files():
    names, w = Y.random_weights(6, tiny=True)
    with pytest.raises(ValueError, match="expected 75 conv layers for YOLOv3.*has 13"):
        Y.map_weights(names, w)                                             # a tiny file given 9 anchors
    fn, fw = Y.random_weights(6)
    with pytest.raises(ValueError, match="expected 13 conv layers for tiny YOLOv3.*has 75"):
        Y.map_weights(fn, fw, tiny=True)                                    # a full file given 6 anchors
    w1 = {k: v for k, v in w.items() if not k.startswith("batch_normalization_9/")}
    with pytest.raises(ValueError, match="expected 11 BatchNormalization layers for tiny YOLOv3.*has 10"):
        Y.map_weights([n for n in names if n != "batch_normalization_9"], w1, tiny=True)
    swapped = list(names)
    i, j = swapped.index("conv2d_9"), swapped.index("conv2d_12")
    swapped[i], swapped[j] = swapped[j], swapped[i]
    with pytest.raises(ValueError, match=r"conv2d_12 \(conv 9\): kernel shape"):
        Y.map_weights(swapped, w, tiny=True)


def test_yolo_picks_the_network_from_the_anchor_count(tmp_path):
    import whenet_b200
    assert Y.read_anchors(TC.ANCHORS).shape == (6, 2)
    p = tmp_path / "seven.txt"
    p.write_text(",".join(str(v) for v in range(14)))
    with pytest.raises(ValueError, match="9 anchors and tiny YOLOv3 6.*has 7"):
        whenet_b200.YOLO(anchors_path=str(p))


# ----------------------------------------------------------------------------------------------- two-head decode
def test_two_head_decode_uses_anchors_345_and_123():
    """Zero logits: every box is its anchor's size in the 416 x 416 frame, so the widths and heights name the anchors."""
    anchors = Y.read_anchors(TC.ANCHORS)
    heads = [np.zeros((13 << l, 13 << l, 18), np.float32) for l in range(2)]
    boxes, scores = TO.decode(heads, anchors, 1, 416, 416)
    assert boxes.shape == (2535, 4) and np.all(scores == np.float32(0.25))
    hw = np.stack([boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]], 1).reshape(-1, 3, 2)
    for l, (lo, hi) in enumerate(((0, 507), (507, 2535))):
        want = anchors[Y.TINY_ANCHOR_MASK[l]][:, ::-1]          # (h, w)
        assert np.allclose(hw[lo // 3:hi // 3], want[None], rtol=1e-5), l
    # three heads keep the full model's mask
    full = [np.zeros((13 << l, 13 << l, 18), np.float32) for l in range(3)]
    fb, _ = O.decode(full, Y.DEFAULT_ANCHORS, 1, 416, 416)
    assert np.allclose(fb[0, 2:] - fb[0, :2], Y.DEFAULT_ANCHORS[6, ::-1], rtol=1e-5)


def test_detector_refuses_other_anchor_counts_without_gpu():
    from whenet_b200 import _lib
    L = _lib.load()
    a = np.zeros(14, np.float32)
    assert L.whenet_det_load_weights(None, None, 0, a.ctypes.data_as(C.c_void_p), 7) == -1
    assert b"9 anchors and tiny YOLOv3 6, got 7" in L.whenet_last_error()
    assert L.whenet_det_load_weights(None, None, 0, a.ctypes.data_as(C.c_void_p), 6) == -1
    assert b"bad arguments" in L.whenet_last_error()
    assert L.whenet_det_debug_maxpool(None, None, 1, 13, 13, 16, 1, None) == -1
