"""The 1x1-convolution kernels alone, every (K, N) pair of the network: CUDA-core (use_tc=0), pw_tc2 (2: one tile per
CTA, cp.async ring) and K2 (3: persistent, TMA, warp-specialised).

Reference for both families: numpy float64 on the SAME 16-bit-rounded inputs, so the only
differences are fp32 accumulation order and the final rounding to the storage type."""
import numpy as np
import pytest

from conftest import SNAP

pytestmark = pytest.mark.gpu


def _bf16_round(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def _layer_shapes():
    from whenet_b200 import arch
    shapes = set()
    for b in arch.blocks():
        if b.has_expand:
            shapes.add((b.cin, b.cexp, "expand"))
        shapes.add((b.cexp, b.cout, "project_res" if b.skip else "project"))
    shapes.add((320, 1280, "expand"))
    return sorted(shapes)


@pytest.fixture(scope="module")
def net():
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision="bf16", max_batch=8)
    yield m
    m.close()


@pytest.mark.parametrize("use_tc", [0, 2, 3])
@pytest.mark.parametrize("K,N,kind", _layer_shapes())
def test_conv1x1_shapes(net, use_tc, K, N, kind):
    rng = np.random.default_rng(K * 1000 + N)
    hw = 49
    M = 5 * hw + 17            # ragged: not a multiple of 128 nor of hw
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    gate = resid = None
    swish = kind == "expand"
    if kind.startswith("project"):
        gate = rng.uniform(0.1, 1.0, ((M + hw - 1) // hw, K)).astype(np.float32)
    if kind == "project_res":
        resid = _bf16_round(rng.standard_normal((M, N)))
    got = net.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, swish=swish, use_tc=use_tc)
    Ag = A.astype(np.float64)
    if gate is not None:
        Ag = Ag * np.repeat(gate, hw, axis=0)[:M]
        if use_tc:
            Ag = _bf16_round(Ag).astype(np.float64)   # the tensor-core path rounds A*gate back to bf16 in smem
    ref = Ag @ W.astype(np.float64) + bias
    if swish:
        ref = ref / (1.0 + np.exp(-ref))
    if resid is not None:
        ref = ref + resid
    err = np.abs(got - ref)
    tol = 2.0 ** -7 * np.abs(ref) + 2e-2          # one bf16 rounding of the output (2^-8 rel) + accumulation noise
    assert np.all(err <= tol), (K, N, kind, float(err.max()), int(np.argmax(err - tol)))


@pytest.mark.parametrize("K,N,res", [(32, 16, False), (96, 24, False), (144, 24, True), (144, 40, False), (240, 40, True)])
def test_conv1x1_per_crop_gate_on_weights(net, K, N, res):
    """hw >= 784: the cp.async kernel tiles per crop and folds the SE gate into the W rows in shared memory."""
    rng = np.random.default_rng(K + N)
    hw, crops = 784, 3
    M = hw * crops
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    gate = rng.uniform(0.1, 1.0, (crops, K)).astype(np.float32)
    resid = _bf16_round(rng.standard_normal((M, N))) if res else None
    got = net.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, use_tc=2)
    ref = np.empty((M, N))
    for c in range(crops):
        Wg = _bf16_round(W * gate[c][:, None]).astype(np.float64)       # the kernel rounds W*gate back to bf16
        ref[c * hw:(c + 1) * hw] = A[c * hw:(c + 1) * hw].astype(np.float64) @ Wg + bias
    if res:
        ref = ref + resid
    err = np.abs(got - ref)
    tol = 2.0 ** -7 * np.abs(ref) + 2e-2
    assert np.all(err <= tol), (K, N, float(err.max()))


@pytest.mark.parametrize("M", [1, 127, 128, 129, 1000])
def test_conv1x1_tc_row_tails(net, M):
    rng = np.random.default_rng(M)
    K, N = 96, 24
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = np.zeros(N, np.float32)
    b = net.debug_conv1x1(A, W, bias, use_tc=0)
    for fam in (2, 3):
        a = net.debug_conv1x1(A, W, bias, use_tc=fam)
        assert np.abs(a - b).max() <= 2.0 ** -6 * max(1.0, np.abs(b).max())


@pytest.mark.parametrize("use_tc", [0, 2, 3])
@pytest.mark.parametrize("K,N", [(480, 80), (1152, 192)])
def test_conv1x1_residual_without_gate(net, use_tc, K, N):
    """Project conv of a block whose depthwise output was already gated by K1's tail: bias + residual, no gate."""
    rng = np.random.default_rng(K + N)
    M = 5 * 49 + 17
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    resid = _bf16_round(rng.standard_normal((M, N)))
    got = net.debug_conv1x1(A, W, bias, gate=None, resid=resid, hw=49, swish=False, use_tc=use_tc)
    ref = A.astype(np.float64) @ W.astype(np.float64) + bias + resid
    assert np.abs(got - ref).max() <= 2.5e-2 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("K,N,hw,res", [(96, 24, 3136, False), (240, 40, 784, True), (480, 80, 196, True), (1152, 192, 49, True),
                                        (1152, 320, 49, False), (320, 1280, 49, None)])
def test_k2_persistent_many_tiles(net, K, N, hw, res):
    """K2 with more tiles than CTAs (every CTA loops over several tiles: ring wrap-around, both MMA warpgroups, gate rows
    reloaded when a tile changes crop), resident and streamed weights, two n tiles (N = 320) and the swish head conv (N = 1280)."""
    rng = np.random.default_rng(K + N)
    M = 2 * 132 * 128 + 3 * 128 + 77
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    head = res is None
    gate = None if head else rng.uniform(0.1, 1.0, ((M + hw - 1) // hw, K)).astype(np.float32)
    resid = _bf16_round(rng.standard_normal((M, N))) if res else None
    got = net.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, swish=head, use_tc=3)
    Ag = A.astype(np.float64)
    if gate is not None:
        Ag = _bf16_round(Ag * np.repeat(gate, hw, axis=0)[:M]).astype(np.float64)
    ref = Ag @ W.astype(np.float64) + bias
    if head:
        ref = ref / (1.0 + np.exp(-ref))
    if resid is not None:
        ref = ref + resid
    err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= 2.0 ** -7, err
    if M % hw == 0 or hw < 784:        # pw_tc2 tiles gated layers per crop while H*W >= 784 and then needs whole crops
        two = net.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, swish=head, use_tc=2)
        assert np.abs(got - two).max() <= 2.0 ** -6 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("K,N,kind", [(16, 96, "expand"), (96, 24, "project"), (144, 24, "project_res"), (672, 192, "project"), (1152, 320, "project"), (320, 1280, "expand")])
def test_conv1x1_fp32_split_bf16(K, N, kind):
    """fp32 parity mode on the tensor core: x = hi + lo bf16 split, three MMAs per product, fp32 accumulation - against
    float64 on the unrounded fp32 inputs (the CUDA-core fp32 kernel is the second reference)."""
    import whenet_b200
    m = whenet_b200.WHENet(None, device=0, precision="fp32", max_batch=8)
    rng = np.random.default_rng(K + N)
    hw = 49
    M = 5 * hw + 17
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    gate = resid = None
    swish = kind == "expand"
    if kind.startswith("project"):
        gate = rng.uniform(0.1, 1.0, ((M + hw - 1) // hw, K)).astype(np.float32)
    if kind == "project_res":
        resid = rng.standard_normal((M, N)).astype(np.float32)
    got = m.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, swish=swish, use_tc=1)
    simt = m.debug_conv1x1(A, W, bias, gate=gate, resid=resid, hw=hw, swish=swish, use_tc=0)
    Ag = A.astype(np.float64)
    if gate is not None:
        Ag = (A * np.repeat(gate, hw, axis=0)[:M]).astype(np.float64)      # the product is formed in fp32 on the device
    ref = Ag @ W.astype(np.float64) + bias
    if swish:
        ref = ref / (1.0 + np.exp(-ref))
    if resid is not None:
        ref = ref + resid
    scale = max(1.0, np.abs(ref).max())
    assert np.abs(got - ref).max() <= 3e-5 * scale, np.abs(got - ref).max()
    assert np.abs(got - simt).max() <= 3e-5 * scale
    m.close()


def test_pw_tc3_matches_pw_tc2_bitwise(net):
    """pw_tc3 (a CTA walks several 128-row tiles of one crop: gate row and W' = 16-bit(W * g) once per CTA, two-deep pipeline over
    the tiles) must give the bits of pw_tc2's per-crop route on the block-1 project shape, every tile of every group - the
    second-to-last tile of a group once raced with the last one for the staging buffer."""
    K, N, hw, crops = 32, 16, 12544, 70
    rng = np.random.default_rng(K + N)
    M = crops * hw
    A = _bf16_round(rng.standard_normal((M, K)))
    W = _bf16_round(rng.standard_normal((K, N)) / np.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    gate = rng.uniform(0.1, 1.0, (crops, K)).astype(np.float32)
    a = net.debug_conv1x1(A, W, bias, gate=gate, hw=hw, swish=False, use_tc=5)
    b = net.debug_conv1x1(A, W, bias, gate=gate, hw=hw, swish=False, use_tc=2)
    assert np.array_equal(a, b)
    ref = _bf16_round(A.astype(np.float64) * np.repeat(gate, hw, axis=0)).astype(np.float64)      # A-side rounding: a bound, not the kernel's W-side rounding
    ref = ref @ W.astype(np.float64) + bias
    assert np.abs(a - ref).max() <= 3e-2 * max(1.0, np.abs(ref).max())
