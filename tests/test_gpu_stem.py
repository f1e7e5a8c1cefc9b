"""The register-blocked stem against the one-pixel-per-thread kernel it replaced, bit for bit.

tests/stem_reference.cu is that kernel, verbatim, compiled here with the library's nvcc flags.  Every output keeps its own
fp32 FMA chain in the same order (bias, then (ky, kx, ci), padding taps included), so the library's stem tap (faithful taps:
the launches of the untapped call) must equal the reference's output exactly, for uint8 and float input, in each storage
mode the stem writes (fp16 in bf16 mode, bf16 with dw1_kd=0, fp16, fp32), at 1, 7, 70 and 512 crops (two streams).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLD, ROOT, SNAP

pytestmark = pytest.mark.gpu

# mode: (precision, options, reference storage type: 0 fp32, 1 fp16 with the tanh swish, 2 bf16 with the tanh swish)
MODES = {
    "bf16": ("bf16", {}, 1),
    "bf16_store": ("bf16", {"dw1_kd": 0}, 2),
    "fp16": ("fp16", {}, 1),
    "fp32": ("fp32", {}, 0),
}
SIZES = [1, 7, 70, 512]


@pytest.fixture(scope="module")
def ref_lib():
    from whenet_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libstem_reference.so")
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-shared", "-o", so, os.path.join(ROOT, "tests", "stem_reference.cu")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        lib = C.CDLL(so)
    lib.stem_reference_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return lib


@pytest.fixture(scope="module")
def crops():
    """2 Sample crops, 2 jitter crops, a uniform-random crop, all-0, all-255 and a one-pixel 0/255 checkerboard."""
    s = np.load(os.path.join(GOLD, "sample_crops.npy"))
    j = np.load(os.path.join(GOLD, "jitter_crops.npy"))[:2]
    rnd = np.random.default_rng(2024).integers(0, 256, (1, 224, 224, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:224, 0:224]
    cb = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], 3, axis=3)
    return np.concatenate([s, j, rnd, np.zeros_like(rnd), np.full_like(rnd, 255), cb])


def _stem_params(m):
    """The BN-folded stem weights, shifts and LUT the library launches with (its packed device image)."""
    sizes = (C.c_int64 * 3)()
    assert m._L.whenet_export_packed(m._h, None, None, None, sizes) == 0
    a32 = np.empty((sizes[0],), np.float32)
    idx = np.empty((sizes[2],), np.int64)
    assert m._L.whenet_export_packed(m._h, a32.ctypes.data_as(C.c_void_p), None, idx.ctypes.data_as(C.c_void_p), sizes) == 0
    return (np.ascontiguousarray(a32[idx[5]:idx[5] + 27 * 32]), np.ascontiguousarray(a32[idx[6]:idx[6] + 32]),
            np.ascontiguousarray(a32[idx[7]:idx[7] + 768]))


def _reference(lib, x, out_type, w, b, lut):
    import torch
    dt = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16}[out_type]
    d_in = torch.from_numpy(x).cuda()
    d_out = torch.empty((x.shape[0], 112, 112, 32), dtype=dt, device="cuda")
    d_lut = torch.from_numpy(lut).cuda()
    torch.cuda.synchronize()
    rc = lib.stem_reference_launch(d_in.data_ptr(), d_out.data_ptr(), int(x.dtype == np.uint8), out_type,
                                   w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), d_lut.data_ptr(), x.shape[0])
    assert rc == 0, "reference stem: CUDA error %d" % rc
    return d_out.float().cpu().numpy()


def _selection(n):
    if n <= 64:
        return list(range(n))
    per = (n + 1) // 2                   # the two half-batch streams: both ends of each half, and a spread between
    sel = sorted({0, 1, 2, 3, 4, 5, 6, 7, per - 2, per - 1, per, per + 1, n - 2, n - 1} |
                 set(np.random.default_rng(n).choice(n, 64, replace=False).tolist()))
    return sel[:64]


@pytest.mark.parametrize("mode", list(MODES))
def test_stem_bitwise_vs_reference(mode, ref_lib, crops):
    import whenet_b200
    from whenet_oracle import preprocess
    prec, opts, out_type = MODES[mode]
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=max(SIZES))
    try:
        for k, v in opts.items():
            m.set_option(k, v)
        w, b, lut = _stem_params(m)
        for n in SIZES:
            x8 = np.ascontiguousarray(crops[np.arange(n) % len(crops)])
            xf = np.ascontiguousarray(preprocess(x8), dtype=np.float32)
            sel = _selection(n)
            for x in (x8, xf):
                m.enable_taps(True, faithful=True, crops=sel)
                m._forward(x)
                got = m.tap("stem").reshape(len(sel), 112, 112, 32)
                m.enable_taps(False)
                ref = _reference(ref_lib, x, out_type, w, b, lut)[sel]
                bad = np.argwhere(got.view(np.uint32) != ref.view(np.uint32))
                assert bad.size == 0, "%s n=%d %s: %d elements differ, first at %s (got %r, ref %r)" % (
                    mode, n, x.dtype, len(bad), bad[0].tolist(), float(got[tuple(bad[0])]), float(ref[tuple(bad[0])]))
    finally:
        m.close()
