"""JPEG decoding of coefficients outside an encoder's range (DESIGN.md section 8.10), without a GPU.  Files come from the
coefficient-level writer in jpeg_coef_writer.py, which is checked first against the oracle's entropy stage.  Then the numpy
IDCT model (oracle/jpeg_decode_oracle.py ``idct_islow``) is pinned against cv2.imdecode by probes that sweep one and two
coefficients over all 64 positions at dequantised values around +-2^13, +-2^14 and +-2^15: the model equals cv2 on every
probe, and each of its 16-bit steps is needed, since the model with that step replaced by an alternative differs from cv2.
Finally the model and tools/jpeg_decode_dump.cu (the kernels' own arithmetic on the CPU) equal cv2 on a seeded matrix of
synthetic files.

cv2's IDCT here is libjpeg-turbo's x86-64 SIMD code; on other hosts the comparisons with cv2 are skipped, and the dump is
compared with the model alone."""
import itertools
import os
import platform
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
cv2 = pytest.importorskip("cv2")
import jpeg_coef_writer as W  # noqa: E402
from test_jpeg_decode_cpu import dump_tool, imdecode, run_dump  # noqa: E402,F401  (dump_tool is a fixture)

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import jpeg_decode_oracle as O  # noqa: E402
from jpeg_oracle import AC_CHROMA, AC_LUMA, DC_CHROMA, DC_LUMA  # noqa: E402

X86 = platform.machine().lower() in ("x86_64", "amd64")
needs_x86 = pytest.mark.skipif(not X86, reason="cv2's IDCT is libjpeg-turbo's x86-64 SIMD code only on x86-64")


def _wrap16(x):
    return ((np.asarray(x, np.int64) + 32768) & 0xFFFF) - 32768


# ---------------------------------------------------------------------------------------------------- the writer
def _check_round_trip(f, blocks, q):
    h, got = O.coefficients(f)
    assert len(got) == len(blocks)
    for c, (g, b) in enumerate(zip(got, blocks)):
        want = np.array(b, np.int64)
        want[..., 0] = _wrap16(want[..., 0])
        assert g.shape == want.shape and np.array_equal(g, want), c
        assert np.array_equal(h["q"][c], q[c]), c


@pytest.mark.parametrize("sampling", list(W.SAMPLING))
def test_writer_round_trip(sampling):
    """The file holds exactly the coefficients and quantisers it was given, for every kind, size and restart interval."""
    for kind in W.KINDS:
        for (h, w), r in [((16, 32), 0), ((37, 53), 3), ((8, 8), 1), ((41, 17), 2)]:
            f, blocks, q = W.synthetic(kind, h, w, sampling, r, seed=1)
            _check_round_trip(f, blocks, q)
            assert (f[2:].find(b"\xff\xc1") >= 0) == (kind in ("wide", "wild"))      # 16-bit DQT under SOF1


def test_writer_custom_tables_and_extremes():
    """Swapped Annex K tables (luma codes chroma and back); AC categories 1, 2, 9 and 10 at both signs, restarts every MCU."""
    swapped = {(0, 0): DC_CHROMA, (1, 0): AC_CHROMA, (0, 1): DC_LUMA, (1, 1): AC_LUMA}
    vals = [0] + [s * v for v in (1, 2, 3, 511, 512, 1023) for s in (1, -1)]
    rng = np.random.default_rng(3)
    blocks = []
    for r, c in W.grid(16, 64, "420"):
        blocks.append(rng.choice(vals, (r, c, 64)))      # DC differences up to +-2046, category 11
    q = [np.full(64, 255), np.arange(1, 65), np.full(64, 1)]
    for tables in (None, swapped):
        f = W.write(blocks, q, 16, 64, "420", restart=1, tables=tables)
        _check_round_trip(f, blocks, q)
        if X86:
            assert np.array_equal(O.decode(f), imdecode(f))


def _one_block(**at):
    b = np.zeros((1, 1, 64), np.int64)
    for k, v in at.items():
        b[0, 0, int(k[1:])] = v
    return [b]


def test_writer_refusals():
    q = [np.ones(64, np.int64)]
    W.write(_one_block(k0=2047, k1=1023, k63=-1023), q, 8, 8, "gray")
    for blocks, qq, why in [
        (_one_block(k0=2048), q, "category 11"),
        (_one_block(k0=-2048), q, "category 11"),
        (_one_block(k1=1024), q, "category 10"),
        (_one_block(k8=-1024), q, "category 10"),
        (_one_block(), [np.zeros(64, np.int64)], "quantiser"),
        (_one_block(), [np.full(64, 65536)], "quantiser"),
        ([np.zeros((2, 1, 64), np.int64)], q, "grids"),
    ]:
        with pytest.raises(ValueError, match=why):
            W.write(blocks, qq, 8, 8, "gray")
    # the coded DC is the difference: 2047 then -1 is a difference of -2048
    two = np.zeros((1, 2, 64), np.int64)
    two[0, :, 0] = [2047, -1]
    with pytest.raises(ValueError, match="category 11"):
        W.write([two], q, 8, 16, "gray")
    with pytest.raises(ValueError, match="not in the Huffman table"):
        W.write(_one_block(k0=5), q, 8, 8, "gray", tables={(0, 0): ([0, 1] + [0] * 14, [0])})


# ---------------------------------------------------------------------------------------------------- probes
PROBE_D = [8191, 8192, 8193, 16383, 16384, 16385, 24576, 32767, 32768, 40000, 49151, 57344]   # q with a coefficient of +-1
PROBE_COLS = 64


def _probe_blocks():
    """Each of the 64 positions alone at +-1, then each of the 2016 pairs at (+1, +1), (+1, -1) and (-1, -1)."""
    out = []
    for i in range(64):
        for s in (1, -1):
            b = np.zeros(64, np.int64)
            b[i] = s
            out.append(b)
    for i, j in itertools.combinations(range(64), 2):
        for s, t in ((1, 1), (1, -1), (-1, -1)):
            b = np.zeros(64, np.int64)
            b[i], b[j] = s, t
            out.append(b)
    return np.array(out)


def _gray_file(blocks, q):
    n = len(blocks)
    rows = -(-n // PROBE_COLS)
    b = np.zeros((rows * PROBE_COLS, 64), np.int64)
    b[:n] = blocks
    return W.write([b.reshape(rows, PROBE_COLS, 64)], [q], rows * 8, PROBE_COLS * 8, "gray")


def _blocks_of(img, n):
    rows = img.shape[0] // 8
    return img.reshape(rows, 8, PROBE_COLS, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)[:n]


@pytest.fixture(scope="module")
def probes():
    """[(name, blocks, q, cv2 samples)]: the sweeps at every dequantised value D (q = D, coefficients +-1, so products
    D and -D modulo 2^16), plus blocks whose DC-only state differs between the coefficients and their products."""
    cases = [("sweep D=%d" % d, _probe_blocks(), np.full(64, d)) for d in PROBE_D]
    # AC coefficients whose product with q = 128 is 0 modulo 2^16, under DC values whose << 2 leaves int16
    b = np.zeros((12, 64), np.int64)
    b[:, 0] = [100, -100, 50, -50, 64, -64, 65, 1, 0, 127, -128, 90]
    b[:6, 8], b[6:9, 15], b[9:, 63] = 512, -512, 512
    cases.append(("zero products", b, np.full(64, 128)))
    # DC-only blocks over the whole DC range at several quantisers
    dc = np.zeros((2 * 1024, 64), np.int64)
    dc[:, 0] = np.arange(-1024, 1024)
    cases += [("DC only q=%d" % q, dc, np.full(64, q)) for q in (8, 16, 33, 64, 255)]
    out = []
    for name, blocks, q in cases:
        f = _gray_file(blocks, q)
        ref = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_GRAYSCALE)
        out.append((name, blocks, q, _blocks_of(ref, len(blocks))))
    return out


def _differing(probes, **steps):
    return {name: int((O.idct_islow(blocks, q, **steps) != ref).any(axis=(1, 2)).sum()) for name, blocks, q, ref in probes}


@needs_x86
def test_probes_model_equals_cv2(probes):
    assert sum(len(p[1]) for p in probes) > 70000
    assert _differing(probes) == {p[0]: 0 for p in probes}


# Each alternative replaces one step of the model; cv2 must differ from it on some probe, so the step is observed.
ALTERNATIVES = {
    "dequant exact": dict(dequant="exact"),
    "no DC-only shortcut": dict(shortcut=None),
    "shortcut decided on products": dict(shortcut="product"),
    "pass 1 even sums exact": dict(pass1_sums=("odd",)),
    "pass 1 odd sums exact": dict(pass1_sums=("even",)),
    "pass 2 even sums exact": dict(pass2_sums=("odd",)),
    "pass 2 odd sums exact": dict(pass2_sums=("even",)),
    "pass 1 rotation sums wrapped": dict(pass1_sums=("even", "odd", "rotation")),
    "pass 2 rotation sums wrapped": dict(pass2_sums=("even", "odd", "rotation")),
    "no saturation between passes": dict(between=None),
    "wrap between passes": dict(between="wrap"),
    "final wrap": dict(final="wrap"),
}


@needs_x86
@pytest.mark.parametrize("alternative", list(ALTERNATIVES))
def test_probes_reject_alternative(probes, alternative):
    d = _differing(probes, **ALTERNATIVES[alternative])
    assert sum(d.values()) > 0, d


def test_model_is_the_c_idct_in_range():
    """Where nothing wraps or saturates, the model is jidctint.c's exact integer IDCT: on coefficients of an encoder's range
    every alternative agrees with it but the final wrap (the C code clamps there too, through its range-limit table)."""
    rng = np.random.default_rng(4)
    blocks = rng.integers(-16, 17, (4000, 64)) * (rng.random((4000, 64)) < 0.3)
    blocks[:, 0] = rng.integers(-128, 128, 4000)
    q = rng.integers(1, 32, 64)
    ref = O.idct_islow(blocks, q)
    for name, steps in ALTERNATIVES.items():
        if name != "final wrap":
            assert np.array_equal(O.idct_islow(blocks, q, **steps), ref), name


# ---------------------------------------------------------------------------------------------------- DC predictions
def _dc_ramp_file(restart=0):
    """A 4:4:4 file whose DC predictions move by +-2047 per block, up for 100 blocks and then down, within each restart
    interval (or the whole frame): the running sum leaves int16 many times, the stored coefficient is its value modulo 2^16."""
    blocks = []
    n = 4 * 64
    per = restart or n
    for c in range(3):
        k = np.arange(n) % per
        steps = np.where(k % 200 < 100, 2047, -2047) * (1 if c != 1 else -1)
        b = np.zeros((n, 64), np.int64)
        for s in range(0, n, per):
            b[s:s + per, 0] = np.cumsum(steps[s:s + per])
        b[::3, 1] = 7
        blocks.append(b.reshape(4, 64, 64))
    q = [np.ones(64, np.int64)] * 3
    return W.write(blocks, q, 32, 512, "444", restart), blocks, q


def test_dc_predictions_leave_int16(dump_tool, tmp_path):
    files = []
    for restart in (0, 150):
        f, blocks, q = _dc_ramp_file(restart)
        assert max(int(np.abs(b[..., 0]).max()) for b in blocks) > 200000
        _check_round_trip(f, blocks, q)
        files.append(f)
    got = run_dump(dump_tool, tmp_path, files)
    for i, (res, g) in enumerate(zip(got, files)):
        assert res[0] == "ok" and np.array_equal(res[1], O.decode(g)), i
        if X86:
            assert np.array_equal(res[1], imdecode(g)), i


# ---------------------------------------------------------------------------------------------------- synthetic matrix
@needs_x86
@pytest.mark.parametrize("sampling", list(W.SAMPLING))
def test_matrix_model_equals_cv2(sampling):
    for name, f in W.matrix(sizes=((16, 32), (37, 53), (64, 80)), restarts=(0, 1, 3), seed=2):
        if "-%s-" % sampling in name:
            assert np.array_equal(O.decode(f), imdecode(f)), name


@pytest.mark.parametrize("bits", [2048, 32])
def test_matrix_dump_equals_model_and_cv2(dump_tool, tmp_path, bits):
    cases = W.matrix(sizes=((16, 32), (37, 53)), restarts=(0, 3), seed=3)
    got = run_dump(dump_tool, tmp_path, [f for _, f in cases], bits)
    for (name, f), res in zip(cases, got):
        assert res[0] == "ok", (name, res)
        assert np.array_equal(res[1], O.decode(f)), name
        if X86:
            assert np.array_equal(res[1], imdecode(f)), name


def test_probe_dump_equals_model(dump_tool, tmp_path):
    """The sweeps through the kernels' arithmetic: two D values per power of two, in gray files."""
    blocks = _probe_blocks()
    files = [_gray_file(blocks, np.full(64, d)) for d in (8192, 16385, 32767, 32768, 49151)]
    for res, f in zip(run_dump(dump_tool, tmp_path, files), files):
        assert res[0] == "ok"
        assert np.array_equal(res[1][..., 0], O.decode(f)[..., 0])
        if X86:
            assert np.array_equal(res[1], imdecode(f))
