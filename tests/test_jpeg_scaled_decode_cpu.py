"""Reduced and gray JPEG decoding without a GPU (DESIGN.md section 8.13).  The numpy model
(oracle/jpeg_scaled_decode_oracle.py) and tools/jpeg_decode_dump.cu --scale (the kernels' own arithmetic on the CPU, under
AddressSanitizer) equal cv2.imdecode with IMREAD_REDUCED_COLOR_d, IMREAD_GRAYSCALE and IMREAD_REDUCED_GRAYSCALE_d on
encoder files and on coefficient-writer files outside an encoder's range, where probes pin each 16- and 32-bit step of the
reduced IDCTs.  Also the ABI and Python argument checks, without a context."""
import ctypes as C
import os
import platform
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
cv2 = pytest.importorskip("cv2")
import jpeg_coef_writer as CW  # noqa: E402
from test_jpeg_cpu import KINDS, SIZES, frame  # noqa: E402
from test_jpeg_decode_cpu import GOLDEN, SAMPLES, SAMPLINGS, dump_tool, encode, strip_dht, with_exif  # noqa: E402,F401

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import jpeg_scaled_decode_oracle as S  # noqa: E402

X86 = platform.machine().lower() in ("x86_64", "amd64")
MODES = [(d, g) for d in (1, 2, 4, 8) for g in (False, True)]
FLAGS = {(1, False): cv2.IMREAD_COLOR, (2, False): cv2.IMREAD_REDUCED_COLOR_2, (4, False): cv2.IMREAD_REDUCED_COLOR_4,
         (8, False): cv2.IMREAD_REDUCED_COLOR_8, (1, True): cv2.IMREAD_GRAYSCALE, (2, True): cv2.IMREAD_REDUCED_GRAYSCALE_2,
         (4, True): cv2.IMREAD_REDUCED_GRAYSCALE_4, (8, True): cv2.IMREAD_REDUCED_GRAYSCALE_8}


def imdecode(buf, d, gray):
    r = cv2.imdecode(np.frombuffer(buf, np.uint8), FLAGS[(d, gray)])
    return r[:, :, None] if gray else r


def run_dump(exe, tmp_path, files, d, gray, bits=2048):
    """One dump run at 1 / d: per file ("ok", frame) or ("einval" / "status", text)."""
    args = []
    for i, f in enumerate(files):
        p = tmp_path / ("f%d.jpg" % i)
        p.write_bytes(f)
        args += [str(p), str(tmp_path / ("f%d.out" % i))]
    r = subprocess.run([exe, str(bits), "--scale", str(d), "1" if gray else "3"] + args, capture_output=True, text=True,
                       env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stderr[-4000:]
    out = []
    for i, line in enumerate(r.stdout.splitlines()):
        kind, rest = line.split(" ", 1)
        if kind == "ok":
            h, w, _ = (int(v) for v in rest.split())
            out.append(("ok", np.fromfile(str(tmp_path / ("f%d.out" % i)), np.uint8).reshape(h, w, 1 if gray else 3)))
        else:
            out.append((kind, rest))
    assert len(out) == len(files)
    return out


def check_files(exe, tmp_path, files, modes=MODES, bits=2048, oracle=True):
    """The model (if ``oracle``) and the dump equal cv2 on every file in every mode."""
    for d, g in modes:
        res = run_dump(exe, tmp_path, files, d, g, bits)
        for i, f in enumerate(files):
            ref = imdecode(f, d, g)
            assert res[i][0] == "ok", (d, g, i, res[i])
            assert res[i][1].shape == ref.shape and np.array_equal(res[i][1], ref), (d, g, i, ref.shape)
            if oracle:
                got = S.decode(f, d, g)
                assert got.shape == ref.shape and np.array_equal(got, ref), (d, g, i)


# ---------------------------------------------------------------------------------------------------- the model's rules
def test_idct_sizes():
    """jpeg_core_output_dimensions' table: luma 8/d, chroma doubled while both sampling ratios divide."""
    assert [S.idct_sizes(2, 2, 3, d) for d in (1, 2, 4, 8)] == [[8, 8, 8], [4, 8, 8], [2, 4, 4], [1, 2, 2]]
    assert [S.idct_sizes(2, 1, 3, d) for d in (1, 2, 4, 8)] == [[8, 8, 8], [4, 4, 4], [2, 2, 2], [1, 1, 1]]
    assert [S.idct_sizes(1, 1, 3, d) for d in (1, 2, 4, 8)] == [[8, 8, 8], [4, 4, 4], [2, 2, 2], [1, 1, 1]]
    assert [S.idct_sizes(1, 1, 1, d) for d in (1, 2, 4, 8)] == [[8], [4], [2], [1]]


def test_output_sizes():
    """ceil(H / d) x ceil(W / d) in every sampling (37 x 53 -> 19 x 27, 10 x 14, 5 x 7)."""
    for s in SAMPLINGS:
        f = encode(frame("noise", 37, 53), 75, s)
        assert [imdecode(f, d, False).shape[:2] for d in (2, 4, 8)] == [(19, 27), (10, 14), (5, 7)]
        assert [S.decode(f, d).shape[:2] for d in (2, 4, 8)] == [(19, 27), (10, 14), (5, 7)]


def test_gray_is_not_cvtcolor():
    """IMREAD_GRAYSCALE is the luma plane, not cvtColor of the colour decode."""
    f = encode(frame("noise", 37, 53), 95, "420")
    luma = imdecode(f, 1, True)[:, :, 0]
    assert np.array_equal(S.decode(f, 1, True)[:, :, 0], luma)
    assert not np.array_equal(cv2.cvtColor(imdecode(f, 1, False), cv2.COLOR_BGR2GRAY), luma)


def test_reduced_8_is_dc():
    """IMREAD_REDUCED_GRAYSCALE_8: clamp(((DC q + 4) >> 3) + 128) per luma block."""
    import jpeg_decode_oracle as D
    for kind in ("noise", "gradient"):
        for q in (50, 95):
            f = encode(frame(kind, 64, 80), q, "420")
            h, blocks = D.coefficients(f)
            dc = blocks[0][..., 0] * h["q"][0][0]
            assert np.array_equal(imdecode(f, 8, True)[:, :, 0], np.clip(((dc + 4) >> 3) + 128, 0, 255))


def test_range_limit_1x1():
    """jpeg_idct_1x1 looks the DC up in the 1024-entry range-limit table through RANGE_MASK: it wraps where a clamp would
    saturate.  Pinned by DC-only blocks at 8 and 16-bit quantisers."""
    if not X86:
        pytest.skip("cv2's reduced IDCTs are libjpeg-turbo's x86-64 code only on x86-64")
    hits = 0
    for dc in (-2047, -1500, -600, -100, 100, 600, 1500, 2047):
        for q in (1, 8, 16, 32, 255, 40000):
            b = np.zeros((1, 1, 64), np.int64)
            b[0, 0, 0] = dc
            f = CW.write([b], [np.full(64, q)], 8, 8, "gray")
            ref = int(imdecode(f, 8, True)[0, 0, 0])
            assert int(S.decode(f, 8, True)[0, 0, 0]) == ref, (dc, q)
            qs = ((q + 32768) & 0xFFFF) - 32768
            clamped = min(255, max(0, ((dc * qs + 4) >> 3) + 128))
            hits += clamped != ref
    assert hits > 0      # a clamp instead of the range-limit table differs from cv2


# ---------------------------------------------------------------------------------------------------- encoder files
@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_matrix_equals_cv2(dump_tool, tmp_path, sampling):
    """Section 8.10's SIZES x qualities 1, 50, 95, 100 x four kinds of content, at every d in colour and gray."""
    files = [encode(frame(KINDS[(i + q) % len(KINDS)], h, w, seed=q), q, sampling)
             for i, (h, w) in enumerate(SIZES) for q in (1, 50, 95, 100)]
    files += [encode(frame(k, 37, 53, seed=7), 75, sampling) for k in KINDS]
    check_files(dump_tool, tmp_path, files)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
def test_odd_sizes_equal_cv2(dump_tool, tmp_path, sampling):
    """1x1, 1x17, 17x1, 7x15 (chroma planes 1-4 samples wide) and 1081x1921."""
    files = [encode(frame("noise", h, w, seed=1), 90, sampling) for h, w in [(1, 1), (1, 17), (17, 1), (7, 15), (9, 33), (33, 17)]]
    check_files(dump_tool, tmp_path, files)
    check_files(dump_tool, tmp_path, [encode(frame("noise", 1081, 1921, seed=3), 95, sampling)], oracle=False)


def test_restarts_dht_exif_samples(dump_tool, tmp_path):
    """Restart intervals 1, 4, 7; files without DHT; EXIF orientations 1-8 in both byte orders; the golden samples."""
    files = [encode(frame("noise", 37, 53, seed=r), 75, s, rst=r) for r in (1, 4, 7) for s in SAMPLINGS]
    files += [strip_dht(encode(frame("noise", 37, 53), 75, s)) for s in SAMPLINGS]
    base = encode(frame("gradient", 40, 66), 90, "422")
    files += [with_exif(base, o, be) for o in range(1, 9) for be in (False, True)]
    files += [open(os.path.join(GOLDEN, s), "rb").read() for s in SAMPLES]
    check_files(dump_tool, tmp_path, files)


def test_short_subsequences(dump_tool, tmp_path):
    files = [encode(frame("noise", 37, 53, seed=2), 95, s, rst=r) for s in SAMPLINGS for r in (0, 3)]
    check_files(dump_tool, tmp_path, files, modes=[(2, False), (8, False), (4, True)], bits=32, oracle=False)


# ---------------------------------------------------------------------------------------------------- coefficient files
def _probe_files():
    """Gray files of probe blocks: DC 0 or +-1023 with one more coefficient at each of the 64 positions at +-255, +-512 and
    +-1023, and blocks of +-1023 signed to drive one column-pass output past 2^31; under flat quantisers 32 (dequantised
    values up to +-32736) and 40000 (products that wrap 16 bits)."""
    blocks = [np.zeros(64, np.int64)]
    for dc in (0, 1023, -1023):
        for k in range(64):
            for v in (255, -255, 512, -512, 1023, -1023):
                b = np.zeros(64, np.int64)
                b[0] = dc
                b[k] = v if k else dc + v // 2
                blocks.append(b)
    # every coefficient at +-1023 with the signs of one output's weights in the column pass, so that the 32-bit sums wrap
    eye = np.eye(8, dtype=np.int64)[None]
    t10, odd = eye[:, 0] * (1 << 15), S._odd_2(eye)
    weights = list(np.sign(S._pass_4(eye)[0])) + list(np.sign(np.stack([t10 + odd, t10 - odd], 1)[0]))
    for w in weights:
        for sign in (1, -1):
            blocks.append((np.repeat(sign * w[:, None], 8, 1) * 1023).reshape(64))
    blocks = np.array(blocks)
    out = []
    for q in (32, 40000):
        for lo in range(0, len(blocks), 256):
            part = blocks[lo:lo + 256]
            out.append(CW.write([part.reshape(1, -1, 64)], [np.full(64, q)], 8, 8 * len(part), "gray"))
    return out


@pytest.mark.skipif(not X86, reason="cv2's reduced IDCTs are libjpeg-turbo's SSE2 code only on x86-64")
def test_reduced_idct_probes():
    """The model of cv2's 4x4 and 2x2 IDCTs equals cv2 on every probe block, and each of its steps is needed: the model with
    that step replaced differs from cv2 on some probe."""
    files = _probe_files()
    ref = {d: [imdecode(f, d, True) for f in files] for d in (2, 4)}

    def differs(d, **steps):
        return sum(not np.array_equal(S.decode(f, d, True, **steps), r) for f, r in zip(files, ref[d]))
    assert differs(2) == 0 and differs(4) == 0
    for steps in (dict(sums="exact"), dict(shortcut=None), dict(shortcut="rows1to7")):
        assert differs(2, **steps) > 0, steps
    for steps in (dict(sums="exact"), dict(col0="int16")):
        assert differs(4, **steps) > 0, steps


def test_coefficient_files(dump_tool, tmp_path):
    """Every kind of coefficient-writer file (dense, sparse, DC-only, row-0-only, 16-bit DQT, ...) in every sampling: the
    dump equals the model at every d in colour and gray, and both equal cv2 (on x86-64, where cv2's IDCTs are
    libjpeg-turbo's SSE2 code).  The probe blocks too, through the dump."""
    files = [CW.synthetic(k, h, w, s, r, seed=5)[0] for k in CW.KINDS for s in CW.SAMPLING
             for (h, w), r in [((16, 32), 0), ((37, 53), 3)]]
    for d, g in MODES:
        res = run_dump(dump_tool, tmp_path, files, d, g)
        for i, f in enumerate(files):
            assert res[i][0] == "ok", (d, g, i, res[i])
            model = S.decode(f, d, g)
            assert np.array_equal(res[i][1], model), (d, g, i)
            if X86:
                assert np.array_equal(model, imdecode(f, d, g)), (d, g, i)
    probes = _probe_files()
    for d in (2, 4, 8):
        for r, f in zip(run_dump(dump_tool, tmp_path, probes, d, True), probes):
            assert r[0] == "ok" and np.array_equal(r[1], S.decode(f, d, True)), d


def test_corrupt_files(dump_tool, tmp_path):
    """Seeded byte flips: each file ends in a frame, a status or a refused header, never a sanitizer report; every frame
    equals cv2's at every d (on x86-64), and the model's wherever the model (whose block-count check is stricter) decodes
    it."""
    rng = np.random.default_rng(91)
    base = [encode(frame("noise", 48, 64, seed=s), 75, s_, rst=2) for s, s_ in enumerate(SAMPLINGS)]
    files = []
    for i in range(60):
        f = bytearray(base[i % len(base)])
        p = int(rng.integers(len(f) // 3, len(f) - 2))
        f[p] ^= int(rng.integers(1, 256))
        files.append(bytes(f))
    decoded = 0
    for d, g in MODES:
        for i, r in enumerate(run_dump(dump_tool, tmp_path, files, d, g)):
            if r[0] == "ok":
                decoded += 1
                try:
                    model = S.decode(files[i], d, g)
                except ValueError:
                    model = None
                assert model is None or np.array_equal(r[1], model), (d, g, i)
                if X86 or d == 1:
                    assert np.array_equal(r[1], imdecode(files[i], d, g)), (d, g, i)
    assert decoded > 0


# ---------------------------------------------------------------------------------------------------- argument checks
def test_abi_argument_checks():
    from whenet_b200 import _lib
    L = _lib.load()
    f = encode(frame("noise", 37, 53), 75, "420")
    hw = (C.c_int32 * 2)()
    msg = C.create_string_buffer(128)
    for d in (1, 2, 4, 8):
        for ch in (1, 3):
            assert L.whenet_jpeg_info_ex(f, len(f), d, ch, hw, msg, len(msg)) == 0
            assert (hw[0], hw[1]) == (-(-37 // d), -(-53 // d))
    for d, ch in [(0, 3), (3, 3), (16, 3), (-2, 3), (2, 2), (2, 0), (1, 4)]:
        assert L.whenet_jpeg_info_ex(f, len(f), d, ch, hw, msg, len(msg)) != 0
        assert msg.value
    buf = C.create_string_buffer(f, len(f))
    ptrs = (C.c_void_p * 1)(C.addressof(buf))
    sizes = (C.c_int64 * 1)(len(f))
    out = (C.c_void_p * 1)(1)
    for d, ch in [(3, 3), (2, 2)]:
        assert L.whenet_decode_jpeg_ex_u8(None, ptrs, sizes, 1, d, ch, out, None) != 0
        assert b"scale_denom" in L.whenet_last_error() or b"channels" in L.whenet_last_error()
    assert L.whenet_decode_jpeg_ex_u8(None, ptrs, sizes, 1, 2, 1, out, None) != 0
    assert b"context" in L.whenet_last_error()


def test_python_argument_checks():
    from whenet_b200 import video
    f = encode(frame("noise", 37, 53), 75, "420")
    assert video.jpeg_info(f) == (37, 53)
    assert [video.jpeg_info(f, reduce=d) for d in (2, 4, 8)] == [(19, 27), (10, 14), (5, 7)]
    for bad in (0, 3, 16, 2.0, "2", True, None):
        with pytest.raises(ValueError, match="reduce"):
            video.jpeg_info(f, reduce=bad)
        with pytest.raises(ValueError, match="reduce"):
            video.decode_jpeg(None, [f], reduce=bad)
    for bad in (1, 0, "yes", None):
        with pytest.raises(ValueError, match="gray"):
            video.decode_jpeg(None, [f], gray=bad)
    with pytest.raises(ValueError, match="not 1 or 3 components|progressive"):
        video.jpeg_info(cv2.imencode(".jpg", frame("noise", 16, 16), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), reduce=2)
