"""Numpy restatement of the GPU JPEG decoder's reduced and gray modes (DESIGN.md section 8.13), written from ITU-T T.81 and
libjpeg's documented behaviour and checked against cv2.imdecode with IMREAD_REDUCED_COLOR_d, IMREAD_GRAYSCALE and
IMREAD_REDUCED_GRAYSCALE_d (OpenCV 4.13, libjpeg-turbo 3.1.2).  It reuses jpeg_decode_oracle's entropy stage and 8x8 IDCT
model and shares no code with csrc/kernels_jpeg_dec.cuh.

    decode(data, reduce=1, gray=False) -> (ceil(H/d), ceil(W/d), 3 or 1) uint8, or ValueError naming the reason

The steps that differ from the full-size colour decode:

  IDCT sizes     libjpeg's jpeg_core_output_dimensions (jdmaster.c): the luma IDCT is m = 8/d samples square; a chroma
                 component's size doubles from m while it stays <= 8 and both its sampling ratios to the luma's divide
                 (4:2:0 at d = 2: chroma 8x8; 4:2:2: chroma as luma; 4:4:4: every component m)
  reduced IDCT   jidctred.c's jpeg_idct_4x4 / jpeg_idct_2x2 (CONST_BITS 13, PASS1_BITS 2, columns first) with the 16- and
                 32-bit steps of libjpeg-turbo's SSE2 versions, which cv2 runs on x86-64 (REDUCED_MODEL; each step is a
                 keyword of idct_4x4 / idct_2x2 so that a test can show cv2 rejects the alternative):
                   - the coefficient x quantiser product modulo 2^16;
                   - multiply-add sums and descales modulo 2^32 (pmaddwd / paddd lanes);
                   - 4x4: a block whose coefficient rows 1, 2, 3, 5, 6, 7 are all zero skips the column pass, and each
                     workspace column is its row-0 value shifted left by PASS1_BITS modulo 2^16; otherwise the column
                     pass saturates to int16;
                   - 2x2: no shortcut; columns 1, 3, 5, 7 of the column pass saturate to int16, but column 0 stays a
                     32-bit value whose row-pass even term (<< 15) is taken modulo 2^32;
                   - the row pass saturates to int16, then clamps to [-128, 127] and adds 128.
                 4x4 ignores coefficient row and column 4, 2x2 reads only indices 0, 1, 3, 5 and 7.
                 jpeg_idct_1x1 (plain C): (DC x q + 4) >> 3 looked up in libjpeg's 1024-entry range-limit table through
                 RANGE_MASK, with the quantiser read as a signed 16-bit multiplier
  upsampling     none where a chroma plane is already at the output size; h2v1 or h2v2 where it is half: fancy
                 (jdsample.c) when m > 1 and the chroma plane is more than 2 samples wide, plain replication otherwise
  gray           IMREAD_GRAYSCALE: the luma plane alone, cropped; the chroma is never decoded to samples
"""
from __future__ import annotations

import numpy as np

import jpeg_decode_oracle as D

SCALES = (1, 2, 4, 8)

# jidctred.c's constants (CONST_BITS 13)
_F = dict(F0211=1730, F0509=4176, F0601=4926, F0720=5906, F0765=6270, F0850=6967, F0899=7373, F1061=8697, F1272=10426,
          F1451=11893, F1847=15137, F2172=17799, F2562=20995, F3624=29692)


def idct_sizes(hs: int, vs: int, ncomp: int, reduce: int) -> list:
    """The IDCT size of each component (jpeg_core_output_dimensions); luma sampling hs x vs, chroma 1 x 1."""
    m = 8 // reduce
    sizes = [m]
    for _ in range(1, ncomp):
        s = m
        while s < 8 and (hs * m) % (2 * s) == 0 and (vs * m) % (2 * s) == 0:
            s *= 2
        sizes.append(s)
    return sizes


def _sat16(x):
    return np.clip(x, -32768, 32767)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _final(x):
    return np.clip(x, -128, 127) + 128


def _deq(coef, q):
    return D._s16(np.asarray(coef, np.int64).reshape(-1, 64) * np.asarray(q, np.int64).reshape(64)).reshape(-1, 8, 8)


def _s32(x):
    return ((x + 2**31) & 0xFFFFFFFF) - 2**31


def _pass_4(d):
    """jpeg_idct_4x4's 1-D transform along axis 1 of d (n, 8, ...): 4 outputs (unscaled, CONST_BITS + 1 fraction bits)."""
    t0 = d[:, 0] * (1 << 14)
    t2 = d[:, 2] * _F["F1847"] - d[:, 6] * _F["F0765"]
    t10, t12 = t0 + t2, t0 - t2
    z1, z2, z3, z4 = d[:, 7], d[:, 5], d[:, 3], d[:, 1]
    o0 = -z1 * _F["F0211"] + z2 * _F["F1451"] - z3 * _F["F2172"] + z4 * _F["F1061"]
    o2 = -z1 * _F["F0509"] - z2 * _F["F0601"] + z3 * _F["F0899"] + z4 * _F["F2562"]
    return np.stack([t10 + o2, t12 + o0, t12 - o0, t10 - o2], 1)


def _odd_2(d):
    return -d[:, 7] * _F["F0720"] + d[:, 5] * _F["F0850"] - d[:, 3] * _F["F1272"] + d[:, 1] * _F["F3624"]


# The model of cv2's reduced IDCTs; tests/test_jpeg_scaled_decode_cpu.py shows cv2 takes none of the alternatives.
REDUCED_MODEL = dict(sums="wrap32", shortcut="rows12356", col0="int32")


def _descale_s(x, n, sums):
    """(x + 2^(n-1)) >> n, the sum taken modulo 2^32 for sums="wrap32" (exact for "exact")."""
    x = x + (1 << (n - 1))
    return (_s32(x) if sums == "wrap32" else x) >> n


def idct_4x4(coef, q, **steps) -> np.ndarray:
    """(n, 64) natural-order coefficients -> (n, 4, 4) samples.  sums: "wrap32" | "exact"; shortcut: "rows12356" (the
    DC-only column shortcut, decided on coefficient rows 1, 2, 3, 5, 6, 7), "rows1to7" or None."""
    st = dict(REDUCED_MODEL, **steps)
    c = np.asarray(coef, np.int64).reshape(-1, 8, 8)
    d = _deq(coef, q)
    ws = _sat16(_descale_s(_pass_4(d), 13 - 2 + 1, st["sums"]))                # (n, 4, 8): columns first
    if st["shortcut"]:
        rows = [1, 2, 3, 5, 6, 7] if st["shortcut"] == "rows12356" else [1, 2, 3, 4, 5, 6, 7]
        z = ~c[:, rows].any(axis=(1, 2))
        ws[z] = np.repeat(D._s16(d[z, :1] * 4), 4, axis=1)
    rows = _sat16(_descale_s(_pass_4(ws.transpose(0, 2, 1)), 13 + 2 + 3 + 1, st["sums"]))   # (n, 4 cols, 4 rows)
    return _final(rows.transpose(0, 2, 1))


def idct_2x2(coef, q, **steps) -> np.ndarray:
    """(n, 64) -> (n, 2, 2).  sums: "wrap32" | "exact"; col0: "int32" (column 0 of the column pass kept in 32 bits, its
    row-pass even term << 15 taken modulo 2^32) or "int16" (saturated like the other columns)."""
    st = dict(REDUCED_MODEL, **steps)
    d = _deq(coef, q)
    t10, o = d[:, 0] * (1 << 15), _odd_2(d)
    ws = _descale_s(np.stack([t10 + o, t10 - o], 1), 13 - 2 + 2, st["sums"])   # (n, 2, 8), 32-bit
    ws16 = _sat16(ws)
    col0 = ws[:, :, 0] if st["col0"] == "int32" else ws16[:, :, 0]
    e = col0 * (1 << 15)
    if st["sums"] == "wrap32":
        e = _s32(e)
    o = _odd_2(ws16.transpose(0, 2, 1))                                         # (n, 2 rows)
    rows = _sat16(_descale_s(np.stack([e + o, e - o], 2), 13 + 2 + 3 + 2, st["sums"]))    # (n, 2 rows, 2 cols)
    return _final(rows)


def range_limit(x):
    """libjpeg's post-IDCT range-limit table (jdmaster.c prepare_range_limit_table) indexed by x & RANGE_MASK (1023)."""
    v = np.asarray(x, np.int64) & 1023
    return np.where(v < 128, v + 128, np.where(v < 512, 255, np.where(v < 896, 0, v - 896)))


def idct_1x1(coef, q) -> np.ndarray:
    """(n, 64) -> (n, 1, 1): jpeg_idct_1x1, DC only."""
    qs = D._s16(int(np.asarray(q).reshape(64)[0]))            # ISLOW_MULT_TYPE is a short
    dc = np.asarray(coef, np.int64).reshape(-1, 64)[:, 0] * qs
    return range_limit(_descale(dc, 3)).reshape(-1, 1, 1)


def idct(coef, q, size: int, **steps) -> np.ndarray:
    if size == 8:
        return D.idct_islow(coef, q)
    if size == 1:
        return idct_1x1(coef, q)
    return {4: idct_4x4, 2: idct_2x2}[size](coef, q, **steps)


def _replicate(p, uh, uv, H, W):
    return np.repeat(np.repeat(p, uv, 0), uh, 1)[:H, :W]


def decode(data: bytes, reduce: int = 1, gray: bool = False, **steps) -> np.ndarray:
    """cv2.imdecode(data, flag) for IMREAD_COLOR / IMREAD_REDUCED_COLOR_d (gray False) or IMREAD_GRAYSCALE /
    IMREAD_REDUCED_GRAYSCALE_d (gray True), d = ``reduce``; ``steps`` replace steps of REDUCED_MODEL."""
    if reduce not in SCALES:
        raise ValueError("reduce must be 1, 2, 4 or 8")
    h, blocks = D.coefficients(data)
    H, W, hs, vs = h["H"], h["W"], h["hs"], h["vs"]
    m = 8 // reduce
    Ho, Wo = -(-H // reduce), -(-W // reduce)
    sizes = idct_sizes(hs, vs, len(blocks), reduce)
    planes = []
    for c, b in enumerate(blocks[:1] if gray else blocks):
        rows, cols = b.shape[:2]
        s = sizes[c]
        px = idct(b.reshape(-1, 64), h["q"][c], s, **steps)
        planes.append(px.reshape(rows, cols, s, s).transpose(0, 2, 1, 3).reshape(rows * s, cols * s))
    Y = planes[0][:Ho, :Wo]
    if gray:
        out = Y[:, :, None]
    elif len(planes) == 1:
        out = np.stack([Y, Y, Y], -1)
    else:
        chroma = []
        for c in (1, 2):
            uh, uv = hs * m // sizes[c], vs * m // sizes[c]
            cw, ch = -(-Wo // uh), -(-Ho // uv)
            p = planes[c][:ch, :cw]
            if uh == uv == 1:
                chroma.append(p)
            elif m > 1:
                chroma.append(D._upsample(p, uh, uv, Ho, Wo))             # replicates a plane at most 2 samples wide
            else:
                chroma.append(_replicate(p, uh, uv, Ho, Wo))
        cb, cr = (p - 128 for p in chroma)
        fix = lambda x: int(x * 65536 + 0.5)        # noqa: E731
        r = Y + ((fix(1.40200) * cr + 32768) >> 16)
        g = Y + ((-fix(0.34414) * cb - fix(0.71414) * cr + 32768) >> 16)
        b = Y + ((fix(1.77200) * cb + 32768) >> 16)
        out = np.stack([b, g, r], -1)
    return np.ascontiguousarray(D._orient(np.clip(out, 0, 255).astype(np.uint8), h["orient"]))
