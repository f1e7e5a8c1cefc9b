"""Numpy restatement of the GPU JPEG decoder (DESIGN.md section 8.10), written from ITU-T T.81 and libjpeg's documented
behaviour and checked against cv2.imdecode(buf, cv2.IMREAD_COLOR) (OpenCV 4.13, libjpeg-turbo 3.1.2).  It shares no code with
csrc/kernels_jpeg_dec.cuh.

    decode(data) -> (H, W, 3) uint8 BGR, or ValueError naming the reason

Subset: SOF0 / SOF1 8-bit Huffman, one interleaved scan, 1 component or 3 (YCbCr) at 4:4:4, 4:2:2 or 4:2:0, DRI / RSTn,
Annex K tables for slots 0 / 1 without DHT, EXIF orientation.  The steps:

  entropy data   T.81 F.2.2: 0xFF 0x00 is a data 0xFF, a run of 0xFF fill bytes before a marker is dropped, RSTn ends a
                 restart interval (DC predictions reset, the next interval starts byte-aligned)
  dequantise     the coefficient x quantiser product taken modulo 2^16 (libjpeg-turbo's SIMD IDCT multiplies in 16-bit lanes)
  IDCT           libjpeg's islow (jidctint.c): CONST_BITS 13, PASS1_BITS 2, columns first, with the 16-bit steps of
                 libjpeg-turbo's SIMD code (idct_islow): the DC-only column shortcut, pairwise sums modulo 2^16, an int16
                 saturation between the passes, then clamped to [-128, 127] and + 128
  upsampling     libjpeg's fancy upsampling (jdsample.c) with the real downsampled width and height replicated at the edges;
                 a chroma plane at most 2 samples wide is replicated instead (jdsample.c uses the fancy path above that)
  colour         jdcolor.c's YCbCr -> RGB tables with 16 fraction bits, written as BGR; 1 component is replicated to B = G = R
  orientation    OpenCV's ExifReader on the first APP1, then cv2's flip / transpose sequence
"""
from __future__ import annotations

import numpy as np

from jpeg_oracle import AC_CHROMA, AC_LUMA, DC_CHROMA, DC_LUMA, ZIGZAG

STD_TABLES = {(0, 0): DC_LUMA, (0, 1): DC_CHROMA, (1, 0): AC_LUMA, (1, 1): AC_CHROMA}     # (class, slot) -> (counts, symbols)


# ---------------------------------------------------------------------------------------------------- headers
def _exif_orientation(d: bytes) -> int:
    """OpenCV's ExifReader: TIFF block, IFD0 entries read until one passes the end; the first orientation tag counts."""
    n = len(d)
    if n < 1:
        return 1
    intel = d[0] == ord("I") and (n < 2 or d[1] == ord("I"))

    def u(off, size):
        if off + size - 1 >= n:
            raise IndexError
        return int.from_bytes(d[off:off + size], "little" if intel else "big")
    try:
        if u(2, 2) != 0x2A:
            return 1
        off = u(4, 4)
        for e in range(u(off, 2)):
            p = off + 2 + 12 * e
            if u(p, 2) == 0x0112:
                v = u(p + 8, 2)
                return v if 1 <= v <= 8 else 1
    except IndexError:
        pass
    return 1


def _huff(counts, symbols):
    """{(length, code): symbol} of a canonical table (T.81 Annex C)."""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            table[(length, code)] = symbols[k]
            code += 1
            k += 1
        code <<= 1
    return table


def parse(data: bytes) -> dict:
    """Header fields of a supported file, or ValueError with the reason."""
    if len(data) < 4 or data[:2] != b"\xff\xd8":
        raise ValueError("not a JPEG file (no SOI)")
    qt, ht, pos, h = {}, {}, 2, {"ri": 0, "orient": 1}
    jfif = adobe = app1 = False
    adobe_transform = 0
    while True:
        if pos >= len(data) or data[pos] != 0xFF:
            raise ValueError("truncated or malformed marker segment")
        while pos < len(data) and data[pos] == 0xFF:
            pos += 1
        if pos >= len(data):
            raise ValueError("truncated marker segment")
        m = data[pos]
        pos += 1
        if m == 0x01 or 0xD0 <= m <= 0xD7:
            continue
        if m in (0xD8, 0xD9):
            raise ValueError("SOI or EOI before any scan")
        length = int.from_bytes(data[pos:pos + 2], "big")
        if length < 2 or pos + length > len(data):
            raise ValueError("truncated marker segment")
        s = data[pos + 2:pos + length]
        pos += length
        if m in (0xC0, 0xC1):
            if s[0] != 8:
                raise ValueError("not 8-bit (12-bit or other sample precision)")
            h["H"], h["W"], nc = int.from_bytes(s[1:3], "big"), int.from_bytes(s[3:5], "big"), s[5]
            if h["H"] == 0:
                raise ValueError("height defined by DNL")
            if nc not in (1, 3):
                raise ValueError("not 1 or 3 components")
            h["comps"] = [(s[6 + 3 * c], s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]) for c in range(nc)]
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise ValueError("progressive JPEG")
        elif m in (0xC3, 0xC7, 0xCB, 0xCF):
            raise ValueError("lossless JPEG")
        elif m in (0xC5, 0xC9, 0xCC, 0xCD):
            raise ValueError("hierarchical or arithmetic-coded JPEG")
        elif m == 0xDB:
            o = 0
            while o < len(s):
                pq, tq = s[o] >> 4, s[o] & 15
                n = 64 * (pq + 1)
                vals = np.frombuffer(s[o + 1:o + 1 + n], ">u2" if pq else "u1").astype(np.int64)
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = vals
                qt[tq] = nat
                o += 1 + n
        elif m == 0xC4:
            o = 0
            while o < len(s):
                tc, th = s[o] >> 4, s[o] & 15
                counts = list(s[o + 1:o + 17])
                ht[(tc, th)] = (counts, list(s[o + 17:o + 17 + sum(counts)]))
                o += 17 + sum(counts)
        elif m == 0xDD:
            h["ri"] = int.from_bytes(s[:2], "big")
        elif m == 0xE0:
            jfif = jfif or s[:5] == b"JFIF\0"
        elif m == 0xE1:
            if not app1 and len(s) > 6:
                h["orient"] = _exif_orientation(s[6:])
            app1 = True
        elif m == 0xEE:
            if len(s) >= 12 and s[:5] == b"Adobe":
                adobe, adobe_transform = True, s[11]
        elif m == 0xDA:
            comps = h["comps"]
            if s[0] != len(comps):
                raise ValueError("non-interleaved scan (a scan without every component)")
            sel = [(s[2 + 2 * i] >> 4, s[2 + 2 * i] & 15) for i in range(s[0])]
            if tuple(s[1 + 2 * s[0]:4 + 2 * s[0]]) != (0, 63, 0):
                raise ValueError("spectral selection or successive approximation in a sequential scan")
            if len(comps) == 3:
                ids = [c[0] for c in comps]
                if not jfif and (adobe_transform == 0 if adobe else ids == [82, 71, 66]):
                    raise ValueError("RGB colour transform")
                if any((c[1], c[2]) != (1, 1) for c in comps[1:]) or (comps[0][1], comps[0][2]) not in ((1, 1), (2, 1), (2, 2)):
                    raise ValueError("unsupported sampling")
                h["hs"], h["vs"] = comps[0][1], comps[0][2]
            else:
                h["hs"] = h["vs"] = 1
            h["q"] = [qt[c[3]] for c in comps]
            h["dc"] = [_huff(*ht.get((0, t[0]), STD_TABLES.get((0, t[0])))) for t in sel]
            h["ac"] = [_huff(*ht.get((1, t[1]), STD_TABLES.get((1, t[1])))) for t in sel]
            h["ecs"] = pos
            return h
        elif not (0xE0 <= m <= 0xEF or m == 0xFE):
            raise ValueError("unknown marker")


# ---------------------------------------------------------------------------------------------------- entropy data
def _intervals(data: bytes) -> list:
    """The entropy-coded data from the start up to the marker that ends it, unstuffed and split at RSTn (numbers checked)."""
    out, cur, i, k = [], bytearray(), 0, 0
    while i < len(data):
        b = data[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        j = i
        while j < len(data) and data[j] == 0xFF:      # fill bytes
            j += 1
        if j >= len(data):
            raise ValueError("truncated entropy-coded data")
        if data[j] == 0:
            cur.append(0xFF)
            i = j + 1
        elif 0xD0 <= data[j] <= 0xD7:
            if data[j] != 0xD0 + (k & 7):
                raise ValueError("restart marker out of sequence")
            out.append(bytes(cur))
            cur, k, i = bytearray(), k + 1, j + 1
        else:
            break
    else:
        raise ValueError("truncated entropy-coded data")
    # after the data: APPn / COM segments, then EOI
    while True:
        while j < len(data) and data[j] == 0xFF:
            j += 1
        if j >= len(data):
            raise ValueError("truncated entropy-coded data")
        if data[j] == 0xD9:
            break
        if not (0xE0 <= data[j] <= 0xEF or data[j] == 0xFE) or j + 3 > len(data):
            raise ValueError("a marker inside the entropy-coded data")
        j += 1 + int.from_bytes(data[j + 1:j + 3], "big")
        if j > len(data) or data[j:j + 1] != b"\xff":
            raise ValueError("truncated entropy-coded data")
    out.append(bytes(cur))
    return out


def _decode_interval(bits: str, nblocks: int, slots, h) -> np.ndarray:
    """nblocks zigzag coefficient rows (DC as differences) of one restart interval, decoded from its bit string."""
    coef = np.zeros((nblocks, 64), np.int64)
    pos = 0

    def symbol(table):
        nonlocal pos
        for length in range(1, 17):
            s = table.get((length, int(bits[pos:pos + length], 2) if pos + length <= len(bits) else -1))
            if s is not None:
                pos += length
                return s
        raise ValueError("an invalid Huffman code")

    def extra(s):
        nonlocal pos
        if pos + s > len(bits):
            raise ValueError("truncated entropy-coded data")
        v = int(bits[pos:pos + s], 2)
        pos += s
        return v if v >= 1 << (s - 1) else v - (1 << s) + 1

    for b in range(nblocks):
        c = slots[b % len(slots)]
        s = symbol(h["dc"][c])
        coef[b, 0] = extra(s) if s else 0
        k = 1
        while k < 64:
            rs = symbol(h["ac"][c])
            r, s = rs >> 4, rs & 15
            if s:
                k += r
                if k > 63:
                    raise ValueError("an AC run past coefficient 63")
                coef[b, k] = extra(s)
                k += 1
            elif r == 15:
                k += 16
                if k > 64:
                    raise ValueError("an AC run past coefficient 63")
            else:
                break
    if bits[pos:].strip("1") or len(bits) - pos >= 8:
        raise ValueError("more or fewer blocks than the frame's MCUs")
    return coef


# ---------------------------------------------------------------------------------------------------- pixels
def _c(x):
    return int(x * 8192 + 0.5)


def _s16(x):
    return ((x + 32768) & 0xFFFF) - 32768


def _idct_1d(d, shift, sums, saturate):
    """One islow pass along axis 1 of d (n, 8, ...) in int64, descaled by shift.  ``sums`` names the pairwise sums taken
    modulo 2^16: "even" (d0 + d4, d0 - d4), "odd" (d7 + d3, d5 + d1) and "rotation" (d2 + d6, d7 + d1, d5 + d3, which
    libjpeg-turbo's SIMD code folds into 32-bit multiply-adds).  ``saturate``: the output is saturated to int16."""
    w = {k: (_s16 if k in sums else (lambda x: x)) for k in ("even", "odd", "rotation")}
    z2, z3 = d[:, 2], d[:, 6]
    z1 = w["rotation"](z2 + z3) * _c(0.541196100)
    t2, t3 = z1 - z3 * _c(1.847759065), z1 + z2 * _c(0.765366865)
    t0, t1 = w["even"](d[:, 0] + d[:, 4]) * 8192, w["even"](d[:, 0] - d[:, 4]) * 8192
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = d[:, 7], d[:, 5], d[:, 3], d[:, 1]
    z1, z2, z3, z4 = w["rotation"](o0 + o3), w["rotation"](o1 + o2), w["odd"](o0 + o2), w["odd"](o1 + o3)
    z5 = (z3 + z4) * _c(1.175875602)
    o0, o1, o2, o3 = o0 * _c(0.298631336), o1 * _c(2.053119869), o2 * _c(3.072711026), o3 * _c(1.501321110)
    z1, z2 = z1 * -_c(0.899976223), z2 * -_c(2.562915447)
    z3, z4 = z3 * -_c(1.961570560) + z5, z4 * -_c(0.390180644) + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    out = np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3], 1)
    if np.abs(d).max(initial=0) <= 32768:                   # int16 inputs: the SIMD code's 32-bit sums never overflow
        assert np.abs(out).max(initial=0) < 2**31 - 2**17
    out = (out + (1 << (shift - 1))) >> shift
    return np.clip(out, -32768, 32767) if saturate else out


# The model of cv2's IDCT, step by step; each keyword of idct_islow names one step, and the values other than these are the
# alternatives tests/test_jpeg_decode_range_cpu.py shows cv2 does not take.
IDCT_MODEL = dict(dequant="wrap", shortcut="coef", pass1_sums=("even", "odd"), pass2_sums=("even", "odd"), between="saturate",
                  final="saturate")


def idct_islow(coef: np.ndarray, q: np.ndarray, **steps) -> np.ndarray:
    """(n, 64) natural-order coefficients -> (n, 8, 8) samples, as libjpeg-turbo's SIMD islow IDCT computes them (x86-64):
      dequant   "wrap": the coefficient x quantiser product modulo 2^16 (16-bit lane multiplies); "exact"
      shortcut  "coef": a block whose coefficient rows 1..7 are all zero skips the column pass, and every workspace row is
                row 0's dequantised value shifted left by PASS1_BITS modulo 2^16; "product": the same, decided on the
                dequantised values; None: no shortcut
      pass1_sums, pass2_sums   the pairwise sums each pass takes modulo 2^16 (see _idct_1d)
      between   "saturate": the column pass output saturated to int16 (a saturating pack); "wrap": modulo 2^16; None: exact
      final     "saturate": clamped to [-128, 127], + 128; "wrap": the low 8 bits, + 128
    """
    s = dict(IDCT_MODEL, **steps)
    coef = np.asarray(coef, np.int64).reshape(-1, 64)
    deq = coef * np.asarray(q, np.int64).reshape(64)
    if s["dequant"] == "wrap":
        deq = _s16(deq)
    d = deq.reshape(-1, 8, 8)
    ws = _idct_1d(d, 11, s["pass1_sums"], s["between"] == "saturate")          # along the rows index: columns first
    if s["between"] == "wrap":
        ws = _s16(ws)
    if s["shortcut"]:
        dc_only = ~(coef if s["shortcut"] == "coef" else deq).reshape(-1, 8, 8)[:, 1:].any(axis=(1, 2))
        ws[dc_only] = np.repeat(_s16(d[dc_only, :1] * 4), 8, axis=1)
    rows = _idct_1d(ws.transpose(0, 2, 1), 18, s["pass2_sums"], True).transpose(0, 2, 1)
    if s["final"] == "wrap":
        return ((rows + 128) & 0xFF)
    return np.clip(rows, -128, 127) + 128


def _upsample(p: np.ndarray, hs: int, vs: int, H: int, W: int) -> np.ndarray:
    """A chroma plane (cropped to its real extent ch x cw) upsampled to H x W."""
    ch, cw = p.shape
    if hs == 1:
        return p[:H, :W]
    if cw <= 2:
        return np.repeat(np.repeat(p, vs, 0), 2, 1)[:H, :W]
    if vs == 1:
        left, right = np.concatenate([p[:, :1], p[:, :-1]], 1), np.concatenate([p[:, 1:], p[:, -1:]], 1)
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * p + left + 1) >> 2
        out[:, 1::2] = (3 * p + right + 2) >> 2
        return out[:H, :W]
    up, down = np.concatenate([p[:1], p[:-1]], 0), np.concatenate([p[1:], p[-1:]], 0)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    for r, far in ((0, up), (1, down)):
        t = 3 * p + far
        tl, tr = np.concatenate([t[:, :1], t[:, :-1]], 1), np.concatenate([t[:, 1:], t[:, -1:]], 1)
        out[r::2, 0::2] = (3 * t + tl + 8) >> 4
        out[r::2, 1::2] = (3 * t + tr + 7) >> 4
    return out[:H, :W]


def _orient(img: np.ndarray, o: int) -> np.ndarray:
    """cv2's ApplyExifOrientation: flips and transposes."""
    t = lambda a: a.transpose(1, 0, 2)      # noqa: E731
    return {1: lambda a: a, 2: lambda a: a[:, ::-1], 3: lambda a: a[::-1, ::-1], 4: lambda a: a[::-1],
            5: t, 6: lambda a: t(a)[:, ::-1], 7: lambda a: t(a)[::-1, ::-1], 8: lambda a: t(a)[::-1]}[o](img)


def coefficients(data: bytes):
    """(header, blocks): the entropy stage alone.  blocks[c] is component c's (rows, cols, 64) int64 grid of quantised
    coefficients in natural order over whole MCUs, DC as the running prediction taken modulo 2^16 (libjpeg keeps it in an
    int and stores it as a 16-bit JCOEF)."""
    h = parse(data)
    H, W, comps, hs, vs = h["H"], h["W"], h["comps"], h["hs"], h["vs"]
    nc = len(comps)
    mcux, mcuy = (W + 8 * hs - 1) // (8 * hs), (H + 8 * vs - 1) // (8 * vs)
    slots = [0] * (hs * vs) + list(range(1, nc))
    bpm, total = len(slots), mcux * mcuy * len(slots)
    per = h["ri"] * bpm if h["ri"] else total
    ivs = _intervals(data[h["ecs"]:])
    if len(ivs) != (total + per - 1) // per:
        raise ValueError("restart markers miscounted")
    zz = np.concatenate([_decode_interval("".join(format(b, "08b") for b in iv), min(per, total - k * per), slots, h)
                         for k, iv in enumerate(ivs)])
    comp_of = np.tile(np.array(slots), total // bpm)
    for k in range(len(ivs)):                            # DC predictions, reset at each interval
        for c in range(nc):
            sel = np.nonzero(comp_of[k * per:(k + 1) * per] == c)[0] + k * per
            zz[sel, 0] = np.cumsum(zz[sel, 0])
    zz[:, 0] = ((zz[:, 0] + 32768) & 0xFFFF) - 32768
    nat = np.zeros_like(zz)
    nat[:, ZIGZAG] = zz
    blocks = []
    for c in range(nc):
        h_c, v_c = (hs, vs) if c == 0 else (1, 1)
        b = nat[comp_of == c]                            # scan order: MCU rows, MCUs, then the component's v x h blocks
        blocks.append(b.reshape(mcuy, mcux, v_c, h_c, 64).transpose(0, 2, 1, 3, 4).reshape(mcuy * v_c, mcux * h_c, 64))
    return h, blocks


def decode(data: bytes, **idct_steps) -> np.ndarray:
    """The BGR frame; ``idct_steps`` replace steps of the IDCT model (see idct_islow)."""
    h, blocks = coefficients(data)
    H, W, hs, vs = h["H"], h["W"], h["hs"], h["vs"]
    nc = len(blocks)
    planes = []
    for c, b in enumerate(blocks):
        rows, cols = b.shape[:2]
        px = idct_islow(b.reshape(-1, 64), h["q"][c], **idct_steps)
        planes.append(px.reshape(rows, cols, 8, 8).transpose(0, 2, 1, 3).reshape(rows * 8, cols * 8))
    Y = planes[0][:H, :W]
    if nc == 1:
        bgr = np.stack([Y, Y, Y], -1)
    else:
        cw, ch = (W + hs - 1) // hs, (H + vs - 1) // vs
        cb, cr = (_upsample(p[:ch, :cw], hs, vs, H, W) - 128 for p in planes[1:])
        fix = lambda x: int(x * 65536 + 0.5)        # noqa: E731
        r = Y + ((fix(1.40200) * cr + 32768) >> 16)
        g = Y + ((-fix(0.34414) * cb - fix(0.71414) * cr + 32768) >> 16)
        b = Y + ((fix(1.77200) * cb + 32768) >> 16)
        bgr = np.stack([b, g, r], -1)
    return np.ascontiguousarray(_orient(np.clip(bgr, 0, 255).astype(np.uint8), h["orient"]))
