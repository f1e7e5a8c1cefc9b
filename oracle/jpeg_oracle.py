"""Baseline JPEG encoder in numpy, byte-identical to ``cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, q])`` (OpenCV 4.13's
bundled libjpeg-turbo with its defaults: 4:2:0, Annex K Huffman tables, no restart markers, JFIF 1.01 APP0).
Written from ITU-T T.81 (Annex K tables, baseline Huffman coding) and the IJG quality rule; DESIGN.md section 8.9.

  ``quant_tables(q)``   luma and chroma quantisation tables (natural order) for quality q
  ``header(H, W, q)``   every byte before the entropy-coded segment (SOI .. SOS)
  ``blocks(bgr, q)``    quantised coefficients of every block in scan order (zigzag), dummy blocks included
  ``encode(bgr, q)``    the whole file
"""
from __future__ import annotations

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63])     # natural index of zigzag position k

# T.81 Annex K.1, natural order
LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                   14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                   49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
CHROMA_Q = np.full(64, 99)
CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# T.81 Annex K.3: (code counts by length 1..16, symbols)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aa"
    "b2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7"
    "a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"))
HUFF_TABLES = ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA))    # DHT order: DC0, AC0, DC1, AC1


def quant_tables(q: int):
    """(luma, chroma) int64 tables in natural order: Annex K scaled by the IJG rule, clamped to [1, 255] (baseline)."""
    s = 5000 // q if q < 50 else 200 - 2 * q
    return tuple(np.clip((t * s + 50) // 100, 1, 255) for t in (LUMA_Q, CHROMA_Q))


def huff_codes(spec):
    """symbol -> (code, length) of a canonical Huffman table (T.81 Annex C)."""
    counts, syms = spec
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            out[syms[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def _seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def header(H: int, W: int, q: int) -> bytes:
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for i, t in enumerate(quant_tables(q)):
        out += _seg(0xDB, bytes([i]) + bytes(int(v) for v in t[ZIGZAG]))
    out += _seg(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for tc, (counts, syms) in HUFF_TABLES:
        out += _seg(0xC4, bytes([tc]) + bytes(counts) + bytes(syms))
    return out + _seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


def _fix(c: float) -> int:
    return int(c * 65536 + 0.5)


def ycc(bgr: np.ndarray):
    """libjpeg's fixed-point RGB -> YCbCr (16 fraction bits), int64 planes."""
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    half = 1 << 15
    off = (128 << 16) + half - 1
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off) >> 16
    return y, cb, cr


def _pad_edge(a: np.ndarray, rows: int, cols: int) -> np.ndarray:
    return np.pad(a, ((0, rows - a.shape[0]), (0, cols - a.shape[1])), mode="edge")


def downsample(c: np.ndarray, H: int, W: int) -> np.ndarray:
    """4:2:0 chroma plane, padded to whole 8x8 blocks: columns replicated to 16 * ceil(ceil(W/2)/8) first, the last row once
    if H is odd, then (a + b + c + d + bias) >> 2 with bias 1, 2, 1, 2, ... along a row, then the last downsampled row down
    to the block boundary."""
    cw, ch = -(-W // 2), -(-H // 2)
    bw, bh = 8 * -(-cw // 8), 8 * -(-ch // 8)
    c = _pad_edge(c, 2 * ch, 2 * bw)
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    s = (s + np.tile([1, 2], bw // 2)[None, :]) >> 2
    return _pad_edge(s, bh, bw)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def fdct_islow(blk: np.ndarray) -> np.ndarray:
    """libjpeg's integer FDCT (CONST_BITS 13, PASS1_BITS 2) of (..., 8, 8) samples already centred on 0; rows first.  The
    result is scaled by 8."""
    CB, PB = 13, 2
    F = {k: int(v * (1 << CB) + 0.5) for k, v in (("0298", 0.298631336), ("0390", 0.390180644), ("0541", 0.541196100),
         ("0765", 0.765366865), ("0899", 0.899976223), ("1175", 1.175875602), ("1501", 1.501321110), ("1847", 1.847759065),
         ("1961", 1.961570560), ("2053", 2.053119869), ("2562", 2.562915447), ("3072", 3.072711026))}

    def one_pass(d, first):
        out = np.empty_like(d)
        t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
        t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
        t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
        t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        sh = CB - PB if first else CB + PB
        if first:
            out[..., 0], out[..., 4] = (t10 + t11) << PB, (t10 - t11) << PB
        else:
            out[..., 0], out[..., 4] = _descale(t10 + t11, PB), _descale(t10 - t11, PB)
        z1 = (t12 + t13) * F["0541"]
        out[..., 2] = _descale(z1 + t13 * F["0765"], sh)
        out[..., 6] = _descale(z1 - t12 * F["1847"], sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * F["1175"]
        t4, t5, t6, t7 = t4 * F["0298"], t5 * F["2053"], t6 * F["3072"], t7 * F["1501"]
        z1, z2 = -z1 * F["0899"], -z2 * F["2562"]
        z3, z4 = -z3 * F["1961"] + z5, -z4 * F["0390"] + z5
        out[..., 7] = _descale(t4 + z1 + z3, sh)
        out[..., 5] = _descale(t5 + z2 + z4, sh)
        out[..., 3] = _descale(t6 + z2 + z3, sh)
        out[..., 1] = _descale(t7 + z1 + z4, sh)
        return out

    rows = one_pass(blk.astype(np.int64), True)
    return np.swapaxes(one_pass(np.swapaxes(rows, -1, -2), False), -1, -2)


def quantise(coef: np.ndarray, table: np.ndarray) -> np.ndarray:
    """Round half away from zero of coef / (8 q): (|x| + 4q) // (8q) with the sign restored."""
    q8 = table.reshape(8, 8) * 8
    return np.sign(coef) * ((np.abs(coef) + q8 // 2) // q8)


def _to_blocks(p: np.ndarray) -> np.ndarray:
    h, w = p.shape
    return p.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)       # (block row, block col, 8, 8)


def blocks(bgr: np.ndarray, q: int) -> np.ndarray:
    """(n_mcu * 6, 64) int64 quantised coefficients in zigzag order, MCU order Y00 Y01 Y10 Y11 Cb Cr.  Dummy luma blocks
    (padding an MCU past the image's last block column or row) have AC 0 and the DC of the block coded just before them."""
    H, W = bgr.shape[:2]
    y, cb, cr = ycc(bgr)
    lq, cq = quant_tables(q)
    by, bx = -(-H // 8), -(-W // 8)
    my, mx = -(-H // 16), -(-W // 16)
    lum = quantise(fdct_islow(_to_blocks(_pad_edge(y, 8 * by, 8 * bx)) - 128), lq)
    chroma = [quantise(fdct_islow(_to_blocks(downsample(c, H, W)) - 128), cq) for c in (cb, cr)]
    out = np.zeros((my, mx, 6, 8, 8), np.int64)
    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        sub = lum[dy::2, dx::2]
        out[:sub.shape[0], :sub.shape[1], i] = sub
    out[:, :, 4], out[:, :, 5] = chroma
    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        rows = 2 * np.arange(my)[:, None] + dy >= by
        cols = 2 * np.arange(mx)[None, :] + dx >= bx
        dummy = rows | cols
        if i > 0:
            out[dummy, i] = 0
            out[dummy, i, 0, 0] = out[dummy, i - 1, 0, 0]
    return out.reshape(-1, 64)[:, ZIGZAG]


def _nbits(v: int) -> int:
    return int(abs(v)).bit_length()


def entropy(coefs: np.ndarray) -> bytes:
    """Baseline Huffman coding of ``blocks()`` output: the stuffed entropy-coded segment, the last byte padded with 1s."""
    tabs = [huff_codes(s) for s in (DC_LUMA, AC_LUMA, DC_CHROMA, AC_CHROMA)]
    acc, nacc, out = 0, 0, bytearray()

    def put(code, length):
        nonlocal acc, nacc
        acc = (acc << length) | code
        nacc += length
        while nacc >= 8:
            nacc -= 8
            byte = (acc >> nacc) & 0xFF
            out.append(byte)
            if byte == 0xFF:
                out.append(0)
        acc &= (1 << nacc) - 1

    def put_value(v, n):
        if n:
            put(v if v >= 0 else v + (1 << n) - 1, n)

    pred = [0, 0, 0]
    for b, blk in enumerate(coefs.tolist()):
        comp = 0 if b % 6 < 4 else b % 6 - 3
        dc_t, ac_t = tabs[0:2] if comp == 0 else tabs[2:4]
        diff = blk[0] - pred[comp]
        pred[comp] = blk[0]
        n = _nbits(diff)
        put(*dc_t[n])
        put_value(diff, n)
        run = 0
        for v in blk[1:]:
            if v == 0:
                run += 1
                continue
            while run > 15:
                put(*ac_t[0xF0])
                run -= 16
            n = _nbits(v)
            put(*ac_t[(run << 4) | n])
            put_value(v, n)
            run = 0
        if run:
            put(*ac_t[0x00])
    if nacc:
        put((1 << (8 - nacc)) - 1, 8 - nacc)
    return bytes(out)


def encode(bgr: np.ndarray, q: int = 95) -> bytes:
    """The whole JPEG file of an (H, W, 3) uint8 BGR frame at quality q in 1..100."""
    bgr = np.asarray(bgr)
    assert bgr.dtype == np.uint8 and bgr.ndim == 3 and bgr.shape[2] == 3 and 1 <= q <= 100
    H, W = bgr.shape[:2]
    return header(H, W, q) + entropy(blocks(bgr, q)) + b"\xff\xd9"
