"""JPEG encoding options in numpy, byte-identical to ``cv2.imencode(".jpg", img, params)`` with OpenCV 4.13's bundled libjpeg-turbo
and the sampling, restart-interval, optimised-Huffman and luma/chroma-quality parameters, and on one-channel images.  Built on
``jpeg_oracle`` (the default file, DESIGN.md section 8.9) and written from ITU-T T.81 (restart intervals, DRI, Annex K.2 code
lengths) and libjpeg's documented ``jpeg_gen_optimal_table``; DESIGN.md section 8.11.

  ``encode_ex(img, q, sampling, restart, optimize, chroma_quality)``   the whole file; ``img`` (H, W, 3) BGR or (H, W) gray
  ``header_ex``, ``blocks_ex``, ``entropy_ex``, ``histograms``, ``gen_optimal_table``   its steps
"""
from __future__ import annotations

import numpy as np

from jpeg_oracle import HUFF_TABLES, ZIGZAG, _nbits, _pad_edge, _seg, _to_blocks, fdct_islow, huff_codes, quant_tables, quantise, ycc


# luma (h, v) sampling factors per sampling string; Cb and Cr are always 1 x 1.  A gray file has one 1 x 1 component.
SAMPLING = {"420": (2, 2), "422": (2, 1), "444": (1, 1)}


def layout(sampling: str, channels: int):
    """(h, v, blocks per MCU, luma blocks per MCU) of a scan."""
    h, v = (1, 1) if channels == 1 else SAMPLING[sampling]
    return h, v, h * v + (0 if channels == 1 else 2), h * v


def header_ex(H: int, W: int, q: int, cq: int | None = None, sampling: str = "420", channels: int = 3, restart: int = 0,
              tables=None) -> bytes:
    """SOI .. SOS with options: luma DQT from q, chroma DQT from cq (default q); the luma sampling factors of ``sampling``;
    DRI when restart > 0; ``tables`` = the DHT specs in DHT order (default Annex K).  Gray files have one DQT, a one-component
    SOF0 and DHT DC0 AC0."""
    cq = q if cq is None else cq
    h, v, _, _ = layout(sampling, channels)
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    qt = (quant_tables(q)[0], quant_tables(cq)[1])[:1 if channels == 1 else 2]
    for i, t in enumerate(qt):
        out += _seg(0xDB, bytes([i]) + bytes(int(x) for x in t[ZIGZAG]))
    comps = [1, h << 4 | v, 0] + ([] if channels == 1 else [2, 0x11, 1, 3, 0x11, 1])
    out += _seg(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([channels] + comps))
    specs = [s for _, s in HUFF_TABLES] if tables is None else list(tables)
    for tc, (counts, syms) in zip([t for t, _ in HUFF_TABLES], specs[:2 if channels == 1 else 4]):
        out += _seg(0xC4, bytes([tc]) + bytes(counts) + bytes(syms))
    if restart:
        out += _seg(0xDD, restart.to_bytes(2, "big"))
    sel = [1, 0x00] + ([] if channels == 1 else [2, 0x11, 3, 0x11])
    return out + _seg(0xDA, bytes([channels] + sel + [0, 63, 0]))


def downsample_ex(c: np.ndarray, H: int, W: int, h: int, v: int) -> np.ndarray:
    """A chroma plane at 1/h x 1/v, padded to whole 8x8 blocks: columns replicated to 8h * ceil(ceil(W/h)/8), rows to
    v * ceil(H/v); then the h x v sums plus a bias that alternates along a row (4:2:0: 1, 2; 4:2:2: 0, 1), shifted down; then
    the last downsampled row replicated to the block boundary."""
    cw, ch = -(-W // h), -(-H // v)
    bw, bh = 8 * -(-cw // 8), 8 * -(-ch // 8)
    c = _pad_edge(c, v * ch, h * bw)
    s = sum(c[dy::v, dx::h] for dy in range(v) for dx in range(h))
    bias = {1: [0, 0], 2: [0, 1], 4: [1, 2]}[h * v]
    s = (s + np.tile(bias, bw // 2)[None, :]) >> {1: 0, 2: 1, 4: 2}[h * v]
    return _pad_edge(s, bh, bw)


def blocks_ex(img: np.ndarray, q: int, cq: int | None = None, sampling: str = "420") -> np.ndarray:
    """(n_mcu * blocks per MCU, 64) int64 quantised zigzag coefficients in scan order.  BGR: luma blocks of an MCU row by row,
    then Cb, Cr; a luma block past the image's last block column or row (only where an MCU has two luma blocks along that axis)
    has AC 0 and the DC of the block before it in the MCU.  Gray (an (H, W) image): the samples themselves, one block per MCU."""
    cq = q if cq is None else cq
    gray = img.ndim == 2
    H, W = img.shape[:2]
    h, v, bpm, ny = layout(sampling, 1 if gray else 3)
    if gray:
        y, chroma_planes = img.astype(np.int64), ()
    else:
        y, cb, cr = ycc(img)
        chroma_planes = (cb, cr)
    lq, cqt = quant_tables(q)[0], quant_tables(cq)[1]
    by, bx = -(-H // 8), -(-W // 8)
    my, mx = -(-H // (8 * v)), -(-W // (8 * h))
    lum = quantise(fdct_islow(_to_blocks(_pad_edge(y, 8 * by, 8 * bx)) - 128), lq)
    out = np.zeros((my, mx, bpm, 8, 8), np.int64)
    for i in range(ny):
        dy, dx = divmod(i, h)
        sub = lum[dy::v, dx::h]
        out[:sub.shape[0], :sub.shape[1], i] = sub
    for j, c in enumerate(chroma_planes):
        out[:, :, ny + j] = quantise(fdct_islow(_to_blocks(downsample_ex(c, H, W, h, v)) - 128), cqt)
    for i in range(1, ny):
        dy, dx = divmod(i, h)
        dummy = (v * np.arange(my)[:, None] + dy >= by) | (h * np.arange(mx)[None, :] + dx >= bx)
        out[dummy, i] = 0
        out[dummy, i, 0, 0] = out[dummy, i - 1, 0, 0]
    return out.reshape(-1, 64)[:, ZIGZAG]


def _symbols(coefs: np.ndarray, bpm: int, ny: int, restart: int):
    """The scan's Huffman symbols in order: (kind, table, symbol, extra bits, count of extra bits), kind "sym"; and a
    ("rst", m) item before the first MCU of every restart interval but the first.  table 0 DC luma, 1 AC luma, 2 DC chroma,
    3 AC chroma.  DC predictions reset to 0 at every interval."""
    pred = [0, 0, 0]
    for b, blk in enumerate(coefs.tolist()):
        mcu, k = divmod(b, bpm)
        if k == 0 and restart and mcu and mcu % restart == 0:
            yield ("rst", (mcu // restart - 1) % 8)
            pred = [0, 0, 0]
        comp = 0 if k < ny else k - ny + 1
        t = 0 if comp == 0 else 2
        diff = blk[0] - pred[comp]
        pred[comp] = blk[0]
        n = _nbits(diff)
        yield ("sym", t, n, diff if diff >= 0 else diff + (1 << n) - 1, n)
        run = 0
        for x in blk[1:]:
            if x == 0:
                run += 1
                continue
            while run > 15:
                yield ("sym", t + 1, 0xF0, 0, 0)
                run -= 16
            n = _nbits(x)
            yield ("sym", t + 1, (run << 4) | n, x if x >= 0 else x + (1 << n) - 1, n)
            run = 0
        if run:
            yield ("sym", t + 1, 0x00, 0, 0)


def histograms(coefs: np.ndarray, bpm: int, ny: int, restart: int = 0) -> np.ndarray:
    """(4, 256) int64 symbol counts of the scan per table (the walk of ``entropy_ex``)."""
    out = np.zeros((4, 256), np.int64)
    for it in _symbols(coefs, bpm, ny, restart):
        if it[0] == "sym":
            out[it[1], it[2]] += 1
    return out


def gen_optimal_table(freq):
    """libjpeg's jpeg_gen_optimal_table on 256 symbol counts: (bits[16] = codes per length 1..16, symbols by length then
    value).  A reserved symbol 256 with count 1 keeps any code from being all 1 bits; each step merges the two smallest
    nonzero counts, ties going to the larger index; lengths past 16 are folded back by the T.81 Annex K.2 adjustment."""
    freq = [int(x) for x in freq] + [1]
    codesize, others = [0] * 257, [-1] * 257
    while True:
        c1 = c2 = -1
        v = 1000000000
        for i in range(257):
            if freq[i] and freq[i] <= v:
                v, c1 = freq[i], i
        v = 1000000000
        for i in range(257):
            if freq[i] and freq[i] <= v and i != c1:
                v, c2 = freq[i], i
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    vals = [j for n in range(1, 33) for j in range(256) if codesize[j] == n]
    return bits[1:17], vals


def entropy_ex(coefs: np.ndarray, bpm: int, ny: int, restart: int = 0, tables=None) -> bytes:
    """The stuffed entropy-coded data: ``tables`` (DHT order, default Annex K), each restart interval padded with 1 bits to a
    byte and followed by RSTm (m = interval mod 8) except the last."""
    specs = [s for _, s in HUFF_TABLES] if tables is None else list(tables)
    tabs = [huff_codes(s) for s in specs]
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

    for it in _symbols(coefs, bpm, ny, restart):
        if it[0] == "rst":
            if nacc:
                put((1 << (8 - nacc)) - 1, 8 - nacc)
            out += bytes([0xFF, 0xD0 + it[1]])
            continue
        _, t, sym, extra, n = it
        put(*tabs[t][sym])
        if n:
            put(extra, n)
    if nacc:
        put((1 << (8 - nacc)) - 1, 8 - nacc)
    return bytes(out)


def encode_ex(img: np.ndarray, q: int = 95, sampling: str = "420", restart: int = 0, optimize: bool = False,
              chroma_quality: int | None = None) -> bytes:
    """The whole file of an (H, W, 3) BGR or (H, W) gray uint8 image, equal to cv2.imencode with QUALITY q (or LUMA_QUALITY q
    and CHROMA_QUALITY chroma_quality, which needs sampling "444"), SAMPLING_FACTOR, RST_INTERVAL restart and OPTIMIZE."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and (img.ndim == 2 or (img.ndim == 3 and img.shape[2] == 3)) and 1 <= q <= 100
    channels = 1 if img.ndim == 2 else 3
    H, W = img.shape[:2]
    _, _, bpm, ny = layout(sampling, channels)
    coefs = blocks_ex(img, q, chroma_quality, sampling)
    tables = None
    if optimize:
        tables = [gen_optimal_table(f) for f in histograms(coefs, bpm, ny, restart)[:2 if channels == 1 else 4]]
    return (header_ex(H, W, q, chroma_quality, sampling, channels, restart, tables)
            + entropy_ex(coefs, bpm, ny, restart, tables) + b"\xff\xd9")
