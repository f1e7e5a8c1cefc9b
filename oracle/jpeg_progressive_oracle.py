"""Progressive JPEG encoding in numpy, byte-identical to ``cv2.imencode(".jpg", img, params + [IMWRITE_JPEG_PROGRESSIVE, 1])``
with OpenCV 4.13's bundled libjpeg-turbo.  The quantised coefficients are ``jpeg_options_oracle.blocks_ex``'s (the same as the
optimised baseline file's); what is new is the entropy coding, restated from ITU-T T.81 Annex G (spectral selection,
successive approximation, EOB runs) and libjpeg's documented progressive Huffman coder (its default scan script, optimal
tables per scan, the 0x7FFF run cap and its 1000-bit correction-bit buffer).  DESIGN.md section 8.12.

  ``encode_progressive(img, q, sampling, restart, chroma_quality)``   the whole file; ``img`` (H, W, 3) BGR or (H, W) gray
  ``scan_script(channels)``, ``scan_units``, ``scan_symbols``, ``scan_data``   its steps
  ``STATS``   counters of the last ``encode_progressive`` call, so tests can show which rules a case reached
"""
from __future__ import annotations

import numpy as np

from jpeg_oracle import _nbits, _seg, huff_codes, quant_tables, ZIGZAG
from jpeg_options_oracle import blocks_ex, gen_optimal_table, layout

# (component indices, Ss, Se, Ah, Al): libjpeg's jpeg_simple_progression for YCbCr and for one component
SCRIPT_COLOR = (((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((0,), 6, 63, 0, 2),
                ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0))
SCRIPT_GRAY = (((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
               ((0,), 1, 63, 1, 0))
EOBRUN_MAX = 0x7FFF
BE_MAX = 1000 - 64 + 1      # a run is flushed once its buffered correction bits exceed this (libjpeg's MAX_CORR_BITS)

STATS: dict = {}


def scan_script(channels: int):
    return SCRIPT_GRAY if channels == 1 else SCRIPT_COLOR


def scan_units(coefs: np.ndarray, H: int, W: int, sampling: str, channels: int, comps):
    """The scan's MCUs in order, each a list of (component, block row in ``coefs``).  Interleaved (several components): the
    frame's MCUs, dummy blocks included.  One component: its own block grid in raster order, ceil(ceil(W h / hmax) / 8) x
    ceil(ceil(H v / vmax) / 8) blocks, which skips the dummy blocks an MCU pads with."""
    h, v, bpm, ny = layout(sampling, channels)
    mx, my = -(-W // (8 * h)), -(-H // (8 * v))
    comp_of = [0] * ny + [1, 2][:bpm - ny]
    if len(comps) > 1:
        return [[(comp_of[b], m * bpm + b) for b in range(bpm)] for m in range(mx * my)]
    c = comps[0]
    if c == 0:
        bw, bh = -(-W // 8), -(-H // 8)
        return [[(0, ((by // v) * mx + bx // h) * bpm + (by % v) * h + bx % h)] for by in range(bh) for bx in range(bw)]
    return [[(c, m * bpm + ny + c - 1)] for m in range(mx * my)]


def _band(blk, Ss, Se, Al):
    """(absolute values >> Al, signs) of zigzag positions Ss..Se"""
    vals = [int(x) for x in blk[Ss:Se + 1]]
    return [abs(x) >> Al for x in vals], [x < 0 for x in vals]


def scan_symbols(coefs: np.ndarray, units, comps, Ss, Se, Ah, Al, restart: int, stats: dict):
    """The scan's items in order: ("sym", table slot, symbol, extra bits, count), ("bits", value, count) for raw bits, and
    ("rst",) at each restart.  Table slot 0 is the DC table of component 0 or the scan's AC table, 1 the chroma DC table."""
    dc = Ss == 0
    pred = [0, 0, 0]
    eobrun, be = 0, []              # pending EOB run and its buffered correction bits

    def flush():
        nonlocal eobrun, be
        if eobrun:
            n = eobrun.bit_length() - 1
            yield ("sym", 0, n << 4, eobrun & ((1 << n) - 1), n)
            for bit in be:
                yield ("bits", bit, 1)
            eobrun, be = 0, []

    for u, mcu in enumerate(units):
        if restart and u and u % restart == 0:
            yield from flush()
            yield ("rst",)
            pred = [0, 0, 0]
        for comp, b in mcu:
            blk = coefs[b]
            if dc and Ah == 0:
                v = int(blk[0]) >> Al
                diff, pred[comp] = v - pred[comp], v
                n = _nbits(diff)
                yield ("sym", 0 if comp == 0 else 1, n, diff if diff >= 0 else diff + (1 << n) - 1, n)
            elif dc:
                yield ("bits", (int(blk[0]) >> Al) & 1, 1)
            elif Ah == 0:
                a, neg = _band(blk, Ss, Se, Al)
                r = 0
                for k, x in enumerate(a):
                    if x == 0:
                        r += 1
                        continue
                    yield from flush()
                    while r > 15:
                        yield ("sym", 0, 0xF0, 0, 0)
                        r -= 16
                    n = x.bit_length()
                    yield ("sym", 0, (r << 4) | n, (~x if neg[k] else x) & ((1 << n) - 1), n)
                    r = 0
                if r:
                    eobrun += 1
                    if eobrun == EOBRUN_MAX:
                        stats["eobrun_cap"] = stats.get("eobrun_cap", 0) + 1
                        yield from flush()
            else:
                a, neg = _band(blk, Ss, Se, Al)
                last_new = max([k for k, x in enumerate(a) if x == 1], default=-1)
                r, br = 0, []
                for k, x in enumerate(a):
                    if x == 0:
                        r += 1
                        continue
                    while r > 15 and k <= last_new:
                        yield from flush()
                        yield ("sym", 0, 0xF0, 0, 0)
                        r -= 16
                        for bit in br:
                            yield ("bits", bit, 1)
                        br = []
                    if x > 1:
                        br.append(x & 1)
                        continue
                    yield from flush()
                    yield ("sym", 0, (r << 4) | 1, 0 if neg[k] else 1, 1)
                    for bit in br:
                        yield ("bits", bit, 1)
                    br, r = [], 0
                if r or br:
                    eobrun += 1
                    be += br
                    if eobrun == EOBRUN_MAX or len(be) > BE_MAX:
                        key = "eobrun_cap" if eobrun == EOBRUN_MAX else "be_cap"
                        stats[key] = stats.get(key, 0) + 1
                        yield from flush()
    yield from flush()


def scan_data(items, tables) -> bytes:
    """The stuffed entropy-coded data of one scan: each restart interval padded with 1 bits and followed by RSTm (m counts
    the scan's intervals mod 8), the last one padded."""
    codes = [huff_codes(t) for t in tables]
    acc, nacc, out, m = 0, 0, bytearray(), 0

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

    for it in items:
        if it[0] == "rst":
            if nacc:
                put((1 << (8 - nacc)) - 1, 8 - nacc)
            out += bytes([0xFF, 0xD0 + m])
            m = (m + 1) & 7
        elif it[0] == "bits":
            put(it[1], it[2])
        else:
            put(*codes[it[1]][it[2]])
            if it[4]:
                put(it[3], it[4])
    if nacc:
        put((1 << (8 - nacc)) - 1, 8 - nacc)
    return bytes(out)


def header_progressive(H: int, W: int, q: int, cq: int, sampling: str, channels: int) -> bytes:
    """SOI, APP0, DQT (luma, then chroma), SOF2"""
    h, v, _, _ = layout(sampling, channels)
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    qt = (quant_tables(q)[0], quant_tables(cq)[1])[:1 if channels == 1 else 2]
    for i, t in enumerate(qt):
        out += _seg(0xDB, bytes([i]) + bytes(int(x) for x in t[ZIGZAG]))
    comps = [1, h << 4 | v, 0] + ([] if channels == 1 else [2, 0x11, 1, 3, 0x11, 1])
    return out + _seg(0xC2, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([channels] + comps))


def encode_progressive(img: np.ndarray, q: int = 95, sampling: str = "420", restart: int = 0,
                       chroma_quality: int | None = None) -> bytes:
    """The whole progressive file of an (H, W, 3) BGR or (H, W) gray uint8 image: the header, then for each scan of
    ``scan_script`` its DHTs (optimal tables from the scan's own symbols; none for a DC refinement scan), DRI before the
    first SOS when ``restart`` > 0, SOS and the data; then EOI.  ``STATS`` gets the counters of this call."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and (img.ndim == 2 or (img.ndim == 3 and img.shape[2] == 3)) and 1 <= q <= 100
    channels = 1 if img.ndim == 2 else 3
    cq = q if chroma_quality is None else chroma_quality
    H, W = img.shape[:2]
    coefs = blocks_ex(img, q, cq, sampling)
    STATS.clear()
    STATS.update(eobrun_cap=0, be_cap=0, units=[])
    out = header_progressive(H, W, q, cq, sampling, channels)
    for sc, (comps, Ss, Se, Ah, Al) in enumerate(scan_script(channels)):
        units = scan_units(coefs, H, W, sampling, channels, comps)
        STATS["units"].append(len(units))
        items = list(scan_symbols(coefs, units, comps, Ss, Se, Ah, Al, restart, STATS))
        tables = []
        if not (Ss == 0 and Ah):
            hist = np.zeros((2, 256), np.int64)
            for it in items:
                if it[0] == "sym":
                    hist[it[1], it[2]] += 1
            nt = 2 if Ss == 0 and len(comps) > 1 else 1
            tables = [gen_optimal_table(hist[t]) for t in range(nt)]
            for t, (counts, syms) in enumerate(tables):
                tc = t if Ss == 0 else 0x10 | (0 if comps[0] == 0 else 1)
                out += _seg(0xC4, bytes([tc]) + bytes(counts) + bytes(syms))
        if sc == 0 and restart:
            out += _seg(0xDD, restart.to_bytes(2, "big"))
        sel = []
        for c in comps:
            t = 0 if c == 0 else 1
            sel += [c + 1, (t << 4 if Ah == 0 else 0) if Ss == 0 else t]
        out += _seg(0xDA, bytes([len(comps)] + sel + [Ss, Se, Ah << 4 | Al]))
        out += scan_data(items, tables)
    return out + b"\xff\xd9"
