"""Coefficient-level baseline JPEG writer for the decoder tests: quantised coefficient blocks in, a valid file out, so that a
test can put any coefficient a baseline file may hold in front of the IDCT (an encoder fed 8-bit pixels never makes most of
them).

    write(blocks, q, H, W, sampling="444", restart=0, tables=None) -> bytes

``blocks`` is one int array per component of shape (rows, cols, 64): quantised coefficients in natural (row-major) order,
DC as its value (the writer codes the differences; a running DC past int16 is allowed, a decoder keeps it modulo 2^16).  The
component block grids are whole MCUs: luma (mcuy * v, mcux * h) blocks and chroma (mcuy, mcux) for the sampling's (h, v).
``q`` holds one 64-entry natural-order table per component; a table with an entry above 255 goes out as a 16-bit DQT under
SOF1.  ``restart`` is the DRI interval in MCUs.  ``tables`` maps (class, slot) to (counts, symbols) and defaults to the
T.81 Annex K tables; luma uses slot 0, chroma slot 1.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
from jpeg_oracle import AC_CHROMA, AC_LUMA, DC_CHROMA, DC_LUMA, ZIGZAG, huff_codes  # noqa: E402

SAMPLING = {"gray": (1, 1), "444": (1, 1), "422": (2, 1), "420": (2, 2)}       # luma (h, v)
ANNEX_K = {(0, 0): DC_LUMA, (1, 0): AC_LUMA, (0, 1): DC_CHROMA, (1, 1): AC_CHROMA}


def grid(H: int, W: int, sampling: str):
    """[(rows, cols)] of each component's block grid for an H x W frame."""
    h, v = SAMPLING[sampling]
    mcux, mcuy = -(-W // (8 * h)), -(-H // (8 * v))
    return [(mcuy * v, mcux * h)] + ([(mcuy, mcux)] * 2 if sampling != "gray" else [])


def _seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def write(blocks, q, H: int, W: int, sampling: str = "444", restart: int = 0, tables=None) -> bytes:
    nc = 1 if sampling == "gray" else 3
    hs, vs = SAMPLING[sampling]
    blocks = [np.asarray(b, np.int64) for b in blocks]
    q = [np.asarray(t, np.int64).reshape(64) for t in q]
    if len(blocks) != nc or len(q) != nc:
        raise ValueError("%d components expected" % nc)
    if [b.shape for b in blocks] != [g + (64,) for g in grid(H, W, sampling)]:
        raise ValueError("block grids %s do not match %dx%d %s" % ([b.shape for b in blocks], H, W, sampling))
    if not 1 <= H <= 65535 or not 1 <= W <= 65535 or not 0 <= restart <= 65535:
        raise ValueError("size or restart interval out of range")
    wide = any(int(t.max()) > 255 for t in q)
    if any(int(t.min()) < 1 or int(t.max()) > 65535 for t in q):
        raise ValueError("quantiser outside [1, 65535]")
    for b in blocks:
        if np.abs(b[..., 1:]).max(initial=0) > 1023:
            raise ValueError("AC coefficient above category 10")
    tables = {**ANNEX_K, **(tables or {})}
    codes = {k: huff_codes(v) for k, v in tables.items()}

    out = bytearray(b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"))
    for c in range(nc):
        out += _seg(0xDB, bytes([(16 if wide else 0) | c]) + b"".join(int(v).to_bytes(2 if wide else 1, "big") for v in q[c][ZIGZAG]))
    sof = bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([nc])
    for c in range(nc):
        sof += bytes([c + 1, (hs << 4 | vs) if c == 0 else 0x11, c])
    out += _seg(0xC1 if wide else 0xC0, sof)
    for (cls, slot), (counts, syms) in sorted(tables.items(), key=lambda kv: (kv[0][1], kv[0][0])):
        if slot < nc:
            out += _seg(0xC4, bytes([cls << 4 | slot]) + bytes(counts) + bytes(syms))
    if restart:
        out += _seg(0xDD, restart.to_bytes(2, "big"))
    out += _seg(0xDA, bytes([nc]) + b"".join(bytes([c + 1, 0x11 * min(c, 1)]) for c in range(nc)) + b"\x00\x3f\x00")

    acc, nacc, seg = 0, 0, bytearray()

    def put(code_len, value=0, n=0):
        nonlocal acc, nacc
        code, length = code_len
        acc, nacc = (acc << length | code) << n | (value if value >= 0 else value + (1 << n) - 1) & ((1 << n) - 1), nacc + length + n
        while nacc >= 8:
            nacc -= 8
            byte = acc >> nacc & 0xFF
            seg.append(byte)
            if byte == 0xFF:
                seg.append(0)
        acc &= (1 << nacc) - 1

    def symbol(table, s):
        if s not in table:
            raise ValueError("symbol 0x%02x is not in the Huffman table" % s)
        return table[s]

    def flush():
        if nacc:
            put(((1 << (8 - nacc)) - 1, 8 - nacc))

    rows, cols = grid(H, W, sampling)[0]
    mcux, mcuy = cols // hs, rows // vs
    pred = [0] * nc
    for m in range(mcux * mcuy):
        if restart and m and m % restart == 0:
            flush()
            seg += bytes([0xFF, 0xD0 + (m // restart - 1) % 8])
            pred = [0] * nc
        my, mx = divmod(m, mcux)
        units = [(0, my * vs + y, mx * hs + x) for y in range(vs) for x in range(hs)] + [(c, my, mx) for c in range(1, nc)]
        for c, by, bx in units:
            blk, slot = blocks[c][by, bx], min(c, 1)
            dc_t, ac_t = codes[(0, slot)], codes[(1, slot)]
            diff = int(blk[0]) - pred[c]
            pred[c] = int(blk[0])
            n = abs(diff).bit_length()
            if n > 11:
                raise ValueError("DC difference %d above category 11" % diff)
            put(symbol(dc_t, n), diff, n)
            run = 0
            for v in blk[ZIGZAG[1:]].tolist():
                if v == 0:
                    run += 1
                    continue
                while run > 15:
                    put(symbol(ac_t, 0xF0))
                    run -= 16
                n = abs(v).bit_length()
                put(symbol(ac_t, run << 4 | n), v, n)
                run = 0
            if run:
                put(symbol(ac_t, 0x00))
    flush()
    return bytes(out + seg + b"\xff\xd9")


# ---------------------------------------------------------------------------------------------------- synthetic files
# Coefficient kinds that reach the IDCT's 16-bit steps (and one that does not):
#   small    |coef| <= 3, q <= 8: the control, nothing wraps or saturates
#   dc       DC only, |DC| <= 1023, q <= 255: the DC-only column shortcut
#   row0     DC and row 0 only (no AC in rows 1..7): the shortcut with horizontal frequencies
#   dense    every AC up to +-1023, q <= 255: products modulo 2^16, saturation between the passes
#   sparse   AC up to +-1023 at 10 % density, q <= 255
#   mid      AC up to +-60 at 20 % density, q <= 40: every product fits in int16, only the sums and the packs act
#   wide     16-bit DQT (SOF1), q 200..3000, AC up to +-5
#   wild     16-bit DQT, q 1..65535, AC up to +-3: any int16 dequantised value
#   mixed    each block one of the kinds above (the 8-bit ones), so neighbouring blocks take different IDCT paths
KINDS = ["small", "dc", "row0", "dense", "sparse", "mid", "wide", "wild", "mixed"]


def _kind_blocks(rng, kind, n):
    b = np.zeros((n, 64), np.int64)
    b[:, 0] = rng.integers(-1023, 1024, n)
    if kind == "small":
        b[:] = rng.integers(-3, 4, (n, 64))
    elif kind == "row0":
        b[:, 1:8] = rng.integers(-1023, 1024, (n, 7)) * (rng.random((n, 7)) < 0.5)
    elif kind == "dense":
        b[:, 1:] = rng.integers(-1023, 1024, (n, 63))
    elif kind == "sparse":
        b[:, 1:] = rng.integers(-1023, 1024, (n, 63)) * (rng.random((n, 63)) < 0.1)
    elif kind == "mid":
        b[:, 0] = rng.integers(-60, 61, n)
        b[:, 1:] = rng.integers(-60, 61, (n, 63)) * (rng.random((n, 63)) < 0.2)
    elif kind == "wide":
        b[:] = rng.integers(-5, 6, (n, 64))
    elif kind == "wild":
        b[:] = rng.integers(-3, 4, (n, 64))
    elif kind == "mixed":
        pick = rng.integers(0, 6, n)
        for k, sub in enumerate(["small", "dc", "row0", "dense", "sparse", "mid"]):
            b[pick == k] = _kind_blocks(rng, sub, n)[pick == k]
    return b


def _kind_q(rng, kind):
    hi = {"small": 8, "mid": 40}.get(kind, 255)
    if kind == "wide":
        return rng.integers(200, 3001, 64)
    if kind == "wild":
        return rng.integers(1, 65536, 64)
    return rng.integers(1, hi + 1, 64)


def synthetic(kind: str, H: int, W: int, sampling: str, restart: int = 0, seed: int = 0):
    """(file, blocks, q) of one seeded file of ``kind`` coefficients."""
    rng = np.random.default_rng([seed, KINDS.index(kind), H, W, list(SAMPLING).index(sampling), restart])
    blocks = [_kind_blocks(rng, kind, r * c).reshape(r, c, 64) for r, c in grid(H, W, sampling)]
    q = [_kind_q(rng, kind) for _ in blocks]
    return write(blocks, q, H, W, sampling, restart), blocks, q


def matrix(sizes=((16, 32), (37, 53)), restarts=(0, 3), seed=0):
    """[(name, file)] of every kind x sampling x size x restart interval."""
    return [("%s-%s-%dx%d-r%d" % (k, s, h, w, r), synthetic(k, h, w, s, r, seed)[0])
            for k in KINDS for s in SAMPLING for h, w in sizes for r in restarts]
