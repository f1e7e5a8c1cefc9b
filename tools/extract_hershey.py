"""Recover OpenCV's FONT_HERSHEY_SIMPLEX glyphs for printable ASCII from the installed cv2 binary and write them as
``headposeestimation-whenet_b200/csrc/hershey_simplex.inc`` (the host text geometry) and ``oracle/hershey_simplex.py`` (the
CPU oracle).  DESIGN.md section 8.8.

OpenCV keeps every Hershey glyph as a string in ``g_HersheyGlyphs`` (an array of ``const char*``) and each face as an ``int``
table: entry 0 holds the face's flags with its base line in the low 4 bits, entries 1..95 the glyph index of ' '..'~'.  The
tool reads them the way putText does:

1. The array: in a position-independent binary each of its slots carries an R_X86_64_RELATIVE relocation whose addend is the
   string's address.  Glyph 0 is "" and glyph 1 is "MWRMNV RMVV PSTS"; the array starts at the relocated slot of glyph 0
   that follows an unrelocated slot and precedes a slot relocated to glyph 1, and runs as long as slots are relocated.
2. The face tables: every 4-byte-aligned run of 96 ints in .rodata whose first entry has base line 9 and whose next 95
   are glyph indices with a blank space glyph.  Several faces share that header; the one whose glyphs render exactly as
   cv2.putText(FONT_HERSHEY_SIMPLEX) is the simplex face.
3. The self-check: every character alone, and all 95 in one string, rendered through oracle/text_oracle.py and compared
   with cv2.putText bit for bit at scales 0.4, 0.5, 1, 2.5 and 7.  Any mismatch is an error.

    python tools/extract_hershey.py            # extract, check, write both files
    python tools/extract_hershey.py --check    # extract, check, and fail if the committed files differ
"""
from __future__ import annotations

import argparse
import os
import struct
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "oracle"))

INC = os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc", "hershey_simplex.inc")
PY = os.path.join(ROOT, "oracle", "hershey_simplex.py")
CHECK_SCALES = (0.4, 0.5, 1.0, 2.5, 7.0)
GLYPH1 = b"MWRMNV RMVV PSTS"
R_X86_64_RELATIVE = 8


class Elf:
    """The few parts of a little-endian ELF64 shared object the extraction reads."""

    def __init__(self, path: str):
        with open(path, "rb") as f:
            self.data = f.read()
        d = self.data
        if d[:4] != b"\x7fELF" or d[4] != 2 or d[5] != 1:
            raise ValueError("%s is not a little-endian ELF64 file" % path)
        shoff, = struct.unpack_from("<Q", d, 0x28)
        shentsize, shnum, shstrndx = struct.unpack_from("<HHH", d, 0x3A)
        raw = [struct.unpack_from("<IIQQQQIIQQ", d, shoff + i * shentsize) for i in range(shnum)]
        names_off = raw[shstrndx][4]
        self.sections = {}
        for name, typ, _flags, addr, off, size, *_ in raw:
            end = d.index(b"\0", names_off + name)
            self.sections[d[names_off + name:end].decode()] = (typ, addr, off, size)

    def section(self, name: str):
        typ, addr, off, size = self.sections[name]
        return addr, self.data[off:off + size]

    def offset(self, vaddr: int) -> int:
        for typ, addr, off, size in self.sections.values():
            if addr and addr <= vaddr < addr + size and typ != 8:     # not SHT_NOBITS
                return off + vaddr - addr
        raise KeyError(hex(vaddr))

    def cstring(self, vaddr: int) -> bytes:
        o = self.offset(vaddr)
        return self.data[o:self.data.index(b"\0", o)]

    def relative_relocs(self) -> dict:
        """r_offset -> addend of every R_X86_64_RELATIVE relocation in .rela.dyn."""
        _, raw = self.section(".rela.dyn")
        r = np.frombuffer(raw, dtype=[("off", "<u8"), ("info", "<u8"), ("add", "<i8")])
        r = r[(r["info"] & 0xFFFFFFFF) == R_X86_64_RELATIVE]
        return dict(zip(r["off"].tolist(), r["add"].tolist()))


def glyph_array(elf: Elf, relocs: dict) -> list:
    rodata_addr, rodata = elf.section(".rodata")
    hits = []
    at = rodata.find(b"\0" + GLYPH1 + b"\0")
    while at >= 0:
        hits.append(rodata_addr + at + 1)
        at = rodata.find(b"\0" + GLYPH1 + b"\0", at + 1)
    # the string is shared by every glyph with the same strokes (simplex 'A' repeats glyph 1): the array starts where the
    # slot before is the empty glyph 0 and the slot before that is not relocated at all
    bases = [o - 8 for o, a in relocs.items() if a in hits and o - 8 in relocs and elf.cstring(relocs[o - 8]) == b""
             and o - 16 not in relocs]
    if len(bases) != 1:
        raise RuntimeError("expected one glyph array starting with \"\", %r; found %d" % (GLYPH1.decode(), len(bases)))
    base = bases[0]
    glyphs = []
    while base + 8 * len(glyphs) in relocs:
        glyphs.append(elf.cstring(relocs[base + 8 * len(glyphs)]).decode("ascii"))
    return glyphs


def face_candidates(elf: Elf, glyphs: list) -> list:
    """(base_line, 95 glyph strings) of every int run in .rodata shaped like a face table with base line 9."""
    _, rodata = elf.section(".rodata")
    a = np.frombuffer(rodata[:len(rodata) // 4 * 4], "<i4").astype(np.int64)
    ok = (a > 0) & (a < len(glyphs))
    run = np.concatenate([[0], np.cumsum(ok)])
    n = len(a) - 96
    starts = np.nonzero((a[:n] >= 0) & (a[:n] < 1 << 16) & ((a[:n] & 15) == 9) &
                        (run[96:96 + n] - run[1:1 + n] == 95))[0]
    out, seen = [], set()
    for s in starts.tolist():
        table = tuple(glyphs[i] for i in a[s + 1:s + 96].tolist())
        if len(table[0]) != 2 or table in seen:        # ' ' has bearings and no strokes
            continue
        seen.add(table)
        out.append((-(int(a[s]) & 15), table))
    return out


def _canvas_check(cv2, base_line: int, glyphs, text: str, scale: float) -> bool:
    import text_oracle as T
    h = int(45 * scale) + 6
    w = int(30 * scale * len(text)) + int(20 * scale) + 6
    org = (int(10 * scale) + 2, int(32 * scale) + 2)
    a = np.zeros((h, w, 3), np.uint8)
    b = a.copy()
    cv2.putText(a, text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, (255, 255, 255), 1, cv2.LINE_8)
    T.put_text(b, text, org, scale, (255, 255, 255), glyphs, base_line)
    return bool(np.array_equal(a, b)) and (text == " " or bool(a.any()))


def self_check(cv2, base_line: int, glyphs, scales=CHECK_SCALES, quick: bool = False) -> list:
    """The characters (or whole-string checks) whose rendering differs from cv2.putText; empty when the table is exact."""
    bad = []
    chars = [chr(c) for c in range(32, 127)]
    for s in scales:
        for ch in chars:
            if not _canvas_check(cv2, base_line, glyphs, ch, s):
                bad.append((ch, s))
                if quick:
                    return bad
        if not _canvas_check(cv2, base_line, glyphs, "".join(chars), s):
            bad.append(("<all>", s))
    return bad


def extract(so_path: str | None = None):
    """(cv2 version, base_line, the 95 glyph strings of ' '..'~'), checked against cv2.putText at every CHECK_SCALES."""
    import cv2
    so_path = so_path or os.path.join(os.path.dirname(cv2.__file__), "cv2.abi3.so")
    elf = Elf(so_path)
    glyphs = glyph_array(elf, elf.relative_relocs())
    found = [c for c in face_candidates(elf, glyphs) if not self_check(cv2, c[0], c[1], scales=(1.0,), quick=True)]
    if len(found) != 1:
        raise RuntimeError("%d face tables render as FONT_HERSHEY_SIMPLEX at scale 1 (want exactly 1)" % len(found))
    base_line, table = found[0]
    bad = self_check(cv2, base_line, table)
    if bad:
        raise RuntimeError("the recovered table differs from cv2.putText at %s" % bad[:10])
    return cv2.__version__, base_line, list(table)


def _c_str(s: str) -> str:
    return '"' + s.replace("\\", "\\\\").replace('"', '\\"') + '"'


HEADER = """{c} Generated by tools/extract_hershey.py from OpenCV {ver} (the cv2 binary's g_HersheyGlyphs and its FONT_HERSHEY_SIMPLEX
{c} face table); checked there against cv2.putText at scales {scales}.  Do not edit.
{c}
{c} The glyphs are the Hershey fonts of Dr. A. V. Hershey (U.S. National Bureau of Standards, 1967; distributed by NTIS), in
{c} the encoding OpenCV ships in modules/imgproc/src/hershey_fonts.cpp.  OpenCV is licensed under the Apache License 2.0.
{c}
{c} Each glyph: its left and right bearing, then the points of its strokes, every coordinate a character minus 'R'; a
{c} space closes a stroke.  Entry i is the character 32 + i.
"""


def render(ver: str, base_line: int, table) -> tuple:
    scales = ", ".join("%g" % s for s in CHECK_SCALES)
    inc = HEADER.format(c="//", ver=ver, scales=scales)
    inc += "constexpr int kHersheyBaseLine = %d;\n" % base_line
    inc += "constexpr const char* kHersheySimplex[95] = {\n"
    inc += "".join("    %s,   // %r\n" % (_c_str(g), chr(32 + i)) for i, g in enumerate(table))
    inc += "};\n"
    py = '"""FONT_HERSHEY_SIMPLEX for printable ASCII (test infrastructure for text_oracle.py).\n\n'
    py += HEADER.format(c="", ver=ver, scales=scales).replace("\n ", "\n").lstrip() + '"""\n'
    py += "BASE_LINE = %d\n\nGLYPHS = (\n" % base_line
    py += "".join("    %r,   # %r\n" % (g, chr(32 + i)) for i, g in enumerate(table))
    py += ")\n"
    return inc, py


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--check", action="store_true", help="fail if the committed files differ from the extraction")
    ap.add_argument("--so", help="the cv2 shared object (default: the installed cv2's)")
    args = ap.parse_args()
    ver, base_line, table = extract(args.so)
    inc, py = render(ver, base_line, table)
    print("cv2 %s: base_line %d, 95 glyphs, self-check passed at scales %s" % (ver, base_line, list(CHECK_SCALES)))
    if args.check:
        same = all(os.path.exists(p) and open(p).read() == t for p, t in ((INC, inc), (PY, py)))
        print("committed tables " + ("match" if same else "DIFFER"))
        return 0 if same else 1
    for p, t in ((INC, inc), (PY, py)):
        with open(p, "w") as f:
            f.write(t)
        print("wrote", os.path.relpath(p, ROOT))
    return 0


if __name__ == "__main__":
    sys.exit(main())
