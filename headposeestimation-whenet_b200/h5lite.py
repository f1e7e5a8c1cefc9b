"""Minimal pure-Python reader for Keras-2.1.6 ``save_weights`` HDF5 files.

The reference loads ``WHENet.h5`` through ``keras.Model.load_weights``
(reference ``whenet.py:15-16``), which needs h5py/libhdf5 - neither exists in
this image.  The file uses only the oldest, simplest HDF5 structures
(SURVEY.md section 8c): superblock v0, v1 object headers, symbol-table groups
(v1 B-tree + SNOD leaves + local heap), contiguous little-endian float32
datasets and v1 attributes holding fixed-length string arrays.  This module
walks exactly those structures and nothing else; anything different raises
``H5FormatError`` instead of guessing.

Public API
----------
``read_keras_weights(path) -> (layer_names, {"<layer>/<weight>:0": ndarray})``
``H5File(path)`` for lower-level access (``attrs``, ``visit`` ...).
"""
from __future__ import annotations

import struct
from collections import OrderedDict

import numpy as np

UNDEF = 0xFFFFFFFFFFFFFFFF


class H5FormatError(ValueError):
    pass


class _Obj:
    """Parsed v1 object header: list of (type, flags, body-bytes)."""

    def __init__(self, msgs):
        self.msgs = msgs

    def first(self, mtype):
        for t, _f, body in self.msgs:
            if t == mtype:
                return body
        return None

    def all(self, mtype):
        return [body for t, _f, body in self.msgs if t == mtype]


class H5File:
    def __init__(self, path):
        with open(path, "rb") as f:
            self.buf = f.read()
        b = self.buf
        if b[:8] != b"\x89HDF\r\n\x1a\n":
            raise H5FormatError("not an HDF5 file: %r" % (path,))
        if b[8] != 0:
            raise H5FormatError("only superblock v0 is supported, got v%d" % b[8])
        if b[13] != 8 or b[14] != 8:
            raise H5FormatError("only 8-byte offsets/lengths are supported")
        base, _free, eof, _drv = struct.unpack_from("<QQQQ", b, 24)
        if base != 0:
            raise H5FormatError("non-zero base address")
        if eof != len(b):
            raise H5FormatError("truncated file: eof=%d size=%d" % (eof, len(b)))
        # root symbol-table entry at byte 56
        _name_off, self.root_addr, cache, _res = struct.unpack_from("<QQII", b, 56)
        self._obj_cache = {}

    # ------------------------------------------------------------------ headers
    def obj(self, addr) -> _Obj:
        o = self._obj_cache.get(addr)
        if o is None:
            o = self._parse_obj(addr)
            self._obj_cache[addr] = o
        return o

    def _parse_obj(self, addr) -> _Obj:
        b = self.buf
        ver, _r, nmsg, _ref, hsize = struct.unpack_from("<BBHII", b, addr)
        if ver != 1:
            raise H5FormatError("only v1 object headers are supported (got %d @%d)" % (ver, addr))
        msgs = []
        # first chunk starts after the 12-byte prefix padded to 8 -> 16
        chunks = [(addr + 16, hsize)]
        while chunks and len(msgs) < nmsg:
            pos, size = chunks.pop(0)
            end = pos + size
            while pos + 8 <= end and len(msgs) < nmsg:
                mtype, msize, mflags = struct.unpack_from("<HHB", b, pos)
                body = b[pos + 8: pos + 8 + msize]
                pos += 8 + msize
                if mtype == 0x10:  # continuation
                    caddr, clen = struct.unpack_from("<QQ", body, 0)
                    chunks.append((caddr, clen))
                msgs.append((mtype, mflags, body))
        return _Obj(msgs)

    # ------------------------------------------------------------------- groups
    def _heap_data(self, heap_addr):
        b = self.buf
        if b[heap_addr:heap_addr + 4] != b"HEAP":
            raise H5FormatError("bad local heap signature @%d" % heap_addr)
        _dsize, _free, daddr = struct.unpack_from("<QQQ", b, heap_addr + 8)
        return daddr

    def _walk_btree(self, addr, heap_data, out):
        b = self.buf
        sig = b[addr:addr + 4]
        if sig == b"TREE":
            ntype, level, nent = struct.unpack_from("<BBH", b, addr + 4)
            if ntype != 0:
                raise H5FormatError("unexpected B-tree node type %d" % ntype)
            pos = addr + 8 + 16  # skip left/right sibling
            # keys and children interleave: key0 child0 key1 child1 ... keyN
            pos += 8
            for _ in range(nent):
                child, = struct.unpack_from("<Q", b, pos)
                pos += 16  # child + next key
                self._walk_btree(child, heap_data, out)
        elif sig == b"SNOD":
            _ver, _r, nsym = struct.unpack_from("<BBH", b, addr + 4)
            pos = addr + 8
            for _ in range(nsym):
                name_off, oaddr = struct.unpack_from("<QQ", b, pos)
                pos += 40
                s = heap_data + name_off
                e = b.index(b"\x00", s)
                out.append((b[s:e].decode("utf-8"), oaddr))
        else:
            raise H5FormatError("bad group node signature %r @%d" % (sig, addr))

    def children(self, addr):
        """[(name, object-header address)] of a group, sorted by name."""
        st = self.obj(addr).first(0x11)
        if st is None:
            return None
        btree, heap = struct.unpack_from("<QQ", st, 0)
        out = []
        self._walk_btree(btree, self._heap_data(heap), out)
        return out

    def is_group(self, addr):
        return self.obj(addr).first(0x11) is not None

    # --------------------------------------------------------------- datatypes
    @staticmethod
    def _parse_dtype(body):
        cls_ver, b0, _b1, _b2, size = struct.unpack_from("<BBBBI", body, 0)
        cls = cls_ver & 0x0F
        if cls == 1:  # floating point
            if b0 & 1:
                raise H5FormatError("big-endian floats unsupported")
            return ("f", size)
        if cls == 0:  # fixed point
            if b0 & 1:
                raise H5FormatError("big-endian ints unsupported")
            return ("i" if (b0 & 8) else "u", size)
        if cls == 3:  # fixed-length string
            return ("S", size)
        if cls == 9:  # variable-length (only vlen strings occur: backend, keras_version)
            return ("V", size)
        raise H5FormatError("unsupported datatype class %d" % cls)

    @staticmethod
    def _parse_dspace(body):
        ver, rank, flags = struct.unpack_from("<BBB", body, 0)
        if ver == 1:
            off = 8
        elif ver == 2:
            off = 4
        else:
            raise H5FormatError("dataspace v%d unsupported" % ver)
        dims = struct.unpack_from("<%dQ" % rank, body, off) if rank else ()
        return tuple(int(d) for d in dims)

    # -------------------------------------------------------------- attributes
    def attrs(self, addr):
        out = OrderedDict()
        for body in self.obj(addr).all(0x0C):
            ver, _r, nsize, tsize, ssize = struct.unpack_from("<BBHHH", body, 0)
            if ver != 1:
                raise H5FormatError("attribute v%d unsupported" % ver)
            pad = lambda n: (n + 7) & ~7
            pos = 8
            name = body[pos:pos + nsize].split(b"\x00", 1)[0].decode("utf-8")
            pos += pad(nsize)
            kind, size = self._parse_dtype(body[pos:pos + tsize])
            pos += pad(tsize)
            dims = self._parse_dspace(body[pos:pos + ssize])
            pos += pad(ssize)
            n = int(np.prod(dims)) if dims else 1
            raw = body[pos:pos + n * size]
            if kind == "V":
                vals = [self._vlen_bytes(raw[i * size:(i + 1) * size]).decode("utf-8")
                        for i in range(n)]
                out[name] = vals if dims else vals[0]
            elif kind == "S":
                vals = [raw[i * size:(i + 1) * size].split(b"\x00", 1)[0].decode("utf-8")
                        for i in range(n)]
                out[name] = vals if dims else vals[0]
            else:
                arr = np.frombuffer(raw, dtype="<%s%d" % (kind, size)).reshape(dims)
                out[name] = arr if dims else arr.reshape(()).item()
        return out

    def _vlen_bytes(self, ref):
        """Resolve one 16-byte vlen reference (length, global-heap address, index)."""
        length, gaddr, idx = struct.unpack_from("<IQI", ref, 0)
        b = self.buf
        if b[gaddr:gaddr + 4] != b"GCOL":
            raise H5FormatError("bad global heap signature @%d" % gaddr)
        csize, = struct.unpack_from("<Q", b, gaddr + 8)
        pos, end = gaddr + 16, gaddr + csize
        while pos + 16 <= end:
            oidx, _ref, _res, osize = struct.unpack_from("<HHIQ", b, pos)
            if oidx == 0:
                break
            if oidx == idx:
                return b[pos + 16: pos + 16 + min(length, osize)]
            pos += 16 + ((osize + 7) & ~7)
        raise H5FormatError("global heap object %d not found" % idx)

    # ----------------------------------------------------------------- datasets
    def dataset(self, addr) -> np.ndarray:
        o = self.obj(addr)
        dt, ds, lay = o.first(0x03), o.first(0x01), o.first(0x08)
        if dt is None or ds is None or lay is None:
            raise H5FormatError("object @%d is not a dataset" % addr)
        if o.first(0x0B) is not None:
            raise H5FormatError("filtered datasets unsupported")
        kind, size = self._parse_dtype(dt)
        dims = self._parse_dspace(ds)
        ver, cls = struct.unpack_from("<BB", lay, 0)
        if ver != 3 or cls != 1:
            raise H5FormatError("only v3 contiguous layout supported (v%d class %d)" % (ver, cls))
        daddr, dsize = struct.unpack_from("<QQ", lay, 2)
        n = int(np.prod(dims)) if dims else 1
        if daddr == UNDEF or dsize != n * size:
            raise H5FormatError("bad contiguous layout")
        arr = np.frombuffer(self.buf, dtype="<%s%d" % (kind, size), count=n, offset=daddr)
        return arr.reshape(dims).copy()

    def visit(self, addr=None, prefix=""):
        """Yield (path, address) of every dataset below ``addr``."""
        addr = self.root_addr if addr is None else addr
        for name, oaddr in self.children(addr):
            path = prefix + name
            if self.is_group(oaddr):
                yield from self.visit(oaddr, path + "/")
            else:
                yield path, oaddr


def read_keras_weights(path):
    """Read a Keras ``save_weights`` file.

    Returns ``(layer_names, weights)``: ``layer_names`` is the root attribute
    in graph order (the order ``load_weights`` consumes layers, reference
    ``whenet.py:16``); ``weights`` maps ``"<layer>/<weight_name>"`` (for
    example ``"conv2d_1/kernel:0"``) to a float32 array.
    """
    f = H5File(path)
    root_attrs = f.attrs(f.root_addr)
    wroot = f.root_addr
    if "layer_names" not in root_attrs:
        # a full ``model.save`` file (what YOLO's load_model reads first, reference yolo_v3/yolo_postprocess.py:75): the
        # layer list and the layer groups sit under "model_weights"
        top = dict(f.children(f.root_addr))
        if "model_weights" in top:
            wroot = top["model_weights"]
            root_attrs = f.attrs(wroot)
    layer_names = list(root_attrs.get("layer_names", []))
    groups = dict(f.children(wroot))
    weights = OrderedDict()
    for lname in layer_names:
        gaddr = groups[lname]
        wnames = f.attrs(gaddr).get("weight_names", [])
        if isinstance(wnames, str):
            wnames = [wnames]
        wnames = list(wnames)  # layers without weights store an empty (non-string) array
        if not wnames:
            continue
        found = {p: a for p, a in f.visit(gaddr)}
        for wn in wnames:
            # weight_names look like "conv2d_1/kernel:0"; dataset path mirrors it
            if wn not in found:
                raise H5FormatError("weight %s missing under layer %s" % (wn, lname))
            weights[wn] = f.dataset(found[wn])
    meta = {k: v for k, v in root_attrs.items() if k != "layer_names"}
    return layer_names, weights, meta
