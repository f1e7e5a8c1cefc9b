"""Video output on the GPU path: JPEG encoding of device BGR frames and a Motion-JPEG AVI writer (DESIGN.md section 8.9).

  ``encode_jpeg``   device (or host) BGR frames -> JPEG files, byte-identical to cv2.imencode(".jpg", frame,
                    [cv2.IMWRITE_JPEG_QUALITY, quality]), encoded by the library's CUDA kernels (``whenet_encode_jpeg_u8``)
  ``MJPGWriter``    writes those files as an MJPG AVI: what reference demo_video.py:46-47,60 writes through
                    cv2.VideoWriter(..., fourcc 'MJPG'), without the frames leaving the GPU uncompressed

The reference's loop becomes::

    results = pipeline.detect_and_estimate_frames(yolo, whenet, frames)
    overlay.draw_heads(whenet, frames, results)
    writer.write(video.encode_jpeg(whenet, frames))
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

import numpy as np

MAX_FRAMES_PER_CALL = 64
MAX_SIDE = 16384


def _frame_list(whenet, frames):
    """(on device?, items, (H, W) per frame) of BGR frames, or ValueError before anything runs."""
    from .whenet import _is_device
    if isinstance(frames, (list, tuple)):
        items, ndim = list(frames), 3
    else:
        items, ndim = [frames], 4
    on_device = [_is_device(f) for f in items]
    if items and any(d != on_device[0] for d in on_device):
        raise ValueError("frames mix CUDA tensors and host arrays")
    dev = bool(on_device and on_device[0])
    for f in items:
        if dev:
            if str(f.dtype) != "torch.uint8" or not f.is_contiguous():
                raise ValueError("frames must be contiguous uint8 tensors")
            if f.device.index != whenet.device:
                raise ValueError("frames are on cuda:%s, WHENet on cuda:%d" % (f.device.index, whenet.device))
        else:
            if not isinstance(f, np.ndarray):
                raise ValueError("frames must be CUDA tensors or numpy arrays, not %s" % type(f).__name__)
            if f.dtype != np.uint8 or not f.flags.c_contiguous:
                raise ValueError("frames must be C-contiguous uint8 arrays")
        if len(f.shape) != ndim or f.shape[-1] != 3:
            raise ValueError("frames must be BGR (n, H, W, 3) or a list of (H, W, 3), not %s" % (tuple(f.shape),))
        H, W = int(f.shape[-3]), int(f.shape[-2])
        if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
            raise ValueError("frame size %dx%d: each side must be in [1, %d]" % (W, H, MAX_SIDE))
    if ndim == 4:
        n = int(frames.shape[0])
        frames_hw = [(int(frames.shape[1]), int(frames.shape[2]))] * n
    else:
        frames_hw = [(int(f.shape[0]), int(f.shape[1])) for f in items]
    return dev, items, frames_hw


def encode_jpeg(whenet, frames, quality: int = 95) -> list:
    """JPEG files of BGR ``frames``, each byte-identical to ``cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY,
    quality])[1].tobytes()`` (baseline, 4:2:0, the standard Huffman tables), encoded on ``whenet``'s GPU and stream.

    ``frames``: what ``overlay.draw_heads`` takes - a contiguous (n, H, W, 3) uint8 CUDA tensor on ``whenet.device`` or a list
    of contiguous (H_i, W_i, 3) ones - or numpy arrays of the same shapes, which are uploaded.  Sides are 1..16384 and
    ``quality`` an int in 1..100; anything else raises ``ValueError`` before anything runs.  Waits for torch's current
    stream, then encodes in groups of 64 frames with one synchronisation each.  Only the compressed bytes leave the GPU.
    Returns one ``bytes`` per frame; n = 0 gives []."""
    import ctypes as C
    from ._lib import check
    from .whenet import _ptr
    if isinstance(quality, (bool, np.bool_)) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError("quality must be an int in [1, 100], not %r" % (quality,))
    dev, items, frames_hw = _frame_list(whenet, frames)
    n = len(frames_hw)
    if n == 0:
        return []
    import torch
    L = whenet._L
    out = []
    data = C.c_void_p()
    offsets = np.zeros(MAX_FRAMES_PER_CALL + 1, np.int64)
    with torch.cuda.device(whenet.device):
        if dev:
            torch.cuda.current_stream().synchronize()       # frames the caller wrote on torch's stream are complete
        for lo in range(0, n, MAX_FRAMES_PER_CALL):
            hi = min(n, lo + MAX_FRAMES_PER_CALL)
            if not isinstance(frames, (list, tuple)):
                H, W = frames_hw[0]
                check(L.whenet_encode_jpeg_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, int(dev), int(quality), C.byref(data),
                                              _ptr(offsets)))
            else:
                ptrs = (C.c_void_p * (hi - lo))(*[_ptr(f) for f in items[lo:hi]])
                hw = np.array(frames_hw[lo:hi], np.int32)
                check(L.whenet_encode_jpeg_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, int(dev), int(quality), C.byref(data),
                                                     _ptr(offsets)))
            for i in range(hi - lo):
                out.append(C.string_at(data.value + int(offsets[i]), int(offsets[i + 1] - offsets[i])))
    return out


# ----------------------------------------------------------------------------------------------------------------- AVI
SEGMENT_LIMIT = 1 << 30      # bytes of one RIFF segment; the file continues in OpenDML 'AVIX' segments past it
SUPER_INDEX_ENTRIES = 1024   # segments one file can hold (its 'indx' is written with room for this many)
_AVIIF_KEYFRAME = 0x10


def jpeg_size(jpeg: bytes):
    """(width, height) from a JPEG's SOF0 segment, or None when ``jpeg`` does not start with SOI or has no SOF0 before SOS."""
    if len(jpeg) < 4 or jpeg[0] != 0xFF or jpeg[1] != 0xD8:
        return None
    pos = 2
    while pos + 4 <= len(jpeg):
        if jpeg[pos] != 0xFF:
            return None
        marker = jpeg[pos + 1]
        if marker == 0xFF:          # fill byte
            pos += 1
            continue
        if marker == 0xDA or marker == 0xD9:
            return None
        length = int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        if marker == 0xC0:
            if pos + 9 > len(jpeg):
                return None
            return int.from_bytes(jpeg[pos + 7:pos + 9], "big"), int.from_bytes(jpeg[pos + 5:pos + 7], "big")
        pos += 2 + length
    return None


class MJPGWriter:
    """A Motion-JPEG AVI file, written on the host from JPEG files (``encode_jpeg``'s output): ``hdrl`` (``avih``, then a
    ``strl`` with ``strh`` vids/MJPG, ``strf`` BITMAPINFOHEADER MJPG, the OpenDML ``indx`` super index, and ``odml``/``dmlh``),
    a ``movi`` list of ``00dc`` chunks padded to even length, an ``ix00`` standard index per ``movi`` list, and ``idx1`` with a
    keyframe entry per frame of the first segment.  Past ``SEGMENT_LIMIT`` bytes the file continues in ``RIFF AVIX`` segments;
    frame counts, sizes and the super index are fixed up on ``close()``.

    ``frame_size`` is ``(width, height)`` as for cv2.VideoWriter; ``fps`` > 0.  ``write`` takes one JPEG or a sequence of them
    and refuses (``ValueError``, nothing written) any item that does not start with SOI or whose SOF0 size differs from
    ``frame_size``.  Use as a context manager or call ``close()``."""

    def __init__(self, path, fps, frame_size):
        fps = float(fps)
        if not (math.isfinite(fps) and fps > 0):
            raise ValueError("fps must be finite and positive, not %r" % (fps,))
        try:
            w, h = (int(v) for v in frame_size)
        except (TypeError, ValueError):
            raise ValueError("frame_size must be (width, height), not %r" % (frame_size,)) from None
        if not (1 <= w <= 65535 and 1 <= h <= 65535):
            raise ValueError("frame_size %r outside [1, 65535]" % (frame_size,))
        self.frame_size = (w, h)
        rate = Fraction(fps).limit_denominator(1 << 16)
        self._rate, self._scale = rate.numerator, rate.denominator
        self._usec = int(round(1e6 / fps))
        self._f = open(path, "wb")
        self._frames = 0              # in the whole file
        self._max_chunk = 0
        self._super = []              # (file offset of an ix00 chunk, its size, frames it indexes)
        self._seg = None
        self._write_headers()
        self._start_segment(first=True)

    # -- layout
    def _write_headers(self):
        f, (w, h) = self._f, self.frame_size
        f.write(b"RIFF\0\0\0\0AVI ")
        self._hdrl = f.tell()
        f.write(b"LIST\0\0\0\0hdrl")
        f.write(b"avih" + struct.pack("<I", 56))
        self._avih = f.tell()
        f.write(struct.pack("<14I", self._usec, 0, 0, 0x10, 0, 0, 1, 0, w, h, 0, 0, 0, 0))     # AVIF_HASINDEX
        strl = f.tell()
        f.write(b"LIST\0\0\0\0strl")
        f.write(b"strh" + struct.pack("<I", 56))
        self._strh = f.tell()
        f.write(b"vidsMJPG" + struct.pack("<IHHIIIIIIiI4H", 0, 0, 0, 0, self._scale, self._rate, 0, 0, 0, -1, 0, 0, 0, w, h))
        f.write(b"strf" + struct.pack("<I", 40))
        f.write(struct.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, b"MJPG", w * h * 3, 0, 0, 0, 0))
        f.write(b"indx" + struct.pack("<I", 24 + 16 * SUPER_INDEX_ENTRIES))
        self._indx = f.tell()
        f.write(struct.pack("<HBBI4s3I", 4, 0, 0, 0, b"00dc", 0, 0, 0) + bytes(16 * SUPER_INDEX_ENTRIES))
        self._fix_list(strl)
        odml = f.tell()
        f.write(b"LIST\0\0\0\0odml" + b"dmlh" + struct.pack("<I", 248))
        self._dmlh = f.tell()
        f.write(bytes(248))
        self._fix_list(odml)
        self._fix_list(self._hdrl)

    def _fix_list(self, start):
        """Set the size field of the chunk or list starting at ``start`` to reach the current end of the file."""
        end = self._f.tell()
        self._f.seek(start + 4)
        self._f.write(struct.pack("<I", end - start - 8))
        self._f.seek(end)

    def _start_segment(self, first):
        f = self._f
        if first:
            riff = 0
        else:
            riff = f.tell()
            f.write(b"RIFF\0\0\0\0AVIX")
        movi = f.tell()
        f.write(b"LIST\0\0\0\0movi")
        self._seg = {"riff": riff, "movi": movi, "first": first, "chunks": []}     # chunks: (data offset, size)

    def _segment_bytes_with(self, size):
        """The segment's size with one more chunk of ``size`` bytes and its index entries."""
        s = self._seg
        k = len(s["chunks"]) + 1
        index = 32 + 8 * k + (8 + 16 * k if s["first"] else 0)
        return self._f.tell() + 8 + size + (size & 1) + index - s["riff"]

    def _end_segment(self):
        f, s = self._f, self._seg
        chunks = s["chunks"]
        ix = f.tell()
        f.write(b"ix00" + struct.pack("<I", 24 + 8 * len(chunks)))
        f.write(struct.pack("<HBBI4sQI", 2, 0, 1, len(chunks), b"00dc", s["movi"], 0))
        f.write(b"".join(struct.pack("<II", off - s["movi"], size) for off, size in chunks))
        self._super.append((ix, 32 + 8 * len(chunks), len(chunks)))
        self._fix_list(s["movi"])
        if s["first"]:
            f.write(b"idx1" + struct.pack("<I", 16 * len(chunks)))
            # offsets relative to the 'movi' fourcc, pointing at each chunk's header
            f.write(b"".join(struct.pack("<4sIII", b"00dc", _AVIIF_KEYFRAME, off - 8 - (s["movi"] + 8), size) for off, size in chunks))
            self._first_frames = len(chunks)
        self._fix_list(s["riff"])
        self._seg = None

    # -- API
    def write(self, jpegs):
        """Append one JPEG file (bytes) or a sequence of them as frames.  Every item is checked before any is written."""
        if self._f is None:
            raise ValueError("write on a closed MJPGWriter")
        items = [jpegs] if isinstance(jpegs, (bytes, bytearray, memoryview)) else list(jpegs)
        for i, j in enumerate(items):
            if not isinstance(j, (bytes, bytearray, memoryview)):
                raise ValueError("item %d is %s, not bytes" % (i, type(j).__name__))
            size = jpeg_size(bytes(j[:65536]))
            if size is None:
                raise ValueError("item %d is not a JPEG file with an SOF0 segment" % i)
            if size != self.frame_size:
                raise ValueError("item %d is %dx%d, the writer's frame_size %dx%d" % ((i,) + size + self.frame_size))
        f = self._f
        for j in items:
            j = bytes(j)
            if self._seg["chunks"] and self._segment_bytes_with(len(j)) > SEGMENT_LIMIT:
                self._end_segment()
                if len(self._super) >= SUPER_INDEX_ENTRIES:
                    raise ValueError("more than %d RIFF segments" % SUPER_INDEX_ENTRIES)
                self._start_segment(first=False)
            f.write(b"00dc" + struct.pack("<I", len(j)))
            self._seg["chunks"].append((f.tell(), len(j)))
            f.write(j)
            if len(j) & 1:
                f.write(b"\0")
            self._frames += 1
            self._max_chunk = max(self._max_chunk, len(j))

    def close(self):
        """Finish the last segment, fix up the headers and close the file."""
        if self._f is None:
            return
        f = self._f
        self._end_segment()
        end = f.tell()
        f.seek(self._avih + 16)                                   # dwTotalFrames: frames of the first RIFF (OpenDML)
        f.write(struct.pack("<I", self._first_frames))
        f.seek(self._avih + 28)                                   # dwSuggestedBufferSize
        f.write(struct.pack("<I", self._max_chunk + 8))
        f.seek(self._strh + 32)                                   # dwLength
        f.write(struct.pack("<I", self._frames))
        f.seek(self._strh + 36)                                   # dwSuggestedBufferSize
        f.write(struct.pack("<I", self._max_chunk + 8))
        f.seek(self._indx + 4)                                    # nEntriesInUse, then the entries
        f.write(struct.pack("<I", len(self._super)))
        f.seek(self._indx + 24)
        f.write(b"".join(struct.pack("<QII", off, size, frames) for off, size, frames in self._super))
        f.seek(self._dmlh)                                        # dwTotalFrames of the whole file
        f.write(struct.pack("<I", self._frames))
        f.seek(end)
        f.close()
        self._f = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False
