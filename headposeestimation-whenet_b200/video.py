"""Video on the GPU path: JPEG encoding and decoding of device BGR frames, YUV frames to BGR, and Motion-JPEG AVI files
(DESIGN.md sections 8.9, 8.10, 8.11 and 8.14).

  ``encode_jpeg``   device (or host) BGR or gray frames -> JPEG files, byte-identical to cv2.imencode(".jpg", frame,
                    params) with the quality, sampling, restart, optimise and chroma-quality parameters, encoded by the
                    library's CUDA kernels (``whenet_encode_jpeg_u8``, ``whenet_encode_jpeg_ex_u8``)
  ``decode_jpeg``   JPEG files -> device BGR frames, pixel-identical to cv2.imdecode(buf, cv2.IMREAD_COLOR), decoded by the
                    library's CUDA kernels (``whenet_decode_jpeg_u8``); at 1/2, 1/4 or 1/8 scale or gray as with
                    IMREAD_REDUCED_* and IMREAD_GRAYSCALE (``whenet_decode_jpeg_ex_u8``, section 8.13)
  ``MJPGWriter``    writes those files as an MJPG AVI: what reference demo_video.py:46-47,60 writes through
                    cv2.VideoWriter(..., fourcc 'MJPG'), without the frames leaving the GPU uncompressed
  ``MJPGReader``    reads the JPEG files of an MJPG AVI (the reference's cap.read(), demo_video.py:44,51)
  ``to_bgr``        NV12, I420, YUYV or UYVY frames (video decoders, raw cameras, capture cards) -> device BGR frames,
                    bit-identical to cv2.cvtColor, converted by the library's CUDA kernel (``whenet_yuv_to_bgr_u8``)

The reference's loop becomes a transcode on the device::

    with video.MJPGReader(src) as r, video.MJPGWriter(dst, r.fps, r.frame_size) as w:
        while (frames := r.read_frames(whenet, 8)) is not None:
            results = pipeline.detect_and_estimate_frames(yolo, whenet, frames)
            overlay.draw_heads(whenet, frames, results, display="full")
            w.write(video.encode_jpeg(whenet, frames))

and a camera or decoder loop that hands out YUV frames stays on the device too::

    results = pipeline.detect_and_estimate_frames(yolo, whenet, frames, pixel_format="yuyv")
    bgr = video.to_bgr(whenet, frames, "yuyv")
    overlay.draw_heads(whenet, bgr, results, display="full")
    writer.write(video.encode_jpeg(whenet, bgr))
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

import numpy as np

MAX_FRAMES_PER_CALL = 64
MAX_SIDE = 16384


SAMPLINGS = {"420": 420, "422": 422, "444": 444}


def _frame_list(whenet, frames):
    """(on device?, items, (H, W) per frame, channels) of BGR frames or one-channel (gray) frames, or ValueError before anything
    runs."""
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
        if len(f.shape) != ndim or f.shape[-1] not in (1, 3):
            raise ValueError("frames must be BGR (n, H, W, 3) or gray (n, H, W, 1), or a list of (H, W, 3) or (H, W, 1), not %s"
                             % (tuple(f.shape),))
        H, W = int(f.shape[-3]), int(f.shape[-2])
        if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
            raise ValueError("frame size %dx%d: each side must be in [1, %d]" % (W, H, MAX_SIDE))
    channels = {int(f.shape[-1]) for f in items}
    if len(channels) > 1:
        raise ValueError("frames mix 1 and 3 channels")
    if ndim == 4:
        n = int(frames.shape[0])
        frames_hw = [(int(frames.shape[1]), int(frames.shape[2]))] * n
    else:
        frames_hw = [(int(f.shape[0]), int(f.shape[1])) for f in items]
    return dev, items, frames_hw, channels.pop() if channels else 3


def _is_int(x, lo, hi):
    return not isinstance(x, (bool, np.bool_)) and isinstance(x, (int, np.integer)) and lo <= x <= hi


def encode_jpeg(whenet, frames, quality: int = 95, *, sampling: str = "420", restart_interval: int = 0, optimize: bool = False,
                chroma_quality=None, progressive: bool = False) -> list:
    """JPEG files of BGR or gray ``frames``, each byte-identical to ``cv2.imencode(".jpg", frame, params)[1].tobytes()``
    (baseline, or progressive), encoded on ``whenet``'s GPU and stream.  ``params`` are:

      - ``[IMWRITE_JPEG_QUALITY, quality]``, or, when ``chroma_quality`` is given and differs from ``quality``,
        ``[IMWRITE_JPEG_LUMA_QUALITY, quality, IMWRITE_JPEG_CHROMA_QUALITY, chroma_quality]``;
      - then ``[IMWRITE_JPEG_SAMPLING_FACTOR, IMWRITE_JPEG_SAMPLING_FACTOR_<sampling>]``;
      - then ``[IMWRITE_JPEG_RST_INTERVAL, restart_interval]`` if it is nonzero;
      - then ``[IMWRITE_JPEG_OPTIMIZE, 1]`` if ``optimize``;
      - then ``[IMWRITE_JPEG_PROGRESSIVE, 1]`` if ``progressive``.

    The defaults give the plain ``[IMWRITE_JPEG_QUALITY, quality]`` file (4:2:0, the standard Huffman tables, no restart
    markers).  ``sampling`` is "420", "422" or "444"; ``restart_interval`` an int in 0..65535 MCUs; ``optimize`` a bool
    (optimal Huffman tables per frame); ``chroma_quality`` None or an int in 1..100.  cv2 silently codes two different
    qualities as 4:4:4, so ``chroma_quality != quality`` requires ``sampling="444"``.  ``progressive`` a bool: libjpeg's
    progressive scan script with optimal tables per scan (DESIGN.md section 8.12), usually smaller than the optimised file;
    ``optimize`` then changes nothing, as in cv2.  MJPG players expect baseline frames, so keep it off for ``MJPGWriter``.

    ``frames``: what ``overlay.draw_heads`` takes - a contiguous (n, H, W, 3) uint8 CUDA tensor on ``whenet.device`` or a list
    of contiguous (H_i, W_i, 3) ones - or numpy arrays of the same shapes, which are uploaded.  Gray frames are (n, H, W, 1)
    or (H_i, W_i, 1) and equal ``cv2.imencode(".jpg", frame[..., 0], params)``; they take the default ``sampling`` and
    ``chroma_quality``, and a call takes one channel count.  Sides are 1..16384.  Anything else raises ``ValueError`` before
    anything runs.  Waits for torch's current stream, then encodes in groups of 64 frames with one synchronisation each.
    Only the compressed bytes leave the GPU.  Returns one ``bytes`` per frame; n = 0 gives []."""
    import ctypes as C
    from ._lib import JpegOptions, check
    from .whenet import _ptr
    if not _is_int(quality, 1, 100):
        raise ValueError("quality must be an int in [1, 100], not %r" % (quality,))
    if sampling not in SAMPLINGS:
        raise ValueError("sampling must be \"420\", \"422\" or \"444\", not %r" % (sampling,))
    if not _is_int(restart_interval, 0, 65535):
        raise ValueError("restart_interval must be an int in [0, 65535] MCUs, not %r" % (restart_interval,))
    if not isinstance(optimize, (bool, np.bool_)):
        raise ValueError("optimize must be a bool, not %r" % (optimize,))
    if not isinstance(progressive, (bool, np.bool_)):
        raise ValueError("progressive must be a bool, not %r" % (progressive,))
    if chroma_quality is not None and not _is_int(chroma_quality, 1, 100):
        raise ValueError("chroma_quality must be None or an int in [1, 100], not %r" % (chroma_quality,))
    cq = quality if chroma_quality is None else int(chroma_quality)
    if cq != quality and sampling != "444":
        raise ValueError("chroma_quality %d != quality %d needs sampling=\"444\" (cv2 codes differing qualities as 4:4:4)"
                         % (cq, quality))
    dev, items, frames_hw, channels = _frame_list(whenet, frames)
    if channels == 1 and (sampling != "420" or cq != quality):
        raise ValueError("gray frames take the default sampling and chroma_quality")
    n = len(frames_hw)
    if n == 0:
        return []
    import torch
    L = whenet._L
    opts = JpegOptions(int(quality), cq, SAMPLINGS[sampling], int(restart_interval), int(bool(optimize)), int(bool(progressive)))
    default = (cq, sampling, restart_interval, bool(optimize), bool(progressive), channels) == (quality, "420", 0, False, False, 3)
    out = []
    data = C.c_void_p()
    offsets = np.zeros(MAX_FRAMES_PER_CALL + 1, np.int64)
    with torch.cuda.device(whenet.device):
        if dev:
            torch.cuda.current_stream().synchronize()       # frames the caller wrote on torch's stream are complete
        for lo in range(0, n, MAX_FRAMES_PER_CALL):
            hi = min(n, lo + MAX_FRAMES_PER_CALL)
            if not isinstance(frames, (list, tuple)) and default:
                H, W = frames_hw[0]
                check(L.whenet_encode_jpeg_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, int(dev), int(quality), C.byref(data),
                                              _ptr(offsets)))
            else:
                src = items[lo:hi] if isinstance(frames, (list, tuple)) else [frames[i] for i in range(lo, hi)]
                ptrs = (C.c_void_p * (hi - lo))(*[_ptr(f) for f in src])
                hw = np.array(frames_hw[lo:hi], np.int32)
                if default:
                    check(L.whenet_encode_jpeg_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, int(dev), int(quality),
                                                         C.byref(data), _ptr(offsets)))
                else:
                    check(L.whenet_encode_jpeg_ex_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, channels, int(dev), C.byref(opts),
                                                     C.byref(data), _ptr(offsets)))
            for i in range(hi - lo):
                out.append(C.string_at(data.value + int(offsets[i]), int(offsets[i + 1] - offsets[i])))
    return out


def to_bgr(whenet, frames, pixel_format: str):
    """YUV ``frames`` -> BGR frames on ``whenet``'s GPU, each bit-identical to ``cv2.cvtColor(frame, COLOR_YUV2BGR_<fmt>)``:
    the frames ``overlay.draw_heads`` and ``encode_jpeg`` take.  ``pixel_format`` is

      - ``"nv12"`` or ``"i420"``: YUV 4:2:0 in cv2's layout, (n, H * 3/2, W) uint8 or a list of (H_i * 3/2, W_i), sides even;
      - ``"yuyv"`` or ``"uyvy"``: packed YUV 4:2:2, (n, H, W, 2) uint8 or a list of (H_i, W_i, 2), W even, any H.

    Frames are a numpy array or a contiguous CUDA tensor on ``whenet.device``, or a list or tuple of them (all host or all
    device); image sides are 1..16384.  Returns a contiguous (n, H, W, 3) uint8 CUDA tensor, or for a list a list of
    (H_i, W_i, 3) ones; n = 0 gives an empty tensor or [].  Waits for torch's current stream, then converts in groups of 64
    frames with one synchronisation each, so the frames are ready on any stream when it returns.  Host frames are uploaded
    at their own size (2 bytes per pixel for 4:2:2, 1.5 for 4:2:0).  Anything else raises ``ValueError`` before anything runs."""
    import ctypes as C
    from ._lib import YUV_LAYOUTS, YUV422_LAYOUTS, check
    from .whenet import _is_device, _ptr
    from .yolo import _frame_list as _yuv_frame_list
    from .yolo import _image_size, _is_422, _yuv422_image_size, _yuv_image_size
    if not isinstance(pixel_format, str) or pixel_format not in {**YUV_LAYOUTS, **YUV422_LAYOUTS}:
        raise ValueError("pixel_format must be 'nv12', 'i420', 'yuyv' or 'uyvy', not %r" % (pixel_format,))
    layout = {**YUV_LAYOUTS, **YUV422_LAYOUTS}[pixel_format]
    ragged = isinstance(frames, (list, tuple))
    if ragged:
        items, dev = _yuv_frame_list(frames, whenet.device, layout)
        sizes = [_image_size(f.shape, layout) for f in items]
    else:
        dev = _is_device(frames)
        if dev:
            if str(frames.dtype) != "torch.uint8" or not frames.is_contiguous():
                raise ValueError("device frames must be a contiguous uint8 CUDA tensor")
            if frames.device.index != whenet.device:
                raise ValueError("frames are on cuda:%s, WHENet on cuda:%d" % (frames.device.index, whenet.device))
        else:
            frames = np.asarray(frames)
            if frames.dtype != np.uint8:
                raise ValueError("frames must be uint8, not %s" % frames.dtype)
            frames = np.ascontiguousarray(frames)
        if _is_422(layout):
            if len(frames.shape) != 4:
                raise ValueError("frames must be (n, H, W, 2) uint8 for a 4:2:2 pixel format, not %s" % (tuple(frames.shape),))
            H, W = _yuv422_image_size(frames.shape[1:], "a frame")
        else:
            if len(frames.shape) != 3:
                raise ValueError("frames must be (n, H * 3/2, W) uint8 for a 4:2:0 pixel format, not %s" % (tuple(frames.shape),))
            H, W = _yuv_image_size(frames.shape[1:], "a frame")
        sizes = [(H, W)] * int(frames.shape[0])
    for H, W in sizes:
        if H > MAX_SIDE or W > MAX_SIDE:
            raise ValueError("frame size %dx%d: each side must be in [1, %d]" % (W, H, MAX_SIDE))
    import torch
    n = len(sizes)
    cuda = "cuda:%d" % whenet.device
    if ragged:
        out = [torch.empty((h, w, 3), dtype=torch.uint8, device=cuda) for h, w in sizes]
    else:
        out = torch.empty((n, H, W, 3), dtype=torch.uint8, device=cuda)
    if n == 0:
        return out
    L = whenet._L
    with torch.cuda.device(whenet.device):
        torch.cuda.current_stream().synchronize()       # the frames and the outputs' memory are done with on torch's stream
        for lo in range(0, n, MAX_FRAMES_PER_CALL):
            hi = min(n, lo + MAX_FRAMES_PER_CALL)
            if ragged:
                ptrs = (C.c_void_p * (hi - lo))(*[_ptr(f).value for f in items[lo:hi]])
                dst = (C.c_void_p * (hi - lo))(*[o.data_ptr() for o in out[lo:hi]])
                hw = np.array(sizes[lo:hi], np.int32).reshape(-1)
                check(L.whenet_yuv_to_bgr_ragged_u8(whenet._h, C.addressof(ptrs), _ptr(hw), hi - lo, int(dev), layout, C.addressof(dst)))
            else:
                check(L.whenet_yuv_to_bgr_u8(whenet._h, _ptr(frames[lo:hi]), hi - lo, H, W, int(dev), layout, _ptr(out[lo:hi])))
            whenet.synchronize()
    return out


def _jpeg_files(files):
    """``files`` as a list of bytes, or ValueError naming the first item that is not bytes-like."""
    if isinstance(files, (bytes, bytearray, memoryview)) or not isinstance(files, (list, tuple)):
        raise ValueError("files must be a list or tuple of bytes-like JPEG files, not %s" % type(files).__name__)
    out = []
    for i, f in enumerate(files):
        if isinstance(f, bytes):
            out.append(f)
        elif isinstance(f, (bytearray, memoryview)) or (isinstance(f, np.ndarray) and f.dtype == np.uint8 and f.ndim == 1):
            out.append(bytes(f))
        else:
            raise ValueError("file %d is %s, not bytes" % (i, type(f).__name__))
    return out


def _decode_mode(reduce, gray):
    """(scale_denom, channels) of decode_jpeg's ``reduce`` and ``gray``, or ValueError."""
    if isinstance(reduce, bool) or not isinstance(reduce, int) or reduce not in (1, 2, 4, 8):
        raise ValueError("reduce must be the int 1, 2, 4 or 8, not %r" % (reduce,))
    if not isinstance(gray, bool):
        raise ValueError("gray must be a bool, not %r" % (gray,))
    return reduce, 1 if gray else 3


def jpeg_info(data: bytes, *, reduce=1):
    """(H, W) of the frame ``decode_jpeg`` makes of ``data`` (after its EXIF orientation) at 1 / ``reduce`` scale:
    (ceil(H / reduce), ceil(W / reduce)) as cv2.imdecode gives with IMREAD_REDUCED_*_``reduce``.  Parsed on the host without
    a GPU; ValueError with the reason for a file outside the supported subset (DESIGN.md sections 8.10 and 8.13)."""
    import ctypes as C
    from ._lib import load
    d, _ = _decode_mode(reduce, False)
    hw = (C.c_int32 * 2)()
    msg = C.create_string_buffer(256)
    if load().whenet_jpeg_info_ex(data, len(data), d, 3, hw, msg, len(msg)) != 0:
        raise ValueError(msg.value.decode("utf-8", "replace"))
    return int(hw[0]), int(hw[1])


def _decode_into(whenet, files, outs, first_index=0, reduce=1, channels=3):
    """Decode ``files`` (bytes) into the contiguous (H, W, channels) uint8 CUDA tensors ``outs`` in groups of 64."""
    import ctypes as C
    import torch
    from ._lib import WhenetError, check
    L = whenet._L
    with torch.cuda.device(whenet.device):
        torch.cuda.current_stream().synchronize()       # the outputs' memory is no longer in use on torch's stream
        for lo in range(0, len(files), MAX_FRAMES_PER_CALL):
            hi = min(len(files), lo + MAX_FRAMES_PER_CALL)
            k = hi - lo
            bufs = [C.create_string_buffer(f, len(f)) for f in files[lo:hi]]
            ptrs = (C.c_void_p * k)(*[C.addressof(b) for b in bufs])
            sizes = (C.c_int64 * k)(*[len(f) for f in files[lo:hi]])
            dst = (C.c_void_p * k)(*[o.data_ptr() for o in outs[lo:hi]])
            status = (C.c_int32 * k)()
            try:
                if reduce == 1 and channels == 3:
                    check(L.whenet_decode_jpeg_u8(whenet._h, ptrs, sizes, k, dst, status))
                else:
                    check(L.whenet_decode_jpeg_ex_u8(whenet._h, ptrs, sizes, k, reduce, channels, dst, status))
            except WhenetError as e:
                bad = next((i for i in range(k) if status[i]), None)
                msg = str(e).split(": ", 1)[-1]
                if bad is not None:
                    msg = "file %d: %s" % (first_index + lo + bad, msg.split(": ", 1)[-1])
                raise ValueError(msg) from None


def decode_jpeg(whenet, files, *, reduce=1, gray=False) -> list:
    """Decode JPEG ``files`` (a list of bytes-like objects) on ``whenet``'s GPU and stream into BGR frames, each equal to
    ``cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)``: baseline or extended-sequential Huffman, 1 or 3 components,
    4:4:4, 4:2:2 or 4:2:0, restart intervals, files without DHT, EXIF orientation applied, sides 1..16384.

    ``reduce`` (1, 2, 4 or 8) decodes at that fraction of the size inside the IDCT, as ``cv2.IMREAD_REDUCED_COLOR_<reduce>``
    does: (ceil(H / reduce), ceil(W / reduce), 3) frames.  ``gray=True`` gives the luma plane alone as (H', W', 1) frames, as
    ``cv2.IMREAD_GRAYSCALE`` (``cv2.IMREAD_REDUCED_GRAYSCALE_<reduce>`` with ``reduce``) does; ``encode_jpeg`` takes them as
    gray frames.  DESIGN.md section 8.13.

    Returns a list of contiguous (H_i, W_i, C) uint8 CUDA tensors on ``whenet.device``, decoded in groups of 64 files with one
    synchronisation each; n = 0 gives [].  Bad arguments, a file outside that subset (checked before any device work) or
    corrupt entropy-coded data raise ``ValueError`` naming the file index and the reason."""
    import torch
    d, channels = _decode_mode(reduce, gray)
    files = _jpeg_files(files)
    if not files:
        return []
    shapes = []
    for i, f in enumerate(files):
        try:
            shapes.append(jpeg_info(f, reduce=d))
        except ValueError as e:
            raise ValueError("file %d: %s" % (i, e)) from None
    outs = [torch.empty((h, w, channels), dtype=torch.uint8, device="cuda:%d" % whenet.device) for h, w in shapes]
    _decode_into(whenet, files, outs, reduce=d, channels=channels)
    return outs


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

    MJPG players expect baseline frames, which is what cv2.VideoWriter writes: encode them with ``progressive=False``.

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


class MJPGReader:
    """The JPEG files of a Motion-JPEG AVI, read on the host: the counterpart of ``MJPGWriter`` and what the reference reads
    through cv2.VideoCapture.  The first video stream whose handler or compression is MJPG (any case) is read; ``fps`` comes
    from its ``strh`` rate / scale and ``frame_size`` = (width, height) from its ``strf``.

    Frames are found through the OpenDML super index (``indx`` -> ``ix##`` standard indexes, across ``AVIX`` segments), else
    ``idx1`` (offsets relative to ``movi`` or absolute, told apart by the first entry), else by walking the ``movi`` lists.
    Chunks of other streams and JUNK are skipped, and a last chunk cut short by the end of the file is not returned.

    ``read(n)`` returns up to n JPEG files as bytes ([] at the end); ``read_frames(whenet, n)`` decodes up to n of them into one
    (k, H, W, 3) uint8 CUDA tensor (``None`` at the end).  ``len()`` is the number of frames.  Use as a context manager or call
    ``close()``."""

    def __init__(self, path):
        self._f = open(path, "rb")
        try:
            self._f.seek(0, 2)
            self._size = self._f.tell()
            self._parse()
        except Exception:
            self._f.close()
            raise
        self._next = 0

    # -- RIFF
    def _read_at(self, off, n):
        self._f.seek(off)
        return self._f.read(n)

    def _chunks(self, start, end):
        """(fourcc, data offset, data size, list type or None) of the chunks in [start, end)."""
        pos = start
        while pos + 8 <= min(end, self._size):
            hdr = self._read_at(pos, 12)
            fcc, size = hdr[:4], struct.unpack("<I", hdr[4:8])[0]
            if fcc in (b"LIST", b"RIFF"):
                yield fcc, pos + 12, size - 4, hdr[8:12]
            else:
                yield fcc, pos + 8, size, None
            pos += 8 + size + (size & 1)

    def _parse(self):
        head = self._read_at(0, 12)
        if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"AVI ":
            raise ValueError("not a RIFF AVI file")
        self._stream = None
        indx = None
        movis, idx1 = [], None
        riffs = [(12, 8 + struct.unpack("<I", head[4:8])[0])]
        pos = riffs[0][1] + (riffs[0][1] & 1)
        while pos + 12 <= self._size:               # AVIX segments
            h = self._read_at(pos, 12)
            size = struct.unpack("<I", h[4:8])[0]
            if h[:4] == b"RIFF" and h[8:12] == b"AVIX":
                riffs.append((pos + 12, pos + 8 + size))
            pos += 8 + size + (size & 1)
        for r, (start, end) in enumerate(riffs):
            for fcc, off, size, kind in self._chunks(start, end):
                if kind == b"hdrl" and r == 0:
                    indx = self._parse_hdrl(off, off + size)
                elif kind == b"movi":
                    movis.append((off - 4, off + size))     # the 'movi' fourcc, the list's end
                elif fcc == b"idx1" and r == 0:
                    idx1 = (off, size)
        if self._stream is None:
            raise ValueError("no MJPG video stream")
        ids = (b"%02ddc" % self._stream, b"%02ddb" % self._stream)
        frames = None
        if indx:
            frames = self._from_indx(indx, ids)
        if not frames and idx1 and movis:
            frames = self._from_idx1(idx1, movis[0][0], ids)
        if not frames:
            frames = []
            for start, end in movis:
                self._walk_movi(start + 4, end, ids, frames)
        self._frames = [(o, n) for o, n in frames if o + n <= self._size]

    def _parse_hdrl(self, start, end):
        n = 0
        for fcc, off, size, kind in self._chunks(start, end):
            if kind != b"strl":
                continue
            strh = strf = indx = None
            for f2, o2, s2, _ in self._chunks(off, off + size):
                if f2 == b"strh":
                    strh = self._read_at(o2, s2)
                elif f2 == b"strf":
                    strf = self._read_at(o2, s2)
                elif f2 == b"indx":
                    indx = (o2, s2)
            if self._stream is None and strh and len(strh) >= 28 and strh[:4] == b"vids":
                handler = strh[4:8].upper()
                comp = strf[16:20].upper() if strf and len(strf) >= 20 else b""
                if handler == b"MJPG" or comp == b"MJPG":
                    scale, rate = struct.unpack("<II", strh[20:28])
                    self.fps = rate / scale if scale else 0.0
                    if strf and len(strf) >= 12:
                        w, h = struct.unpack("<ii", strf[4:12])
                    else:
                        w, h = struct.unpack("<HH", strh[52:56]) if len(strh) >= 56 else (0, 0)
                    self.frame_size = (int(w), abs(int(h)))
                    self._stream = n
                    return indx
            n += 1
        return None

    def _from_indx(self, indx, ids):
        off, size = indx
        d = self._read_at(off, size)
        if len(d) < 24:
            return None
        longs, sub, itype, entries = struct.unpack("<HBBI", d[:8])
        if itype != 0 or longs != 4:                # AVI_INDEX_OF_INDEXES
            return None
        frames = []
        for e in range(entries):
            if 24 + 16 * e + 16 > len(d):
                break
            qoff, qsize, _ = struct.unpack("<QII", d[24 + 16 * e:40 + 16 * e])
            ix = self._read_at(qoff, qsize)
            if len(ix) < 32:
                break
            longs, sub, itype, n, cid, base = struct.unpack("<HBBI4sQ", ix[8:28])
            if itype != 1 or longs != 2 or cid not in ids:
                return None
            for k in range(n):
                if 32 + 8 * k + 8 > len(ix):
                    break
                o, s = struct.unpack("<II", ix[32 + 8 * k:40 + 8 * k])
                frames.append((base + o, s & 0x7FFFFFFF))
        return frames

    def _from_idx1(self, idx1, movi, ids):
        off, size = idx1
        d = self._read_at(off, size)
        entries = [struct.unpack("<4sIII", d[i:i + 16]) for i in range(0, len(d) - 15, 16)]
        if not entries:
            return None
        first = entries[0]
        base = movi if self._read_at(movi + first[2], 4) == first[0] else 0
        return [(base + o + 8, s) for cid, _, o, s in entries if cid in ids]

    def _walk_movi(self, start, end, ids, frames):
        for fcc, off, size, kind in self._chunks(start, end):
            if kind is not None:
                self._walk_movi(off, off + size, ids, frames)       # LIST rec
            elif fcc in ids:
                frames.append((off, size))

    # -- API
    def __len__(self):
        return len(self._frames)

    def read(self, n=1):
        """Up to ``n`` more JPEG files as bytes; [] at the end."""
        if self._f is None:
            raise ValueError("read on a closed MJPGReader")
        out = []
        for off, size in self._frames[self._next:self._next + max(0, int(n))]:
            out.append(self._read_at(off, size))
        self._next += len(out)
        return out

    def read_frames(self, whenet, n=1, *, reduce=1, gray=False):
        """Up to ``n`` more frames decoded on ``whenet``'s GPU into one (k, H, W, 3) uint8 CUDA tensor, or None at the end.  A
        frame whose size differs from ``frame_size`` raises ValueError.  ``reduce`` and ``gray`` are decode_jpeg's
        (cv2.IMREAD_REDUCED_COLOR_<reduce>, cv2.IMREAD_GRAYSCALE, cv2.IMREAD_REDUCED_GRAYSCALE_<reduce>): the tensor is then
        (k, ceil(H / reduce), ceil(W / reduce), 3 or 1), and each frame is checked against the reduced ``frame_size``."""
        import torch
        d, channels = _decode_mode(reduce, gray)
        first = self._next
        files = self.read(n)
        if not files:
            return None
        w, h = self.frame_size
        w, h = -(-w // d), -(-h // d)
        for i, f in enumerate(files):
            try:
                hw = jpeg_info(f, reduce=d)
            except ValueError as e:
                raise ValueError("frame %d: %s" % (first + i, e)) from None
            if hw != (h, w):
                raise ValueError("frame %d is %dx%d, the stream's frame_size %dx%d" % (first + i, hw[1], hw[0], w, h))
        out = torch.empty((len(files), h, w, channels), dtype=torch.uint8, device="cuda:%d" % whenet.device)
        _decode_into(whenet, files, list(out), first_index=first, reduce=d, channels=channels)
        return out

    def close(self):
        if self._f is not None:
            self._f.close()
            self._f = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False
