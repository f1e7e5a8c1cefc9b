"""Host-side mirror of the reference's ``yolo_v3/yolo_postprocess.py`` ``YOLO`` class: same constructor keywords, same
``detect`` result - letterbox, Darknet-53, decode and NMS run in ``libwhenet_b200.so`` (hand-written sm_90a CUDA).

``YOLO(**vars(args))`` from reference ``demo_video.py:41`` works: unknown keywords are kept as attributes, as the
reference's ``self.__dict__.update(kwargs)`` does.  ``model_path=None`` means seeded random weights (``yolo_arch.random_weights``),
flagged by ``self.random_weights``; the reference's trained ``head_detect.h5`` is not shipped.

As in the reference (yolo_postprocess.py:71-79), the anchors pick the network: 9 anchors mean YOLOv3 (``yolo_body``), 6 mean
tiny YOLOv3 (``tiny_yolo_body``, ``self.tiny``).

``model_image_size`` is (h, w), multiples of 32 up to 608 per side (``whenet_det_create_ex``) or, above that, up to 4096
(``whenet_det_create_large``, DESIGN.md 8.6): a 1080p camera letterboxes to 1088 x 1920 with no downscale, so small heads
keep their pixels.  The reference's image-sized mode, ``model_image_size=(None, None)``, letterboxes each W x H image to
(H - H % 32, W - W % 32); it is refused here, and for a camera of known size the explicit size gives the same result:
(1056, 1920) for 1920 x 1080 frames, (704, 1280) for 1280 x 720, (2144, 3840) for 3840 x 2160.

``max_boxes`` (keyword only, 1..256, default 20 as in the reference's ``yolo_eval``) caps the boxes kept per class in every
``detect`` / ``detect_frames`` call and so in ``pipeline.detect_and_estimate(_frames)``: crowds at high resolution hold more
than 20 heads.

``precision`` (keyword only) is ``"bf16"`` (the default: bf16 activations, fp32 accumulation) or ``"fp32"``, the parity mode:
fp32 activations and every conv as three bf16 MMAs on the hi / lo split of activations and weights (DESIGN.md 8.3).  The
reference runs its detector in float32.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Tuple

import numpy as np

from . import _lib, h5lite, yolo_arch
from ._lib import check
from .whenet import _is_device, _ptr

_PRECISIONS = {"bf16": _lib.PRECISIONS["bf16"], "fp32": _lib.PRECISIONS["fp32"]}


def _tensor_list(layers):
    """Mapped layers -> the ABI's tensor list (kernel, then BN gamma/beta/mean/var or bias, in table order)."""
    arrs, names = [], []
    for d in layers:
        keys = ["kernel"] + (["gamma", "beta", "moving_mean", "moving_variance"] if "gamma" in d else ["bias"])
        for k in keys:
            arrs.append(np.ascontiguousarray(d[k], np.float32))
            names.append(("%s/%s:0" % (d["name"], k)).encode())
    t = (_lib.Tensor * len(arrs))()
    for i, (a, nm) in enumerate(zip(arrs, names)):
        t[i].name = nm
        t[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
        t[i].ndim = a.ndim
        for j in range(a.ndim):
            t[i].dims[j] = a.shape[j]
    return t, (arrs, names)


def _pixel_layout(pixel_format) -> int:
    """``pixel_format`` -> the C entries' yuv_layout: 0 for "bgr" (packed 8-bit BGR, the *_u8 entries), WHENET_YUV_NV12 for
    "nv12", WHENET_YUV_I420 for "i420" (the *_yuv_u8 entries), WHENET_YUV_YUYV for "yuyv", WHENET_YUV_UYVY for "uyvy" (the
    *_yuv422_u8 entries).  Raises ValueError otherwise."""
    if isinstance(pixel_format, str):
        if pixel_format == "bgr":
            return 0
        if pixel_format in _lib.YUV_LAYOUTS:
            return _lib.YUV_LAYOUTS[pixel_format]
        if pixel_format in _lib.YUV422_LAYOUTS:
            return _lib.YUV422_LAYOUTS[pixel_format]
    raise ValueError("pixel_format must be 'bgr', 'nv12', 'i420', 'yuyv' or 'uyvy', not %r" % (pixel_format,))


def _is_422(layout: int) -> bool:
    """Whether a yuv_layout is packed 4:2:2 (YUYV or UYVY)."""
    return layout in _lib.YUV422_LAYOUTS.values()


def _entry_name(stem: str, layout: int) -> str:
    """The C entry for frames of ``layout``: ``stem``_u8 (BGR), ``stem``_yuv_u8 (4:2:0) or ``stem``_yuv422_u8 (4:2:2)."""
    return stem + ("_yuv422_u8" if _is_422(layout) else "_yuv_u8" if layout else "_u8")


def _yuv422_image_size(shape, what: str) -> Tuple[int, int]:
    """The shape of a packed YUV 4:2:2 frame, (H, W, 2) -> its image size (H, W); ValueError naming ``what`` unless the shape
    is 3-D with two channels, at least one row and an even width of at least 2."""
    if len(shape) != 3 or int(shape[2]) != 2:
        raise ValueError("%s must be (H, W, 2) uint8 for a 4:2:2 pixel format, not %s" % (what, tuple(shape)))
    h, w = int(shape[0]), int(shape[1])
    if h < 1:
        raise ValueError("%s has no rows" % what)
    if w < 2 or w % 2:
        raise ValueError("%s is %d pixels wide: a 4:2:2 frame has an even width" % (what, w))
    return h, w


def _yuv_image_size(shape, what: str) -> Tuple[int, int]:
    """The shape of a YUV 4:2:0 frame in cv2's layout, (H * 3/2, W) -> its image size (H, W); ValueError naming ``what``
    unless the shape is 2-D with a row count divisible by 3 and an even width (so H and W are even and at least 2)."""
    if len(shape) != 2:
        raise ValueError("%s must be (H * 3/2, W) uint8 for a 4:2:0 pixel format, not %s" % (what, tuple(shape)))
    rows, w = (int(v) for v in shape)
    if rows < 3 or rows % 3:
        raise ValueError("%s has %d rows: a 4:2:0 frame has H * 3/2 rows, a positive multiple of 3" % (what, rows))
    if w < 2 or w % 2:
        raise ValueError("%s is %d pixels wide: a 4:2:0 frame has an even width" % (what, w))
    return rows // 3 * 2, w


def _image_size(shape, layout: int) -> Tuple[int, int]:
    """(H, W) of a checked frame of the given layout: (H, W, 3) BGR, (H * 3/2, W) YUV 4:2:0 or (H, W, 2) YUV 4:2:2."""
    return (int(shape[0]), int(shape[1])) if not layout or _is_422(layout) else (int(shape[0]) // 3 * 2, int(shape[1]))


def _frame_list(frames, device: int, layout: int = 0):
    """A list or tuple of (H_i, W_i, 3) uint8 frames (4:2:0 layouts: (H_i * 3/2, W_i); 4:2:2: (H_i, W_i, 2)), all numpy arrays or all contiguous CUDA
    tensors on ``device`` -> (list of C-contiguous frames, whether they are on the device).  Raises ValueError otherwise."""
    frames = list(frames)
    dev = [_is_device(f) for f in frames]
    if any(dev) and not all(dev):
        raise ValueError("a frame list must be all host (numpy) or all device (CUDA tensor) frames, not a mix")
    out = []
    for i, f in enumerate(frames):
        if dev[i]:
            if str(f.dtype) != "torch.uint8" or not f.is_contiguous():
                raise ValueError("frame %d: device frames must be contiguous uint8 CUDA tensors" % i)
            if f.device.index != device:
                raise ValueError("frame %d is on cuda:%s, not on cuda:%d" % (i, f.device.index, device))
        else:
            f = np.asarray(f)
            if f.dtype != np.uint8:
                raise ValueError("frame %d: frames must be uint8, not %s" % (i, f.dtype))
            f = np.ascontiguousarray(f)
        if _is_422(layout):
            _yuv422_image_size(f.shape, "frame %d" % i)
        elif layout:
            _yuv_image_size(f.shape, "frame %d" % i)
        elif len(f.shape) != 3 or f.shape[2] != 3 or f.shape[0] < 1 or f.shape[1] < 1:
            raise ValueError("frame %d: frames must be (H, W, 3) uint8, not %s" % (i, tuple(f.shape)))
        out.append(f)
    return out, bool(dev) and dev[0]


def _frame_table(frames, layout: int = 0):
    """Frames of a list -> the ragged entries' arguments: a ctypes array of their addresses and their image sizes (H, W) as
    int32 pairs (keep both alive over the call)."""
    ptrs = (C.c_void_p * len(frames))(*(_ptr(f).value for f in frames))
    hw = np.array([_image_size(f.shape, layout) for f in frames], np.int32).reshape(-1)
    return ptrs, hw


class YOLO:
    max_boxes = 20          # per class and frame (the reference's yolo_eval default); the constructor's keyword sets it
    def __init__(self, model_path=None, anchors_path=None, classes_path=None, score=0.3, iou=0.45, model_image_size=(416, 416),
                 gpu_num=1, *, device: Optional[int] = None, max_frames: int = 8, seed: int = 0, precision: str = "bf16", max_boxes: int = 20,
                 **kwargs):
        if precision not in _PRECISIONS:
            raise ValueError("precision must be one of %s, not %r" % (sorted(_PRECISIONS), precision))
        if isinstance(max_boxes, bool) or not isinstance(max_boxes, (int, np.integer)) or not 1 <= max_boxes <= 256:
            raise ValueError("max_boxes must be an int in [1, 256], not %r" % (max_boxes,))
        self.__dict__.update(kwargs)
        self.precision = precision
        self.max_boxes = int(max_boxes)
        self.model_path, self.anchors_path, self.classes_path = model_path, anchors_path, classes_path
        self.score, self.iou, self.gpu_num = float(score), float(iou), gpu_num
        size = tuple(model_image_size)
        if len(size) != 2 or None in size:
            raise ValueError("model_image_size (None, None) (image-sized input) is not supported; use multiples of 32")
        yolo_arch.check_size(*size, max_size=yolo_arch.LARGE_MAX_SIZE)
        self.model_image_size = size
        self.anchors = yolo_arch.read_anchors(os.path.expanduser(anchors_path)) if anchors_path else yolo_arch.DEFAULT_ANCHORS.copy()
        if self.anchors.shape not in ((9, 2), (6, 2)):
            raise ValueError("YOLOv3 needs 9 anchors and tiny YOLOv3 6, %s has %d" % (anchors_path, len(self.anchors)))
        self.tiny = len(self.anchors) == 6
        self.class_names = yolo_arch.read_classes(os.path.expanduser(classes_path)) if classes_path else list(yolo_arch.DEFAULT_CLASSES)
        self.random_weights = model_path is None
        if model_path is None:
            names, w = yolo_arch.random_weights(seed, len(self.class_names), tiny=self.tiny)
        else:
            mp = os.path.expanduser(os.fspath(model_path))
            if not mp.endswith(".h5"):
                raise ValueError("Keras model or weights must be a .h5 file.")     # yolo_postprocess.py:68
            names, w, _meta = h5lite.read_keras_weights(mp)
        layers, num_classes = yolo_arch.map_weights(names, w, tiny=self.tiny)
        if num_classes != len(self.class_names):
            raise ValueError("Mismatch between model and given anchor and class sizes: the model has %d classes, %d class names"
                             % (num_classes, len(self.class_names)))
        self.num_classes = num_classes
        self.device = int(os.environ.get("LOCAL_RANK", "0")) if device is None else int(device)
        self.max_frames = int(max_frames)
        self._L = _lib.load()
        self._h = C.c_void_p()
        create = self._L.whenet_det_create_ex if max(size) <= yolo_arch.MAX_SIZE else self._L.whenet_det_create_large
        check(create(C.byref(self._h), self.device, size[0], size[1], self.max_frames, _PRECISIONS[precision]))
        try:
            self.load_layers(layers)
        except Exception:
            self.close()            # a detector that could not take its weights frees its device memory at once
            raise

    def load_layers(self, layers, anchors=None):
        """Mapped layers (``yolo_arch.map_weights``) -> device.  ``anchors`` ((w, h) pairs, 9 or 6) replace the detector's
        and with their count the network: pass them to load the layers of the other network into a live detector."""
        a = self.anchors if anchors is None else np.asarray(anchors, np.float64).reshape(-1, 2)
        t, keep = _tensor_list(layers)
        a32 = np.ascontiguousarray(a, np.float32)
        check(self._L.whenet_det_load_weights(self._h, t, len(t), _ptr(a32), len(a32)))
        del keep
        self.anchors, self.tiny = a, len(a) == 6
        self.num_classes = self._L.whenet_det_num_classes(self._h)

    # ------------------------------------------------------------------ reference surface
    def detect(self, image) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """reference yolo_postprocess.py:180-205: PIL RGB image or (H, W, 3) RGB uint8 array -> (boxes (k,4) float32
        (y_min, x_min, y_max, x_max), scores (k,) float32, classes (k,) int32)."""
        a = np.asarray(image.convert("RGB") if hasattr(image, "convert") else image)
        return self._detect(a[None], swap_rb=False)[0]

    def detect_frames(self, frames_bgr, *, pixel_format: str = "bgr") -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """A batch of BGR frames of one size (n, H, W, 3) uint8, numpy or a CUDA tensor -> one detect() tuple per frame.

        ``frames_bgr`` may also be a list or tuple of (H_i, W_i, 3) uint8 BGR frames of any sizes, all numpy arrays or all
        contiguous CUDA tensors on the detector's device.  Frames of one size are stacked and run as the batch above; frames of
        several sizes run ``max_frames`` at a time through ``whenet_det_detect_ragged_u8``, each letterboxed on its own, and
        each frame's tuple is what ``detect_frames`` gives that frame alone.

        ``pixel_format="nv12"`` or ``"i420"`` takes YUV 4:2:0 video frames in cv2's layout instead: (n, H * 3/2, W) uint8, or a
        list or tuple of (H_i * 3/2, W_i) frames, H and W even.  The letterbox converts each pixel as it reads it, and the
        result is the bits ``detect_frames`` gives on ``cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12 / _I420)``.

        ``pixel_format="yuyv"`` or ``"uyvy"`` takes packed YUV 4:2:2 camera frames: (n, H, W, 2) uint8, or a list or tuple of
        (H_i, W_i, 2) frames, W even, any H.  The result is the bits ``detect_frames`` gives on
        ``cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_YUYV / _UYVY)``."""
        layout = _pixel_layout(pixel_format)
        if not isinstance(frames_bgr, (list, tuple)):
            return self._detect(frames_bgr, swap_rb=True, layout=layout)
        frames, dev = _frame_list(frames_bgr, self.device, layout)
        if not frames:
            return []
        if len({tuple(f.shape) for f in frames}) == 1:
            if dev:
                import torch
                with torch.cuda.device(self.device):
                    stacked = torch.stack(frames)
                    torch.cuda.current_stream().synchronize()   # the detector copies it on its own stream
                return self._detect(stacked, swap_rb=True, layout=layout)
            return self._detect(np.stack(frames), swap_rb=True, layout=layout)
        out = []
        for off in range(0, len(frames), self.max_frames):
            out += self._detect_ragged(frames[off:off + self.max_frames], dev, layout=layout)
        return out

    def _detect_ragged(self, frames, dev: bool, max_boxes: Optional[int] = None, layout: int = 0):
        max_boxes = self.max_boxes if max_boxes is None else max_boxes
        nb = len(frames)
        ptrs, hw = _frame_table(frames, layout)
        slots = self.num_classes * max_boxes
        boxes = np.empty((nb, slots, 4), np.float32)
        scores = np.empty((nb, slots), np.float32)
        classes = np.empty((nb, slots), np.int32)
        counts = np.empty((nb,), np.int32)
        fn = getattr(self._L, _entry_name("whenet_det_detect_ragged", layout))
        check(fn(self._h, C.addressof(ptrs), _ptr(hw), nb, int(dev), layout or 1, self.score, self.iou, max_boxes,
                 _ptr(boxes), _ptr(scores), _ptr(classes), _ptr(counts)))
        return [(boxes[i, :counts[i]].copy(), scores[i, :counts[i]].copy(), classes[i, :counts[i]].copy()) for i in range(nb)]

    def _detect(self, frames, swap_rb: bool, max_boxes: Optional[int] = None, layout: int = 0):
        max_boxes = self.max_boxes if max_boxes is None else max_boxes
        dev = _is_device(frames)
        if not dev:
            frames = np.ascontiguousarray(frames, dtype=np.uint8)
        elif not frames.is_contiguous() or str(frames.dtype) != "torch.uint8":
            raise ValueError("device frames must be a contiguous uint8 CUDA tensor")
        if _is_422(layout):
            if len(frames.shape) != 4:
                raise ValueError("frames must be (n, H, W, 2) uint8 for a 4:2:2 pixel format, not %s" % (tuple(frames.shape),))
            H, W = _yuv422_image_size(frames.shape[1:], "a frame")
            n = int(frames.shape[0])
            entry, code = "whenet_det_detect_yuv422_u8", layout
        elif layout:
            if len(frames.shape) != 3:
                raise ValueError("frames must be (n, H * 3/2, W) uint8 for a 4:2:0 pixel format, not %s" % (tuple(frames.shape),))
            H, W = _yuv_image_size(frames.shape[1:], "a frame")
            n = int(frames.shape[0])
            entry, code = "whenet_det_detect_yuv_u8", layout
        elif len(frames.shape) != 4 or frames.shape[3] != 3:
            raise ValueError("frames must be (n, H, W, 3) uint8")
        else:
            n, H, W = (int(v) for v in frames.shape[:3])
            entry, code = "whenet_det_detect_u8", int(swap_rb)
        out = []
        for off in range(0, n, self.max_frames):
            nb = min(self.max_frames, n - off)
            slots = self.num_classes * max_boxes
            boxes = np.empty((nb, slots, 4), np.float32)
            scores = np.empty((nb, slots), np.float32)
            classes = np.empty((nb, slots), np.int32)
            counts = np.empty((nb,), np.int32)
            check(getattr(self._L, entry)(self._h, _ptr(frames[off:off + nb]), nb, H, W, int(dev), code, self.score, self.iou, max_boxes,
                                          _ptr(boxes), _ptr(scores), _ptr(classes), _ptr(counts)))
            for i in range(nb):
                k = int(counts[i])
                out.append((boxes[i, :k].copy(), scores[i, :k].copy(), classes[i, :k].copy()))
        return out

    # ------------------------------------------------------------------ test hooks
    def tap(self, layer: int) -> np.ndarray:
        """float32 output of conv ``layer`` (0..74, tiny: 0..12) of the last call, (-1) its letterboxed canvas, or (100 + i)
        the max-pooled input of tiny conv i, flat."""
        n = C.c_size_t(0)
        check(self._L.whenet_det_debug_tap(self._h, int(layer), None, 0, C.byref(n)))
        out = np.empty((n.value,), np.float32)
        check(self._L.whenet_det_debug_tap(self._h, int(layer), _ptr(out), n.value, C.byref(n)))
        return out

    def debug_conv(self, x, w, bias, k: int, stride: int, leaky: bool = True, resid=None, up=None):
        """One conv through the implicit-GEMM kernel (see whenet_det_debug_conv).  x (n,H,W,C), up (n,H/2,W/2,Cu) or None."""
        x = np.ascontiguousarray(x, np.float32)
        w = np.ascontiguousarray(w, np.float32)
        bias = np.ascontiguousarray(bias, np.float32)
        n, H, W, cx = x.shape
        c_up = 0 if up is None else up.shape[3]
        up = None if up is None else np.ascontiguousarray(up, np.float32)
        resid = None if resid is None else np.ascontiguousarray(resid, np.float32)
        cout = w.shape[3]
        out = np.empty((n, H // stride, W // stride, cout), np.float32)
        check(self._L.whenet_det_debug_conv(self._h, _ptr(x), _ptr(up), n, H, W, cx + c_up, c_up, _ptr(w), _ptr(bias), k, stride, cout,
                                            int(leaky), _ptr(resid), _ptr(out)))
        return out

    def debug_maxpool(self, x, stride: int):
        """The device 2x2 max-pool (TF SAME) of x (n,H,W,C), rounded to bf16 on the way in (fp32 detector: as given)
        -> (n, ceil(H/s), ceil(W/s), C)."""
        x = np.ascontiguousarray(x, np.float32)
        n, H, W, c = x.shape
        out = np.empty((n, -(-H // stride), -(-W // stride), c), np.float32)
        check(self._L.whenet_det_debug_maxpool(self._h, _ptr(x), n, H, W, c, int(stride), _ptr(out)))
        return out

    def debug_decode(self, heads, img_h: int, img_w: int, max_boxes: int = 20):
        """Raw fp32 head tensors [(n,gh,gw,3(5+C)) x 3 (tiny: 2)] -> per-frame (boxes, scores, classes) through the device
        decode + NMS."""
        hs = [np.ascontiguousarray(h, np.float32) for h in heads]
        if len(hs) != len(yolo_arch.heads(self.tiny)):
            raise ValueError("%d head tensors for a detector with %d heads" % (len(hs), len(yolo_arch.heads(self.tiny))))
        n = hs[0].shape[0]
        slots = self.num_classes * max_boxes
        boxes = np.empty((n, slots, 4), np.float32)
        scores = np.empty((n, slots), np.float32)
        classes = np.empty((n, slots), np.int32)
        counts = np.empty((n,), np.int32)
        check(self._L.whenet_det_debug_decode(self._h, _ptr(hs[0]), _ptr(hs[1]), _ptr(hs[2]) if len(hs) > 2 else None, n, img_h, img_w, self.score, self.iou, max_boxes,
                                              _ptr(boxes), _ptr(scores), _ptr(classes), _ptr(counts)))
        return [(boxes[i, :counts[i]].copy(), scores[i, :counts[i]].copy(), classes[i, :counts[i]].copy()) for i in range(n)]

    def debug_force_large_decode(self, on: bool = True):
        """Run decode + NMS through the route for more than 24,576 candidates whatever the size (see
        whenet_det_debug_force_large_decode); False restores the choice by candidate count."""
        check(self._L.whenet_det_debug_force_large_decode(self._h, int(bool(on))))

    def synchronize(self):
        check(self._L.whenet_det_synchronize(self._h))

    def close_session(self):
        """reference yolo_postprocess.py:177-178"""
        self.close()

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.whenet_det_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
