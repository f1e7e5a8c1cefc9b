"""Host-side mirror of the reference's ``whenet.py``: same class, same methods,
same argument meaning and error behaviour - the arithmetic runs in
``libwhenet_b200.so`` (hand-written sm_90a CUDA) instead of Keras/TensorFlow.

Reference surface kept (SURVEY.md section 8b):
  ``WHENet(snapshot=None)``                      reference whenet.py:7-20
  ``.model.predict(x, batch_size=8)``            reference whenet.py:14,27  -> [(N,120),(N,66),(N,66)] float32 logits
  ``.model.summary()``                           reference demo.py:22
  ``.idx_tensor`` / ``.idx_tensor_yaw``          reference whenet.py:17-20
  ``.get_angle(img)``                            reference whenet.py:22-34  -> (yaw, pitch, roll) float32 (N,)

There is no CPU fallback: without the shared library or an H100 the constructor raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from . import _lib, arch, crops as _crops, weights as _weights
from ._lib import WhenetError, check


def _ptr(a):
    """Raw address of a numpy array / torch tensor / int."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    raise TypeError("cannot take the address of %r" % type(a))


def _is_device(a) -> bool:
    return hasattr(a, "is_cuda") and bool(a.is_cuda)


class WHENetModel:
    """What the reference exposes as ``WHENet.model`` (a ``keras.models.Model``):
    only ``predict``, ``summary`` and ``load_weights`` are reachable from the
    reference's callers (whenet.py:16,27; demo.py:22)."""

    def __init__(self, owner: "WHENet"):
        self._o = owner

    def load_weights(self, snapshot):
        self._o._load(snapshot)

    def predict(self, x, batch_size: int = 8, verbose: int = 0):
        """Normalised float input (N,224,224,3) -> [yaw(N,120), pitch(N,66), roll(N,66)] logits.

        ``batch_size`` is accepted for signature compatibility (reference
        whenet.py:27); results do not depend on it (the kernels are batch
        invariant), so the library picks its own chunking.
        """
        x = np.asarray(x)
        self._o._check_shape(x)
        x = np.ascontiguousarray(x, dtype=np.float32)
        _ang, logits = self._o._forward(x, want_logits=True)
        return [logits[:, :120].copy(), logits[:, 120:186].copy(), logits[:, 186:].copy()]

    def summary(self, print_fn=print):
        lines = ["WHENet (EfficientNet-B0 backbone, H100-native CUDA path, precision=%s)" % self._o.precision,
                 "%-22s %-18s %-10s" % ("Layer", "Output shape", "Params"), "=" * 54]
        total = 0
        def row(name, shape, params):
            nonlocal total
            total += params
            lines.append("%-22s %-18s %-10d" % (name, shape, params))
        row("stem conv3x3 s2+bn", "(112,112,32)", 27 * 32 + 4 * 32)
        for b in arch.blocks():
            p = (b.cin * b.cexp + 4 * b.cexp if b.has_expand else 0) + b.k * b.k * b.cexp + 4 * b.cexp \
                + b.cexp * b.cse + b.cse + b.cse * b.cexp + b.cexp + b.cexp * b.cout + 4 * b.cout
            row("mbconv%d k%d s%d e%d" % (b.idx, b.k, b.s, b.cexp // b.cin), "(%d,%d,%d)" % (b.hout, b.hout, b.cout), p)
        row("head conv1x1+bn", "(7,7,1280)", 320 * 1280 + 4 * 1280)
        row("global_average_pool", "(1280,)", 0)
        row("yaw_new", "(120,)", 1280 * 120 + 120)
        row("pitch_new", "(66,)", 1280 * 66 + 66)
        row("roll_new", "(66,)", 1280 * 66 + 66)
        lines.append("=" * 54)
        lines.append("Total params: %d" % total)
        for ln in lines:
            print_fn(ln)


class WHENet:
    def __init__(self, snapshot=None, *, device: Optional[int] = None, precision: Optional[str] = None,
                 max_batch: int = 512):
        self.precision = precision or os.environ.get("WHENET_PRECISION", "fp32")
        if self.precision not in _lib.PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(_lib.PRECISIONS))
        self.device = int(os.environ.get("LOCAL_RANK", "0")) if device is None else int(device)
        self.max_batch = int(max_batch)
        self._L = _lib.load()
        self._h = C.c_void_p()
        check(self._L.whenet_create(C.byref(self._h), self.device, self.max_batch, _lib.PRECISIONS[self.precision]))
        self.model = WHENetModel(self)
        self._load(snapshot)
        # reference whenet.py:17-20
        self.idx_tensor = np.array([idx for idx in range(66)], dtype=np.float32)
        self.idx_tensor_yaw = np.array([idx for idx in range(120)], dtype=np.float32)

    # ------------------------------------------------------------------ plumbing
    PACKED_FORMAT = "whenet-b200-packed-v3"

    def _load(self, snapshot):
        if snapshot is not None and os.fspath(snapshot).endswith(".safetensors"):
            from . import stlite
            z, meta = stlite.load(os.fspath(snapshot)) if os.path.exists(os.fspath(snapshot)) else (None, {})
            if z is not None and meta.get("format") == self.PACKED_FORMAT:
                return self._import_packed(z, meta)
        _names, w = _weights.load_snapshot(snapshot)
        arr = (_lib.Tensor * len(w))()
        keep = []
        for i, (name, a) in enumerate(w.items()):
            a = np.ascontiguousarray(a, dtype=np.float32)
            keep.append(a)
            arr[i].name = name.encode()
            arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[i].ndim = a.ndim
            for d in range(a.ndim):
                arr[i].dims[d] = a.shape[d]
        check(self._L.whenet_load_weights(self._h, arr, len(w)))

    def _import_packed(self, z, meta):
        """The device image exported by ``export_packed``: BN already folded, kernels already transposed / rounded to the
        storage type - uploaded as is (replaces the HDF5 walk + fold + repack of reference whenet.py:15-16)."""
        if meta.get("precision") != self.precision:
            raise ValueError("packed weights were exported for precision %r, this model is %r" % (meta.get("precision"), self.precision))
        a32 = np.ascontiguousarray(z["arena_f32"], dtype=np.float32)
        a16 = np.ascontiguousarray(z["arena_16"], dtype=np.uint16)
        idx = np.ascontiguousarray(z["index"], dtype=np.int64)
        check(self._L.whenet_import_packed(self._h, _ptr(a32), a32.size, _ptr(a16) if a16.size else None, a16.size, _ptr(idx), idx.size))

    def export_packed(self, path):
        """Persist the packed device image of the loaded weights (fp32 arena, 16-bit arena in this model's storage type,
        index) as one .safetensors file; ``WHENet(path, precision=<same>)`` loads it without touching the Keras tensors."""
        from . import stlite
        sizes = (C.c_int64 * 3)()
        check(self._L.whenet_export_packed(self._h, None, None, None, sizes))
        a32 = np.empty((sizes[0],), np.float32)
        a16 = np.empty((sizes[1],), np.uint16)
        idx = np.empty((sizes[2],), np.int64)
        check(self._L.whenet_export_packed(self._h, _ptr(a32), _ptr(a16) if a16.size else None, _ptr(idx), sizes))
        stlite.save(path, {"arena_f32": a32, "arena_16": a16, "index": idx},
                    {"format": self.PACKED_FORMAT, "precision": self.precision, "library": self._L.whenet_version().decode()})

    @staticmethod
    def _check_shape(x):
        if x.ndim != 4 or tuple(x.shape[1:]) != (224, 224, 3):
            # Keras: "Error when checking input: expected input_1 to have shape (224, 224, 3) but got ..."
            raise ValueError("Error when checking input: expected input_1 to have shape (224, 224, 3) "
                             "but got array with shape %s" % (tuple(x.shape[1:]) if x.ndim >= 1 else x.shape,))

    def _forward(self, x: np.ndarray, want_logits: bool = False):
        """x: contiguous host array, uint8 (raw RGB) or float32 (normalised)."""
        n = x.shape[0]
        angles = np.empty((n, 3), dtype=np.float32)
        logits = np.empty((n, 252), dtype=np.float32) if want_logits else None
        fn = self._L.whenet_forward_u8 if x.dtype == np.uint8 else self._L.whenet_forward_f32
        for off in range(0, n, self.max_batch):
            nb = min(self.max_batch, n - off)
            check(fn(self._h, _ptr(x[off:off + nb]), nb, 0, _ptr(angles[off:off + nb]),
                     _ptr(logits[off:off + nb]) if want_logits else None, 0))
        return angles, logits

    # ------------------------------------------------------------------ reference surface
    def get_angle(self, img):
        """reference whenet.py:22-34.  ``img``: (N,224,224,3) RGB, values 0..255."""
        img = np.asarray(img)
        self._check_shape(img)
        if img.shape[0] == 0:
            z = np.zeros((0,), dtype=np.float32)
            return z, z.copy(), z.copy()
        if img.dtype == np.uint8:
            x = np.ascontiguousarray(img)           # normalised on the device through the float64-built table
        else:
            mean = [0.485, 0.456, 0.406]            # whenet.py:23-26, evaluated on the host exactly as there
            std = [0.229, 0.224, 0.225]
            x = img / 255
            x = (x - mean) / std
            x = np.ascontiguousarray(x, dtype=np.float32)
        angles, _ = self._forward(x)
        return angles[:, 0].copy(), angles[:, 1].copy(), angles[:, 2].copy()

    # ------------------------------------------------------------------ GPU extras (device-resident, async)
    def forward_device(self, crops_u8, angles_out, logits_out=None, n: Optional[int] = None):
        """Device-resident forward: ``crops_u8`` (n,224,224,3) uint8 CUDA tensor, ``angles_out`` (n,3)
        float32 CUDA tensor; asynchronous on the context's stream."""
        n = int(crops_u8.shape[0]) if n is None else int(n)
        check(self._L.whenet_forward_u8(self._h, _ptr(crops_u8), n, 1, _ptr(angles_out), _ptr(logits_out), 1))

    def forward_host(self, crops_u8, angles_out, logits_out=None, n: Optional[int] = None):
        """Host buffers (numpy or pinned tensors) in, host buffers out; synchronous."""
        n = int(crops_u8.shape[0]) if n is None else int(n)
        check(self._L.whenet_forward_u8(self._h, _ptr(crops_u8), n, 0, _ptr(angles_out), _ptr(logits_out), 0))

    def get_angle_from_frame(self, frame_bgr, boxes, margin: bool = True, return_crops: bool = False):
        """Stream path (reference demo_video.py:11-28 for ALL heads of a frame in one batch): ``frame_bgr`` is the
        H x W x 3 uint8 frame as cv2 delivers it, ``boxes`` the detector output (M,4) = (y_min, x_min, y_max, x_max).
        Crops are cut, colour-swapped and resized on the GPU (bit-identical to cv2.resize) and never visit the host."""
        import torch
        frame = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
        if frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be H x W x 3 uint8")
        rects = _crops.rects_from_boxes(boxes, frame.shape[0], frame.shape[1], margin)
        m = rects.shape[0]
        if m == 0:
            z = np.zeros((0,), dtype=np.float32)
            return z, z.copy(), z.copy()
        with torch.cuda.device(self.device):
            d_crops = torch.empty((m, 224, 224, 3), dtype=torch.uint8, device="cuda")
            d_ang = torch.empty((m, 3), dtype=torch.float32, device="cuda")
            check(self._L.whenet_crop_resize_u8(self._h, _ptr(frame), frame.shape[0], frame.shape[1], 0,
                                                _ptr(rects), m, 1, _ptr(d_crops)))
            for off in range(0, m, self.max_batch):
                nb = min(self.max_batch, m - off)
                check(self._L.whenet_forward_u8(self._h, _ptr(d_crops[off:off + nb]), nb, 1, _ptr(d_ang[off:off + nb]), None, 1))
            self.synchronize()
            ang = d_ang.cpu().numpy()
            out = (ang[:, 0].copy(), ang[:, 1].copy(), ang[:, 2].copy())
            return out + (d_crops.cpu().numpy(),) if return_crops else out

    def forward_host_to_device(self, crops_u8, angles_out, logits_out=None, n: Optional[int] = None):
        """Pinned host crops in, DEVICE angles out; asynchronous (H2D on the copy stream, double-buffered across calls)."""
        n = int(crops_u8.shape[0]) if n is None else int(n)
        check(self._L.whenet_forward_u8(self._h, _ptr(crops_u8), n, 0, _ptr(angles_out), _ptr(logits_out), 1))

    def forward_host_async(self, crops_u8, angles_out, logits_out=None, n: Optional[int] = None):
        """Queue H2D + forward + D2H for PINNED host buffers and return; at most two calls in flight, call
        ``synchronize()`` before reading the outputs.  Consecutive calls overlap upload and compute."""
        n = int(crops_u8.shape[0]) if n is None else int(n)
        check(self._L.whenet_forward_u8_async(self._h, _ptr(crops_u8), n, _ptr(angles_out), _ptr(logits_out)))

    def set_stream(self, stream_ptr: Optional[int]):
        """Run on a caller-owned CUDA stream.  ``0`` (torch's default stream) is passed as
        cudaStreamLegacy (handle 0x1) because a NULL handle means "back to the internal stream";
        ``None`` restores the internal stream.  Work queued after a switch runs after all work queued before it, and
        ``synchronize()`` covers both; the previous stream must still exist at the switch (torch's streams are pooled, so
        from Python it always does).  Setting the current stream again costs nothing.  Host inputs are uploaded on the
        context's copy stream, which does not wait for this stream: they must hold their data when the call is made."""
        if stream_ptr is None:
            check(self._L.whenet_set_stream(self._h, None))
        else:
            check(self._L.whenet_set_stream(self._h, C.c_void_p(stream_ptr if stream_ptr else 1)))

    def synchronize(self):
        check(self._L.whenet_synchronize(self._h))

    def set_option(self, key: str, value: int):
        check(self._L.whenet_set_option(self._h, key.encode(), int(value)))

    def enable_taps(self, on: bool = True, faithful: bool = False, crops=None):
        """Record intermediate tensors of the next forwards (``tap``).  ``faithful=False``: the first chunk of at most 8
        crops, on a one-stream route with ungated depthwise outputs.  ``faithful=True``: every chunk at any batch, on the
        route of the untapped call (in-place gated depthwise outputs are named ``dwg%d``); ``crops`` limits the taps to
        those crop indices of each call, in that order (at most 64; None: every crop)."""
        sel = np.ascontiguousarray(np.asarray([] if crops is None else list(crops), dtype=np.int32))
        check(self._L.whenet_debug_tap_crops(self._h, _ptr(sel) if sel.size else None, int(sel.size)))
        check(self._L.whenet_debug_enable_taps(self._h, (2 if faithful else 1) if on else 0))

    def tap(self, name: str) -> np.ndarray:
        n = C.c_size_t(0)
        check(self._L.whenet_debug_tap(self._h, name.encode(), None, 0, C.byref(n)))
        out = np.empty((n.value,), dtype=np.float32)
        check(self._L.whenet_debug_tap(self._h, name.encode(), _ptr(out), n.value, C.byref(n)))
        return out

    def debug_conv1x1(self, A, W, bias, gate=None, resid=None, hw=None, swish=False, use_tc=False):
        """One 1x1 conv through the chosen kernel family (test hook; see whenet_debug_conv1x1)."""
        A = np.ascontiguousarray(A, np.float32); W = np.ascontiguousarray(W, np.float32)
        bias = np.ascontiguousarray(bias, np.float32)
        M, K = A.shape
        N = W.shape[1]
        gate = None if gate is None else np.ascontiguousarray(gate, np.float32)
        resid = None if resid is None else np.ascontiguousarray(resid, np.float32)
        out = np.empty((M, N), np.float32)
        check(self._L.whenet_debug_conv1x1(self._h, int(use_tc), _ptr(A), _ptr(W), _ptr(bias), _ptr(gate), _ptr(resid),
                                           _ptr(out), M, K, N, int(hw or M), int(swish)))
        return out

    def debug_decode(self, logits) -> np.ndarray:
        """(N,252) float32 logits -> (N,3) angles through the device decode (reference utils.py:7-11, whenet.py:31-33)."""
        logits = np.ascontiguousarray(logits, np.float32)
        out = np.empty((logits.shape[0], 3), np.float32)
        check(self._L.whenet_debug_decode(self._h, _ptr(logits), logits.shape[0], _ptr(out)))
        return out

    def debug_raise_timeout(self):
        """Test hook: a device kernel raises the mbarrier-timeout flag; the next synchronising call must fail."""
        check(self._L.whenet_debug_raise_timeout(self._h))

    def set_k1_plan(self, block: int, th: int, tw: int, r: int, cc: int, nt: int = 256, nb: int = 1) -> bool:
        """Tuning hook (see whenet_debug_set_k1_plan); returns False when the plan cannot run."""
        return self._L.whenet_debug_set_k1_plan(self._h, block, th, tw, r, cc, nt, nb) == 0

    def enable_profile(self, on: bool = True):
        check(self._L.whenet_profile_enable(self._h, int(on)))

    def read_profile(self):
        cap = 256
        arr = (_lib.KernelStat * cap)()
        n = self._L.whenet_profile_read(self._h, arr, cap)
        if n < 0:
            check(n)
        return [{"name": arr[i].name.decode(), "ms": float(arr[i].ms), "launches": int(arr[i].launches),
                 "bytes": float(arr[i].bytes), "flops": float(arr[i].flops)} for i in range(min(n, cap))]

    def launch_count(self) -> int:
        return int(self._L.whenet_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.whenet_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
