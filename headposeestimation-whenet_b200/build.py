"""Build ``libwhenet_b200.so`` in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "obj")
LIB = os.path.join(HERE, "libwhenet_b200.so")
_SIMT_TC = ["kernels_simt.cuh", "kernels_tc.cuh"]
_ABI = os.path.join("..", "..", "include", "whenet_b200.h")
# translation unit -> the headers it depends on (a unit is recompiled when it or one of them is newer than its object)
UNITS = {
    "whenet_api.cu": _SIMT_TC + ["api_error.h", "kernels_fused.cuh", "kernels_k2.cuh", "kernels_tc32.cuh", "kernels_dwse.cuh", "kernels_k1x.cuh", "frames_api.h", "jpeg_api.h", _ABI],
    "frames_api.cu": ["kernels_crop.cuh", "yuv.cuh", "kernels_overlay.cuh", "hershey_simplex.inc", "frames_api.h", "api_error.h", _ABI],
    "inst_k1_bf16.cu": _SIMT_TC + ["kernels_fused.cuh", "kernels_dwse.cuh", "kernels_k1x.cuh"],
    "inst_k1_f16.cu": _SIMT_TC + ["kernels_fused.cuh"],
    "inst_dwse.cu": _SIMT_TC + ["kernels_fused.cuh", "kernels_dwse.cuh"],
    "inst_pw.cu": _SIMT_TC + ["kernels_fused.cuh", "kernels_k2.cuh"],
    "inst_yolo.cu": _SIMT_TC + ["kernels_yolo.cuh", "yuv.cuh"],
    "inst_yolo32.cu": _SIMT_TC + ["kernels_yolo.cuh", "kernels_yolo32.cuh", "yuv.cuh"],
    "yolo_api.cu": _SIMT_TC + ["kernels_yolo.cuh", "kernels_yolo32.cuh", "yuv.cuh", "api_error.h", _ABI],
    "jpeg_api.cu": ["kernels_jpeg.cuh", "jpeg_api.h", "api_error.h", "jpeg_decode.inc", "kernels_jpeg_dec.cuh", _ABI],
}
SOURCES = list(UNITS)
HEADERS = sorted({h for hs in UNITS.values() for h in hs})

# no --use_fast_math: precise expf / division are required by the fp32 parity mode.  -ffp-contract=off: the host overlay
# geometry rounds its double expressions as CPython does, never through a fused multiply-add.
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC,-ffp-contract=off"]


def _obj(src: str) -> str:
    return os.path.join(OBJ, os.path.splitext(src)[0] + ".o")


def _unit_stale(src: str) -> bool:
    o = _obj(src)
    if not os.path.exists(o):
        return True
    t = os.path.getmtime(o)
    deps = [os.path.join(CSRC, d) for d in [src] + UNITS[src]] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _stale() -> bool:
    """The library is older than one of its sources (objects are a build cache: their absence alone triggers nothing)."""
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, d) for d in SOURCES + HEADERS] + [os.path.abspath(__file__)]     # build.py holds the flags
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """Compile the stale translation units side by side (one nvcc process each) and link them into the in-tree library."""
    if not force and not _stale():
        return LIB
    from concurrent.futures import ThreadPoolExecutor
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)
    todo = [s for s in SOURCES if force or _unit_stale(s)]

    def compile_unit(src):
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas=-v"] if verbose else []) + ["-c", "-o", _obj(src), os.path.join(CSRC, src)]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        return src, subprocess.run(cmd, capture_output=True, text=True)

    with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
        results = list(ex.map(compile_unit, todo))
    for src, r in results:
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            print(r.stderr, file=sys.stderr)
    r = subprocess.run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + [_obj(s) for s in SOURCES],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
