"""whenet_b200 - H100-native WHENet per-crop forward (hand-written sm_90a CUDA behind a C ABI).

The directory is named ``headposeestimation-whenet_b200`` (not importable as
is); import it as ``whenet_b200`` through the shim package at the repo root.
"""
from .whenet import WHENet, WHENetModel  # noqa: F401
from .yolo import YOLO  # noqa: F401
from . import arch, build, crops, dp, overlay, pipeline, video, weights, yolo_arch  # noqa: F401
from ._lib import WhenetError, lib_path  # noqa: F401

__all__ = ["WHENet", "WHENetModel", "YOLO", "WhenetError", "arch", "build", "crops", "dp", "overlay", "pipeline", "video", "weights",
           "yolo_arch", "lib_path"]
