"""Shapes and sizes the tiny YOLOv3 GPU tests (test_gpu_yolo_tiny.py) run, in one place so that the host-side plan test
(test_yolo_tiny_plans.py) can prove they reach every conv tile plan the library can choose for the tiny network."""
import os

from yolo_cases import CLASS_SIZES, FRAMES, MODEL_SIZES  # noqa: F401  (the same sizes and frames as the full model)

ANCHORS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_yolo_anchors.txt")

# whenet_det_debug_conv cases of the 3x3 concat conv (tiny conv 10: [upsample(128 ch), 256 ch] -> 256), as in yolo_cases:
# (n, H, W, cin, c_up, cout, k, stride, mode, un), un the tile width the planner picks on 132 SMs
DEBUG_CONVS = [
    (1, 26, 20, 384, 128, 256, 3, 1, "cat", 32),        # H != W
    (2, 26, 26, 384, 128, 256, 3, 1, "cat", 32),        # 676 pixels a frame: tiles straddle frames
    (1, 2, 2, 384, 128, 256, 3, 1, "cat", 32),          # conv 10 at 32 x 32: every tap but the centre reads padding
    (1, 26, 26, 384, 128, 256, 3, 1, "cat", 32),        # conv 10 at 416 x 416
    (1, 38, 38, 384, 128, 256, 3, 1, "cat", 32),        # conv 10 at 608 x 608
    (1, 96, 104, 192, 64, 128, 3, 1, "cat", 64),        # a 64-wide tile
]

# whenet_det_debug_maxpool cases: (n, H, W, C, stride)
POOLS = [(n, H, W, C, s) for n in (1, 3) for (H, W) in ((13, 13), (26, 26), (7, 12), (12, 7)) for C in (16, 64, 1024) for s in (1, 2)]
