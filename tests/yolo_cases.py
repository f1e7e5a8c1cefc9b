"""Shapes and sizes the YOLOv3 detector's GPU tests run, in one place so that the host-side plan test
(test_yolo_plans.py) can prove they reach every conv tile plan the library can choose, and the Pillow letterbox
helper both the CPU and the GPU letterbox tests compare against."""
import numpy as np

# model input sizes (h, w) of the per-layer, end-to-end and canvas tests (one class).  (448, 608) alone reaches every tile
# plan a one-class model can choose on 132 SMs; (32, 32) has a 1 x 1 coarse grid; the non-square ones catch swapped H/W
# index math.
MODEL_SIZES = [(416, 416), (608, 608), (448, 608), (608, 448), (32, 32), (96, 160)]

# frame (h, w) letterboxed to each model size: they pad along each axis in turn (and at (416, 416) fill it exactly once)
FRAMES = {(416, 416): (720, 1280), (608, 608): (1080, 720), (448, 608): (600, 600), (608, 448): (500, 1000),
          (32, 32): (45, 30), (96, 160): (200, 150)}

# class count -> model input sizes whose three output convs are checked against the oracle
CLASS_SIZES = {2: [(416, 416)], 80: [(416, 416), (608, 608)]}

# whenet_det_debug_conv cases: (n, H, W, cin, c_up, cout, k, stride, mode, un) with cin the total input channels and un the
# tile width the planner picks on 132 SMs (test_yolo_plans.py checks it)
DEBUG_CONVS = [
    (2, 13, 20, 64, 0, 64, 3, 1, "leaky", 32),          # H != W, tiles straddle frames
    (2, 13, 20, 64, 0, 32, 3, 2, "leaky", 32),          # odd H, even W at stride 2
    (1, 20, 13, 64, 0, 32, 3, 2, "leaky", 32),          # even H, odd W at stride 2
    (2, 10, 14, 192, 128, 64, 1, 1, "cat", 32),         # concat, H != W
    (1, 13, 20, 128, 0, 128, 3, 1, "res", 32),          # residual, H != W
    (1, 152, 144, 64, 0, 64, 3, 1, "leaky", 64),
    (1, 144, 152, 64, 0, 64, 3, 1, "res", 64),
    (1, 104, 112, 64, 0, 256, 3, 1, "leaky", 128),      # 128-wide tile, three-stage ring
    (1, 112, 104, 64, 0, 256, 3, 1, "res", 128),
    (1, 208, 200, 64, 0, 256, 3, 2, "leaky", 128),      # stride 2 at 128 wide
    (2, 76, 72, 64, 0, 255, 1, 1, "f32", 64),           # 80-class head width: 63-column tail tile
]


def pil_letterbox(img, size):
    """The reference's letterbox_image (utils.py:23-34) on Pillow itself; ``size`` = (w, h)."""
    from PIL import Image
    im = Image.fromarray(img)
    iw, ih = im.size
    w, h = size
    scale = min(w / iw, h / ih)
    nw, nh = int(iw * scale), int(ih * scale)
    im = im.resize((nw, nh), Image.BICUBIC)
    new = Image.new("RGB", size, (128, 128, 128))
    new.paste(im, ((w - nw) // 2, (h - nh) // 2))
    return np.asarray(new)


def int_round_differ():
    """A frame size (W, H) whose letterbox extent differs between int() (utils.py:28) and round() (model.py:159) at 416."""
    for W in range(300, 2000):
        H = 333
        s = min(416 / W, 416 / H)
        if int(W * s) != round(W * s) or int(H * s) != round(H * s):
            return W, H
    raise AssertionError("no such size")


def nan_iou_heads(n=1):
    """416 x 416 one-class heads, zero logits (score 0.25) except two coarse cells whose candidates score 1 and whose exp(t_w),
    exp(t_h) overflow: both boxes are (-inf, -inf, inf, inf) and their IoU is NaN."""
    heads = [np.zeros((n, 13 << l, 13 << l, 18), np.float32) for l in range(3)]
    for y, x in ((2, 3), (9, 7)):
        heads[0][:, y, x, 2:4] = 100
        heads[0][:, y, x, 4:6] = 200
    return heads


# frame sizes (W, H) of the Pillow letterbox tests
SIZES = [(1, 1), (2, 3), (3, 2), (7, 5), (13, 13), (31, 17), (64, 48), (99, 101), (100, 300), (300, 100), (415, 415), (416, 416),
         (417, 417), (416, 234), (234, 416), (640, 480), (480, 640), (500, 499), (800, 600), (1280, 720), (1920, 1080), (1080, 1920),
         (1000, 5), (123, 457), (333, 222), (208, 208), (832, 832), (200, 100), (57, 911), int_round_differ()]
