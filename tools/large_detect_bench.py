"""The detector at model inputs above 608 (DESIGN.md 8.6) on one GPU: ms per frame and TFLOP/s of whole detect_frames calls
for YOLOv3 and tiny YOLOv3 at 1088 x 1920 (n = 1, 4) and 2176 x 3840 (n = 1), three alternating rounds after a warm-up; the
kernel split of each from torch.profiler in a separate pass; both decode + NMS routes at 416^2 and 608^2 (n = 1, 8) from
their kernel times; and detect_and_estimate_frames at 1088 x 1920 with about 20 heads per frame.  Prints the card's name,
power limit and max SM clock of the same run.

    python tools/large_detect_bench.py [--iters 20] [--out large_detect_bench.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from detect_bench import TINY_ANCHORS, card, frame1080, kernel_table, set_objectness_for_boxes, time_calls  # noqa: E402

DECODE = ("yolo_decode_nms_kernel", "yolo_decode_kernel", "yolo_nms_kernel", "yolo_pack_kernel")


def _decode_ms(kt):
    return sum(r[1] for r in kt if any(r[0].endswith(k) for k in DECODE))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import whenet_b200
    from whenet_b200 import yolo_arch as Y
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "calls": [], "routes": []}
    print("card:", res["card"])
    f = frame1080()
    # whole calls: (network, size, n), three alternating rounds over the cases of one detector
    for tiny in (False, True):
        anchors = TINY_ANCHORS if tiny else None
        for size, ns in (((1088, 1920), (1, 4)), ((2176, 3840), (1,))):
            m = whenet_b200.YOLO(None, anchors_path=anchors, model_image_size=size, max_frames=max(ns), score=0.3)
            flops = 2.0 * Y.macs_per_frame(*size, tiny=tiny)
            inputs = {n: torch.from_numpy(np.stack([f] * n)[:, :, :, ::-1].copy()).cuda() for n in ns}
            for n in ns:
                time_calls(lambda: m.detect_frames(inputs[n]), 2)          # warm-up: graph capture, module load
            secs = {n: [] for n in ns}
            for _ in range(3):
                for n in ns:
                    secs[n].append(time_calls(lambda: m.detect_frames(inputs[n]), a.iters))
            for n in ns:
                kt = kernel_table(lambda: m.detect_frames(inputs[n]))
                sec = min(secs[n])
                body = sum(r[1] for r in kt) - _decode_ms(kt)
                r = {"network": "tiny YOLOv3" if tiny else "YOLOv3", "size": size, "n": n, "ms_per_frame_rounds": [s * 1e3 / n for s in secs[n]],
                     "ms_per_frame": sec * 1e3 / n, "tflops_call": flops * n / sec / 1e12, "decode_nms_ms": _decode_ms(kt),
                     "body_ms": body, "kernels": kt}
                res["calls"].append(r)
                print("%s %dx%d n=%d: %.3f ms/frame (rounds %s), %.1f TFLOP/s (call); kernels: body %.3f ms, decode+NMS %.3f ms" %
                      (r["network"], size[0], size[1], n, r["ms_per_frame"], ", ".join("%.3f" % v for v in r["ms_per_frame_rounds"]),
                       r["tflops_call"], body, r["decode_nms_ms"]))
                for k in kt[:8]:
                    print("    %-40s %8.4f ms  x%d" % tuple(k))
            m.close()
    # both decode routes where both run: kernel time of decode + NMS alone, alternating the routes
    for size in (416, 608):
        m = whenet_b200.YOLO(None, model_image_size=(size, size), max_frames=8, score=0.3)
        for n in (1, 8):
            d = torch.from_numpy(np.stack([f] * n)[:, :, :, ::-1].copy()).cuda()
            ms = {False: [], True: []}
            for _ in range(3):
                for forced in (False, True):
                    m.debug_force_large_decode(forced)
                    ms[forced].append(_decode_ms(kernel_table(lambda: m.detect_frames(d))))
            m.debug_force_large_decode(False)
            r = {"size": size, "n": n, "one_cta_ms": ms[False], "three_kernel_ms": ms[True]}
            res["routes"].append(r)
            print("decode+NMS %d^2 n=%d: one-CTA kernel %s ms, three kernels %s ms" %
                  (size, n, ", ".join("%.4f" % v for v in ms[False]), ", ".join("%.4f" % v for v in ms[True])))
        m.close()
    # the pipeline at 1088 x 1920 with about 20 heads per frame
    m = whenet_b200.YOLO(None, model_image_size=(1088, 1920), max_frames=4)
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=128)
    best = set_objectness_for_boxes(m, f, False)
    frames = torch.from_numpy(np.stack([f] * 4)[:, :, :, ::-1].copy()).cuda()
    time_calls(lambda: whenet_b200.pipeline.detect_and_estimate_frames(m, wn, frames), 2)
    sec = min(time_calls(lambda: whenet_b200.pipeline.detect_and_estimate_frames(m, wn, frames), a.iters) for _ in range(3))
    res["pipeline"] = {"boxes_per_frame": best[1], "ms_per_frame": sec * 1e3 / 4}
    print("detect_and_estimate_frames 4 x 1080p at 1088x1920, %d boxes/frame: %.3f ms/frame" % (best[1], sec * 1e3 / 4))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
