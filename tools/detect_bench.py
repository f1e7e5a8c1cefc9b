"""Detector throughput on one GPU: frames/s and TFLOP/s of whenet_b200.YOLO at 416^2 and 608^2 for n = 1 and 8 frames per
call, a per-kernel breakdown from CUDA events (torch.profiler), and the full detect_and_estimate frames/s with the head
biases set so that each frame yields about 20 boxes.  Prints the card's name, power limit and max SM clock of the same run.
``--tiny`` measures tiny YOLOv3 (the 6 anchors of tests/golden/tiny_yolo_anchors.txt) instead of YOLOv3; ``--precision fp32``
the detector's fp32 parity mode (and WHENet's fp32 mode in the detect_and_estimate row) instead of bf16.

    python tools/detect_bench.py [--tiny] [--precision {bf16,fp32}] [--iters 50] [--out detect_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BF16_DENSE = 989e12        # H100 SXM data sheet, dense BF16 (700 W part)
TINY_ANCHORS = os.path.join(ROOT, "tests", "golden", "tiny_yolo_anchors.txt")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return "unknown (%s)" % e


def frame1080(seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:1080, 0:1920]
    img = np.stack([127 + 120 * np.sin(x / (17 + 5 * c) + y / (23 + c) + rng.random() * 6) for c in range(3)], -1)
    return np.clip(img + rng.normal(0, 6, img.shape), 0, 255).astype(np.uint8)


def set_objectness_for_boxes(m, frame, tiny, target=20):
    """Load seeded random weights into detector ``m`` with the objectness bias of every head anchor set to the value in
    -1..3 (steps of 0.25) whose detections on ``frame`` (BGR) come closest to ``target`` boxes -> (bias, boxes)."""
    from whenet_b200 import yolo_arch as Y
    names, w = Y.random_weights(0, tiny=tiny)
    layers, _ = Y.map_weights(names, w, tiny=tiny)

    def load(bias):
        for i in Y.heads(tiny):
            b = np.zeros_like(layers[i]["bias"])
            b[4::6] = bias
            layers[i]["bias"] = b
        m.load_layers(layers)

    best = None
    for bias in np.arange(-1.0, 3.01, 0.25):
        load(bias)
        k = len(m.detect(frame[:, :, ::-1].copy())[0])
        if best is None or abs(k - target) < abs(best[1] - target):
            best = (bias, k)
    load(best[0])
    return best


def time_calls(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def kernel_table(fn):
    """Per-kernel CUDA time of one call (torch.profiler, CUDA activities), grouped by kernel name."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rows = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.split("(")[0].replace("void ", "")
            for k0 in ("yolo_conv0_kernel", "yolo_conv0_32_kernel"):
                if k0 + "<" in e.name:
                    name = k0
            for kern in ("conv_igemm_kernel", "conv_igemm32_kernel"):
                for mode in "0123":
                    if "%s<%s" % (kern, mode) in e.name:
                        name = "%s[%s]" % (kern.replace("_kernel", ""), {"0": "leaky", "1": "leaky+res", "2": "concat", "3": "head fp32"}[mode])
            r = rows.setdefault(name, [0.0, 0])
            r[0] += e.device_time_total / 1e3
            r[1] += 1
    return sorted(([k, round(v[0], 4), v[1]] for k, v in rows.items()), key=lambda r: -r[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    ap.add_argument("--tiny", action="store_true", help="tiny YOLOv3 (6 anchors) instead of YOLOv3")
    ap.add_argument("--precision", choices=("bf16", "fp32"), default="bf16", help="the detector's precision (default bf16)")
    a = ap.parse_args()
    import torch
    import whenet_b200
    from whenet_b200 import yolo_arch as Y
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    anchors = TINY_ANCHORS if a.tiny else None
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "network": "tiny YOLOv3" if a.tiny else "YOLOv3",
           "precision": a.precision, "runs": []}
    print("card:", res["card"], " network:", res["network"], " precision:", a.precision)
    f = frame1080()
    for size in (416, 608):
        m = whenet_b200.YOLO(None, anchors_path=anchors, model_image_size=(size, size), max_frames=8, precision=a.precision)
        flops = 2.0 * Y.macs_per_frame(size, size, tiny=a.tiny)
        for n in (1, 8):
            frames = np.stack([f] * n)[:, :, :, ::-1].copy()
            d_frames = torch.from_numpy(frames).cuda()
            sec = time_calls(lambda: m.detect_frames(d_frames), a.iters)
            kt = kernel_table(lambda: m.detect_frames(d_frames))
            gpu_ms = sum(r[1] for r in kt)
            r = {"size": size, "n": n, "ms_per_call": sec * 1e3, "ms_per_frame": sec * 1e3 / n, "frames_per_s": n / sec,
                 "tflops_call": flops * n / sec / 1e12, "kernel_ms_sum": gpu_ms, "tflops_kernels": flops * n / (gpu_ms / 1e3) / 1e12,
                 "share_of_bf16_dense_peak_kernels": flops * n / (gpu_ms / 1e3) / PEAK_BF16_DENSE, "kernels": kt}
            res["runs"].append(r)
            print("%d^2 n=%d: %.3f ms/frame  %.1f frames/s  %.1f TFLOP/s (call)  kernels %.3f ms = %.1f TFLOP/s (%.1f%% of 989)" %
                  (size, n, r["ms_per_frame"], r["frames_per_s"], r["tflops_call"], gpu_ms, r["tflops_kernels"],
                   100 * r["share_of_bf16_dense_peak_kernels"]))
            for k in kt[:8]:
                print("    %-40s %8.4f ms  x%d" % tuple(k))
        m.close()
    # full pipeline: head objectness biases raised so that about 20 boxes survive NMS per frame
    m = whenet_b200.YOLO(None, anchors_path=anchors, max_frames=1, precision=a.precision)
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision=a.precision, max_batch=64)
    best = set_objectness_for_boxes(m, f, a.tiny)
    sec = time_calls(lambda: whenet_b200.pipeline.detect_and_estimate(m, wn, f), a.iters)
    res["pipeline"] = {"boxes_per_frame": best[1], "objectness_bias": float(best[0]), "ms_per_frame": sec * 1e3, "frames_per_s": 1 / sec}
    print("detect_and_estimate 1080p -> 416^2, %d boxes/frame: %.3f ms/frame, %.1f frames/s" % (best[1], sec * 1e3, 1 / sec))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
