"""Frames -> head poses on one GPU: the per-frame loop (pipeline.detect_and_estimate once per frame) against
pipeline.detect_and_estimate_frames at n = 1, 8 and 32 frames per call, from device frames and from host numpy frames (the
difference is the upload share).  1080p synthetic frames, YOLOv3 at 416^2 (``--tiny``: tiny YOLOv3) with the head objectness
biases set so that about 20 boxes survive per frame, WHENet in bf16.  Every shape is warmed up before it is timed, the batched
results are checked bit for bit against the per-frame results on the timed frames, and a torch.profiler kernel table of one
n = 8 call is taken in a separate run.  Prints the card's name, power limit and max SM clock of the same run.

    python tools/pipeline_bench.py [--tiny] [--iters 20] [--max-frames 8] [--out pipeline_bench.json]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from detect_bench import TINY_ANCHORS, card, frame1080, kernel_table, set_objectness_for_boxes, time_calls  # noqa: E402  (puts the repository on sys.path)


def same(a, b):
    return len(a) == len(b) and all(all(np.array_equal(x, y, equal_nan=True) for x, y in zip(p, q)) for p, q in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--max-frames", type=int, default=8, help="detector frames per call (chunk size)")
    ap.add_argument("--tiny", action="store_true", help="tiny YOLOv3 (6 anchors) instead of YOLOv3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import whenet_b200
    from whenet_b200 import pipeline
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "network": "tiny YOLOv3" if a.tiny else "YOLOv3",
           "input": "416x416", "frames": "1080x1920", "max_frames": a.max_frames, "whenet": "bf16"}
    print("card:", res["card"], " network:", res["network"], " detector chunk:", a.max_frames)
    m = whenet_b200.YOLO(None, anchors_path=TINY_ANCHORS if a.tiny else None, max_frames=a.max_frames)
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16")
    res["objectness_bias"], _k = set_objectness_for_boxes(m, frame1080(), a.tiny)
    res["objectness_bias"] = float(res["objectness_bias"])
    # 32 distinct frames on which the per-frame path runs (it raises on a head whose slice is empty)
    frames, seed = [], 0
    while len(frames) < 32:
        f = frame1080(seed)
        seed += 1
        try:
            pipeline.detect_and_estimate(m, wn, f)
        except whenet_b200.WhenetError:
            continue
        frames.append(f)
    host = np.stack(frames)
    dev = torch.from_numpy(host).cuda()
    per_frame = [pipeline.detect_and_estimate(m, wn, f) for f in frames]
    res["boxes_per_frame"] = float(np.mean([len(r[0]) for r in per_frame]))
    print("%.1f boxes per frame (objectness bias %.2f), %d frames" % (res["boxes_per_frame"], res["objectness_bias"], len(frames)))

    sec = time_calls(lambda: [pipeline.detect_and_estimate(m, wn, f) for f in frames], a.iters) / len(frames)
    rows = [{"path": "detect_and_estimate per frame", "n": 1, "source": "host", "ms_per_frame": sec * 1e3, "frames_per_s": 1 / sec}]
    for n in (1, 8, 32):
        for src, x in (("device", dev[:n]), ("host", host[:n])):
            got = pipeline.detect_and_estimate_frames(m, wn, x)          # warm-up of this shape, and the equality check
            assert same(got, per_frame[:n]), "batched results differ from the per-frame path (n=%d, %s frames)" % (n, src)
            sec = time_calls(lambda: pipeline.detect_and_estimate_frames(m, wn, x), a.iters) / n
            rows.append({"path": "detect_and_estimate_frames", "n": n, "source": src, "ms_per_frame": sec * 1e3, "frames_per_s": 1 / sec})
    res["runs"] = rows
    for r in rows:
        print("%-30s n=%-3d %-6s frames: %7.3f ms/frame  %7.1f frames/s" % (r["path"], r["n"], r["source"], r["ms_per_frame"], r["frames_per_s"]))
    kt = kernel_table(lambda: pipeline.detect_and_estimate_frames(m, wn, dev[:8]))
    res["kernels_n8_device"] = kt
    print("kernels of one detect_and_estimate_frames call, n=8 device frames (sum %.3f ms):" % sum(r[1] for r in kt))
    for k in kt[:16]:
        print("    %-48s %8.4f ms  x%d" % tuple(k))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)
    m.close()
    wn.close()


if __name__ == "__main__":
    main()
