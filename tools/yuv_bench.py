"""Head poses from BGR, NV12 and I420 video frames on one GPU: pipeline.detect_and_estimate_frames on 8 frames of 1080p per
call, from host numpy frames and from device frames, for YOLOv3 and tiny YOLOv3 at 416^2 (head objectness biases set so that
about 20 boxes survive per frame, as tools/pipeline_bench.py does), WHENet in bf16.

The YUV frames are made from synthetic BGR scenes; the BGR arm runs on cv2.cvtColor(yuv, COLOR_YUV2BGR_NV12 / _I420) of the
same frames, and every YUV arm's boxes, scores and angles are checked bit for bit against it.  Every arm is warmed up, then the
arms are timed in alternation over several rounds (the spread across rounds is reported with the median).  Prints the card's
name, power limit and max SM clock of the same run.

    python tools/yuv_bench.py [--iters 20] [--rounds 3] [--out yuv_bench.json]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from detect_bench import ROOT, TINY_ANCHORS, card, frame1080, set_objectness_for_boxes, time_calls  # noqa: E402  (puts the repository on sys.path)

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import yuv_oracle  # noqa: E402

N_FRAMES = 8


def same(a, b):
    return len(a) == len(b) and all(all(np.array_equal(x, y, equal_nan=True) for x, y in zip(p, q)) for p, q in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import pipeline
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "input": "416x416", "frames": "1080x1920", "frames_per_call": N_FRAMES,
           "whenet": "bf16", "runs": []}
    print("card:", res["card"])
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16")
    codes = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420}
    for tiny in (False, True):
        net = "tiny YOLOv3" if tiny else "YOLOv3"
        m = whenet_b200.YOLO(None, anchors_path=TINY_ANCHORS if tiny else None, max_frames=N_FRAMES)
        bias, _k = set_objectness_for_boxes(m, frame1080(), tiny)
        arms = {}
        for fmt in ("nv12", "i420"):
            yuv = np.stack([yuv_oracle.bgr_to_yuv420(frame1080(100 + s), fmt) for s in range(N_FRAMES)])
            bgr = np.stack([cv2.cvtColor(f, codes[fmt]) for f in yuv])
            want = pipeline.detect_and_estimate_frames(m, wn, bgr)
            for src, x, xb in (("host", yuv, bgr), ("device", torch.from_numpy(yuv).cuda(), torch.from_numpy(bgr).cuda())):
                got = pipeline.detect_and_estimate_frames(m, wn, x, pixel_format=fmt)
                assert same(got, want), "%s %s %s frames differ from the BGR path on cv2.cvtColor's output" % (net, fmt, src)
                arms[(fmt, src)] = (lambda x=x, fmt=fmt: pipeline.detect_and_estimate_frames(m, wn, x, pixel_format=fmt))
                if fmt == "nv12":       # the BGR arm on the converted frames of one layout
                    arms[("bgr", src)] = (lambda xb=xb: pipeline.detect_and_estimate_frames(m, wn, xb))
            boxes = float(np.mean([len(r[0]) for r in want]))
        torch.cuda.synchronize()
        samples = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                samples[k].append(time_calls(fn, a.iters) / N_FRAMES * 1e3)
        print("%s, objectness bias %.2f, %.1f boxes per frame:" % (net, bias, boxes))
        for (fmt, src), ms in sorted(samples.items(), key=lambda kv: (kv[0][1], kv[0][0])):
            row = {"network": net, "pixel_format": fmt, "source": src, "ms_per_frame": float(np.median(ms)), "min": float(min(ms)),
                   "max": float(max(ms)), "boxes_per_frame": boxes}
            res["runs"].append(row)
            print("    %-6s %-6s frames: %7.3f ms/frame (rounds %.3f..%.3f)" % (src, fmt, row["ms_per_frame"], row["min"], row["max"]))
        m.close()
    wn.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
