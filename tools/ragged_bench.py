"""Head poses for a camera set of mixed frame sizes: eight 1080p-class frames of eight different sizes, about 20 heads each,
through pipeline.detect_and_estimate_frames (detector at 416^2, WHENet bf16) - one call per size group (eight calls of one
frame: what frames of different sizes needed before the per-frame entries) against one call on the list.  Both arms' results
are checked bit for bit on the timed frames, for host and device frames, YOLOv3 and tiny YOLOv3.  Prints the card's name,
power limit and max SM clock of the same run.  ``--profile`` instead prints the torch.profiler kernel table of one call on
the list (take it in a run of its own: tracing slows the host).

    python tools/ragged_bench.py [--iters 30] [--profile] [--out ragged_bench.json]
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

# (H, W): landscape, portrait and cropped 1080p-class cameras
SIZES = [(1080, 1920), (1920, 1080), (1080, 1440), (1200, 1920), (1024, 1920), (1080, 1800), (960, 1920), (1152, 2048)]


def frame(h, w, seed):
    """A 1080p synthetic frame (detect_bench.frame1080) cut or tiled to h x w, BGR."""
    f = frame1080(seed)
    f = np.tile(f, (2, 2, 1))[:h, :w]
    return np.ascontiguousarray(f[:, :, ::-1])


def same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v, equal_nan=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--profile", action="store_true", help="print the kernel table of one call on the list instead of timing")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import whenet_b200
    from whenet_b200 import pipeline
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "sizes": SIZES, "runs": []}
    print("card:", res["card"])
    frames = [frame(h, w, seed=i) for i, (h, w) in enumerate(SIZES)]
    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=256)
    for tiny in (False, True):
        net = "tiny YOLOv3" if tiny else "YOLOv3"
        yolo = whenet_b200.YOLO(None, anchors_path=TINY_ANCHORS if tiny else None, max_frames=8)
        bias, k = set_objectness_for_boxes(yolo, frame1080(), tiny)
        for src in ("host", "device"):
            x = frames if src == "host" else [torch.from_numpy(f).cuda() for f in frames]
            torch.cuda.synchronize()
            groups = [f[None] for f in x]
            per_group = lambda: [r for g in groups for r in pipeline.detect_and_estimate_frames(yolo, wn, g)]  # noqa: E731
            ragged = lambda: pipeline.detect_and_estimate_frames(yolo, wn, x)  # noqa: E731
            if a.profile:
                kt = kernel_table(ragged)
                res["runs"].append({"network": net, "source": src, "kernels": kt})
                print("%s, %s frames, one call on the list: %.3f ms of kernels" % (net, src, sum(r[1] for r in kt)))
                for row in kt:
                    print("    %-48s %8.4f ms  x%d" % tuple(row))
                continue
            ref, got = per_group(), ragged()            # warm-up of every size list, and the bitwise check
            same(got, ref)
            heads = sum(len(r[0]) for r in got)
            t_group = time_calls(per_group, a.iters)
            t_ragged = time_calls(ragged, a.iters)
            same(ragged(), ref)
            r = {"network": net, "source": src, "objectness_bias": float(bias), "heads": heads,
                 "ms_per_frame_per_size_group": t_group * 1e3 / len(frames), "ms_per_frame_one_call": t_ragged * 1e3 / len(frames),
                 "speedup": t_group / t_ragged}
            res["runs"].append(r)
            print("%-11s %-6s %3d heads: one call per size group %.3f ms/frame, one call on the list %.3f ms/frame (x%.2f)"
                  % (net, src, heads, r["ms_per_frame_per_size_group"], r["ms_per_frame_one_call"], r["speedup"]))
        yolo.close()
    wn.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
