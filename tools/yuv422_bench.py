"""YUYV camera frames and YUV -> BGR conversion on one GPU (DESIGN.md section 8.14):

  detect   pipeline.detect_and_estimate_frames on 8 frames of 1080p per call from host and device YUYV frames, against the
           same call on the BGR frames cv2.cvtColor makes of them (YOLOv3 at 416^2 with head objectness biases set so that about
           20 boxes survive per frame, as tools/yuv_bench.py does; WHENet in bf16)
  to_bgr   video.to_bgr per 1080p and 2160p frame (8 frames per call) for NV12, I420, YUYV and UYVY from device and host frames,
           against downloading the device frames, cv2.cvtColor on the host and uploading the BGR frames; plus the kernel's device
           time from the context's CUDA-event profile and the HBM bandwidth that implies
  loop     the NV12 annotate loop (detect_and_estimate_frames -> BGR frames -> draw_heads(display="full") -> encode_jpeg) with
           to_bgr, against the same loop with download + cvtColor + upload in place of to_bgr

Every arm's output is checked bit for bit against its reference after every round (detections and angles, BGR frames, JPEG
bytes).  Every arm is warmed up, then the arms of a part are timed in alternation over --rounds rounds of --iters calls each;
the median round and the spread are reported.  Prints the card's name, power limit and max SM clock of the same run.

    python tools/yuv422_bench.py [--iters 10] [--rounds 5] [--out yuv422_bench.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from detect_bench import ROOT, card, frame1080, set_objectness_for_boxes  # noqa: E402  (puts the repository on sys.path)

sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import yuv422_oracle  # noqa: E402
import yuv_oracle  # noqa: E402

N_FRAMES = 8


def same(a, b):
    return len(a) == len(b) and all(all(np.array_equal(x, y, equal_nan=True) for x, y in zip(p, q)) for p, q in zip(a, b))


def scene(H, W, seed):
    f = frame1080(seed)
    return f if (H, W) == (1080, 1920) else np.ascontiguousarray(np.tile(f, (H // 1080, W // 1920, 1)))


def timed_rounds(arms, check, iters, rounds):
    """arms: name -> fn; check(name, output) raises on a mismatch.  -> name -> list of per-call ms, one per round."""
    import torch
    for k, fn in arms.items():            # warm-up
        check(k, fn())
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(iters):
                out = fn()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t) / iters * 1e3)
            check(k, out)
    return ms


def report(res, part, ms, per, extra=None):
    for k, v in ms.items():
        row = {"part": part, "arm": k, "ms_per_frame": float(np.median(v)) / per, "min": min(v) / per, "max": max(v) / per, "rounds": len(v)}
        row.update((extra or {}).get(k, {}))
        res["runs"].append(row)
        print("  %-34s %8.3f ms/frame (rounds %.3f..%.3f)" % (k, row["ms_per_frame"], row["min"], row["max"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    res = {"card": card(), "device": torch.cuda.get_device_name(0), "frames_per_call": N_FRAMES, "iters": a.iters, "rounds": a.rounds, "runs": []}
    print("card:", res["card"])
    codes = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420, "yuyv": cv2.COLOR_YUV2BGR_YUYV, "uyvy": cv2.COLOR_YUV2BGR_UYVY}

    def make(fmt, H, W, seeds):
        conv = {}
        for s in set(seeds):
            x = scene(H, W, s)[:, :, ::-1]
            conv[s] = yuv422_oracle.bgr_to_yuv422(x, fmt) if fmt in ("yuyv", "uyvy") else yuv_oracle.bgr_to_yuv420(x, fmt)
        return np.stack([conv[s] for s in seeds])

    wn = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16")
    m = whenet_b200.YOLO(None, max_frames=N_FRAMES)
    bias, _k = set_objectness_for_boxes(m, frame1080(), False)

    # ------------------------------------------------------------------------------------------------ detect
    yuyv = make("yuyv", 1080, 1920, range(100, 100 + N_FRAMES))
    bgr = np.stack([cv2.cvtColor(f, codes["yuyv"]) for f in yuyv])
    d_yuyv, d_bgr = torch.from_numpy(yuyv).cuda(), torch.from_numpy(bgr).cuda()
    want = pipeline.detect_and_estimate_frames(m, wn, bgr)
    arms = {"host yuyv": lambda: pipeline.detect_and_estimate_frames(m, wn, yuyv, pixel_format="yuyv"),
            "host bgr": lambda: pipeline.detect_and_estimate_frames(m, wn, bgr),
            "device yuyv": lambda: pipeline.detect_and_estimate_frames(m, wn, d_yuyv, pixel_format="yuyv"),
            "device bgr": lambda: pipeline.detect_and_estimate_frames(m, wn, d_bgr)}

    def check_det(k, out):
        assert same(out, want), "%s: results differ from the BGR path on cv2.cvtColor's output" % k

    print("detect_and_estimate_frames, YOLOv3 416x416 (objectness bias %.2f, %.1f boxes per frame), 1080p:"
          % (bias, np.mean([len(r[0]) for r in want])))
    report(res, "detect", timed_rounds(arms, check_det, a.iters, a.rounds), N_FRAMES)

    # ------------------------------------------------------------------------------------------------ to_bgr
    for H, W in ((1080, 1920), (2160, 3840)):
        print("to_bgr, %dx%d:" % (W, H))
        arms, refs, extra = {}, {}, {}
        for fmt in ("nv12", "i420", "yuyv", "uyvy"):
            host = make(fmt, H, W, [0, 1, 2, 3] * (N_FRAMES // 4))
            dev = torch.from_numpy(host).cuda()
            refs[fmt] = torch.from_numpy(np.stack([cv2.cvtColor(f, codes[fmt]) for f in host])).cuda()

            def cv_arm(dev=dev, fmt=fmt):
                h = dev.cpu().numpy()
                return torch.from_numpy(np.stack([cv2.cvtColor(f, codes[fmt]) for f in h])).cuda()
            arms["%s device to_bgr" % fmt] = lambda dev=dev, fmt=fmt: video.to_bgr(wn, dev, fmt)
            arms["%s host to_bgr" % fmt] = lambda host=host, fmt=fmt: video.to_bgr(wn, host, fmt)
            arms["%s download+cvtColor+upload" % fmt] = cv_arm
            # the kernel's device time alone: the context's CUDA events around each launch
            video.to_bgr(wn, dev, fmt)
            wn.enable_profile(True)
            wn.read_profile()
            for _ in range(a.iters):
                video.to_bgr(wn, dev, fmt)
            st = [s for s in wn.read_profile() if s["name"] == "yuv_to_bgr"][0]
            wn.enable_profile(False)
            us = st["ms"] / st["launches"] / N_FRAMES * 1e3
            gbs = st["bytes"] / st["launches"] / (st["ms"] / st["launches"] * 1e-3) / 1e9
            extra["%s device to_bgr" % fmt] = {"kernel_us_per_frame": us, "kernel_GB_per_s": gbs}
            print("  %-34s %8.2f us/frame of kernel time, %.0f GB/s" % (fmt + " kernel", us, gbs))

        def check_bgr(k, out):
            assert torch.equal(out, refs[k.split()[0]]), "%s: frames differ from cv2.cvtColor" % k
        report(res, "to_bgr %dx%d" % (W, H), timed_rounds(arms, check_bgr, a.iters, a.rounds), N_FRAMES, extra)

    # ------------------------------------------------------------------------------------------------ NV12 annotate loop
    nv12 = torch.from_numpy(make("nv12", 1080, 1920, range(200, 200 + N_FRAMES))).cuda()

    def loop(convert):
        results = pipeline.detect_and_estimate_frames(m, wn, nv12, pixel_format="nv12")
        frames = convert()
        overlay.draw_heads(wn, frames, results, display="full")
        return video.encode_jpeg(wn, frames)

    def host_convert():
        h = nv12.cpu().numpy()
        return torch.from_numpy(np.stack([cv2.cvtColor(f, codes["nv12"]) for f in h])).cuda()
    want_jpeg = loop(host_convert)
    arms = {"loop with to_bgr": lambda: loop(lambda: video.to_bgr(wn, nv12, "nv12")), "loop with host cvtColor": lambda: loop(host_convert)}

    def check_loop(k, out):
        assert out == want_jpeg, "%s: JPEG files differ" % k
    print("NV12 annotate loop (detect_and_estimate_frames, BGR frames, draw_heads full, encode_jpeg), 1080p:")
    report(res, "nv12 loop", timed_rounds(arms, check_loop, a.iters, a.rounds), N_FRAMES)
    m.close()
    wn.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
