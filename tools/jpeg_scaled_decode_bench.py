"""Reduced and gray JPEG decoding on the GPU (DESIGN.md section 8.13): video.decode_jpeg at d = 1, 2, 4 and 8 in colour and
gray against cv2.imdecode with the matching IMREAD_* flag + upload per frame, on 8 synthetic annotated 1080p frames (as
tools/jpeg_decode_bench.py makes them) and 8 at 2160x3840, quality 95.  All arms alternate within each repetition and every
GPU frame is checked equal to cv2's on every repetition.  Then a torch.profiler split of the GPU decode per mode.  Prints the
card it ran on.  Usage: python tools/jpeg_scaled_decode_bench.py [reps]"""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT]


def frames_at(H, W, n, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([xx * 255 // W, yy * 255 // H, (xx + yy) * 255 // (H + W)], -1)
    frames = np.clip(base[None] + rng.integers(-8, 9, (n, H, W, 3)), 0, 255).astype(np.uint8)
    res = []
    for _ in range(n):
        y0, x0 = rng.uniform(40, H - 160, 20), rng.uniform(0, W - 160, 20)
        s = rng.uniform(40, 160, 20)
        b = np.stack([y0, x0, y0 + s, x0 + s * 0.8], 1).astype(np.float32)
        res.append((b, np.ones(20, np.float32), rng.uniform(-90, 90, (20, 3)).astype(np.float32)))
    return frames, res


def main(reps=10):
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import overlay, video
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    flags = {(1, False): cv2.IMREAD_COLOR, (2, False): cv2.IMREAD_REDUCED_COLOR_2, (4, False): cv2.IMREAD_REDUCED_COLOR_4,
             (8, False): cv2.IMREAD_REDUCED_COLOR_8, (1, True): cv2.IMREAD_GRAYSCALE, (2, True): cv2.IMREAD_REDUCED_GRAYSCALE_2,
             (4, True): cv2.IMREAD_REDUCED_GRAYSCALE_4, (8, True): cv2.IMREAD_REDUCED_GRAYSCALE_8}
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=32)
    for H, W in [(1080, 1920), (2160, 3840)]:
        frames, res = frames_at(H, W, 8, 0)
        dev = torch.from_numpy(frames).cuda()
        overlay.draw_heads(wn, dev, res, display="full")
        files = video.encode_jpeg(wn, dev, 95)
        n = len(files)
        t = {(m, a): [] for m in flags for a in ("gpu", "cv2")}
        for rep in range(reps + 1):
            for m, fl in flags.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = video.decode_jpeg(wn, files, reduce=m[0], gray=m[1])
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                ref = []
                for f in files:
                    r = cv2.imdecode(np.frombuffer(f, np.uint8), fl)
                    ref.append(torch.from_numpy(r[:, :, None] if m[1] else r).cuda())
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                assert all(torch.equal(a, b) for a, b in zip(got, ref)), (H, W, m)
                if rep:
                    t[(m, "gpu")].append((t1 - t0) * 1e3 / n)
                    t[(m, "cv2")].append((t2 - t1) * 1e3 / n)
        full = np.median(t[((1, False), "gpu")])
        print("\n%dx%d, quality 95, %d frames per call, ms per frame (median of %d; min-max)" % (H, W, n, reps))
        print("| d | mode | decode_jpeg | cv2.imdecode + upload | speed-up | vs full-size decode_jpeg |")
        print("|---|---|---|---|---|---|")
        for m in flags:
            g, c = np.array(t[(m, "gpu")]), np.array(t[(m, "cv2")])
            print("| %d | %s | %.3f (%.3f-%.3f) | %.2f | %.0fx | %.2f |" % (m[0], "gray" if m[1] else "colour", np.median(g), g.min(),
                                                                        g.max(), np.median(c), np.median(c) / np.median(g), np.median(g) / full))
        from torch.profiler import ProfilerActivity, profile
        for m in flags:
            video.decode_jpeg(wn, files, reduce=m[0], gray=m[1])
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    video.decode_jpeg(wn, files, reduce=m[0], gray=m[1])
                torch.cuda.synchronize()
            split = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.self_device_time_total > 0:
                    name = e.key.split("<")[0].split("(")[0].replace("void ", "").replace("whenet::jpegdec::", "").replace("whenet::jpeg::", "")
                    split[name] = split.get(name, 0) + e.self_device_time_total / 5 / n
            top = sorted(split.items(), key=lambda kv: -kv[1])
            print("profile d=%d %s: device %.1f us/frame: %s" % (m[0], "gray" if m[1] else "colour", sum(split.values()),
                                                               ", ".join("%s %.1f" % kv for kv in top[:6])))
    wn.close()


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
