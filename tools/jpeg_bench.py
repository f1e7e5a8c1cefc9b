"""JPEG encoding of device frames: video.encode_jpeg against download + cv2.imencode per frame, on 8 synthetic annotated 1080p
frames (a gradient plus noise, 20 heads each drawn with draw_heads(display="full")), the two arms alternating and checked
byte-equal on every repetition; then the chain detect_and_estimate_frames + draw_heads + encode_jpeg against
detect_and_estimate_frames + draw_heads.  Prints the card it ran on.  Usage: python tools/jpeg_bench.py [quality]

``python tools/jpeg_bench.py --options [quality]`` times the option sets of DESIGN.md section 8.11 instead (default, 4:4:4,
optimised tables, a restart interval of one MCU row, 4:4:4 + optimised; progressive alone and at 4:4:4, section 8.12), each against download + cv2.imencode with the same
parameters on the same frames, arms alternating and checked byte-equal every repetition; then, with torch.profiler, the
kernel time of the optimised path's histogram and table build and of each progressive kernel.  ``--default-only`` prints one JSON line with the default
path's per-frame time (for comparing two builds)."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT]


def annotated_frames(wn, n=8, H=1080, W=1920):
    """The benchmark's frames: a gradient plus noise with 20 heads each drawn with draw_heads(display="full"), on the device."""
    import torch
    from whenet_b200 import overlay
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([xx * 255 // W, yy * 255 // H, (xx + yy) * 255 // (H + W)], -1)
    frames = np.clip(base[None] + rng.integers(-8, 9, (n, H, W, 3)), 0, 255).astype(np.uint8)
    res = []
    for _ in range(n):
        y0, x0 = rng.uniform(40, H - 160, 20), rng.uniform(0, W - 160, 20)
        s = rng.uniform(40, 160, 20)
        b = np.stack([y0, x0, y0 + s, x0 + s * 0.8], 1).astype(np.float32)
        res.append((b, np.ones(20, np.float32), rng.uniform(-90, 90, (20, 3)).astype(np.float32)))
    dev = torch.from_numpy(frames).cuda()
    overlay.draw_heads(wn, dev, res, display="full")
    torch.cuda.synchronize()
    return dev


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def cv2_params(quality, sampling="420", restart_interval=0, optimize=False, progressive=False):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)]
    if restart_interval:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart_interval]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if progressive:
        p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    return p


def options(quality=95, reps=20):
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import video
    print(card())
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=32)
    dev = annotated_frames(wn)
    n = dev.shape[0]
    sets = [("default", {}), ("444", dict(sampling="444")), ("optimize", dict(optimize=True)),
            ("restart 1 MCU row", dict(restart_interval=(1920 + 15) // 16)), ("444 + optimize", dict(sampling="444", optimize=True)),
            ("progressive", dict(progressive=True)), ("444 + progressive", dict(sampling="444", progressive=True))]
    times = {name: ([], []) for name, _ in sets}
    sizes = {}
    for r in range(reps + 2):
        for name, kw in sets:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = video.encode_jpeg(wn, dev, quality, **kw)
            t1 = time.perf_counter()
            host = dev.cpu().numpy()
            ref = [cv2.imencode(".jpg", host[f], cv2_params(quality, **kw))[1].tobytes() for f in range(n)]
            t2 = time.perf_counter()
            assert got == ref, "encode_jpeg(%s) differs from cv2.imencode" % name
            sizes[name] = sum(len(g) for g in got) / n
            if r >= 2:
                times[name][0].append(t1 - t0); times[name][1].append(t2 - t1)
    print("quality %d, %d x 1920x1080 annotated frames, median of %d calls, bytes equal to cv2 every time" % (quality, n, reps))
    print("%-20s %10s %12s %16s %9s" % ("options", "bytes", "encode_jpeg", "download+cv2", "speed-up"))
    for name, _ in sets:
        g, h = np.median(times[name][0]) * 1e3 / n, np.median(times[name][1]) * 1e3 / n
        print("%-20s %10d %9.3f ms %13.3f ms %8.1fx" % (name, sizes[name], g, h, h / g))

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            video.encode_jpeg(wn, dev, quality, optimize=True)
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if "jpeg" in e.key:
            per[e.key] = e.device_time_total / 10 / n / 1e3
    total = sum(per.values())
    print("optimize=True kernels, ms per frame (torch.profiler, 10 calls of %d frames):" % n)
    for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
        print("  %8.4f  %s" % (v, k[:100]))
    opt = sum(v for k, v in per.items() if "code_kernel<2" in k or "huff_build" in k)
    print("  histogram + table build: %.4f ms per frame of %.4f ms of kernels" % (opt, total))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            video.encode_jpeg(wn, dev, quality, progressive=True)
        torch.cuda.synchronize()
    per = {e.key: e.device_time_total / 10 / n / 1e3 for e in prof.key_averages() if "jpeg" in e.key}
    print("progressive=True kernels, ms per frame (torch.profiler, 10 calls of %d frames):" % n)
    for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
        print("  %8.4f  %s" % (v, k[:100]))
    print("  total %.4f ms per frame of kernels" % sum(per.values()))


def default_only(quality=95, reps=20):
    import json
    import torch
    import whenet_b200
    from whenet_b200 import video
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=32)
    dev = annotated_frames(wn)
    n = dev.shape[0]
    t = []
    for r in range(reps + 3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        video.encode_jpeg(wn, dev, quality)
        if r >= 3:
            t.append(time.perf_counter() - t0)
    print(json.dumps({"card": card(), "encode_ms_per_frame": float(np.median(t) * 1e3 / n)}))


def main(quality=95, reps=20):
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    print(card())
    n, H, W = 8, 1080, 1920
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([xx * 255 // W, yy * 255 // H, (xx + yy) * 255 // (H + W)], -1)
    frames = np.clip(base[None] + rng.integers(-8, 9, (n, H, W, 3)), 0, 255).astype(np.uint8)
    res = []
    for _ in range(n):
        y0, x0 = rng.uniform(40, H - 160, 20), rng.uniform(0, W - 160, 20)
        s = rng.uniform(40, 160, 20)
        b = np.stack([y0, x0, y0 + s, x0 + s * 0.8], 1).astype(np.float32)
        res.append((b, np.ones(20, np.float32), rng.uniform(-90, 90, (20, 3)).astype(np.float32)))
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=32)
    dev = torch.from_numpy(frames).cuda()
    overlay.draw_heads(wn, dev, res, display="full")
    torch.cuda.synchronize()

    t_gpu, t_host, nbytes = [], [], 0
    for r in range(reps + 2):
        t0 = time.perf_counter()
        got = video.encode_jpeg(wn, dev, quality)
        t1 = time.perf_counter()
        host = dev.cpu().numpy()
        ref = [cv2.imencode(".jpg", host[f], [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes() for f in range(n)]
        t2 = time.perf_counter()
        assert got == ref, "encode_jpeg differs from cv2.imencode"
        nbytes = sum(len(g) for g in got)
        if r >= 2:
            t_gpu.append(t1 - t0); t_host.append(t2 - t1)
    g, h = np.median(t_gpu) * 1e3 / n, np.median(t_host) * 1e3 / n
    print("quality %d, %d x %dx%d frames, %.2f MB of JPEG per frame" % (quality, n, W, H, nbytes / n / 1e6))
    print("encode_jpeg          %.3f ms per frame (median of %d calls of %d frames, bytes equal to cv2 every time)" % (g, reps, n))
    print("download+imencode    %.3f ms per frame" % h)
    print("speed-up             %.1fx%s" % (h / g, "" if h / g >= 10 else "  (below the 10x aim)"))

    yolo = whenet_b200.YOLO(None, max_frames=8)
    for _ in range(3):
        overlay.draw_heads(wn, dev, pipeline.detect_and_estimate_frames(yolo, wn, dev), display="full")
        video.encode_jpeg(wn, dev, quality)
    a, b = [], []
    for r in range(reps):
        t0 = time.perf_counter()
        out = pipeline.detect_and_estimate_frames(yolo, wn, dev)
        overlay.draw_heads(wn, dev, out, display="full")
        t1 = time.perf_counter()
        out = pipeline.detect_and_estimate_frames(yolo, wn, dev)
        overlay.draw_heads(wn, dev, out, display="full")
        video.encode_jpeg(wn, dev, quality)
        t2 = time.perf_counter()
        a.append(t1 - t0); b.append(t2 - t1)
    print("chain detect+estimate+draw          %.3f ms per frame" % (np.median(a) * 1e3 / n))
    print("chain detect+estimate+draw+encode   %.3f ms per frame" % (np.median(b) * 1e3 / n))


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    q = int(args[0]) if args else 95
    if "--options" in sys.argv:
        options(q)
    elif "--default-only" in sys.argv:
        default_only(q)
    else:
        main(q)
