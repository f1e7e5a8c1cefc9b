"""JPEG encoding of device frames: video.encode_jpeg against download + cv2.imencode per frame, on 8 synthetic annotated 1080p
frames (a gradient plus noise, 20 heads each drawn with draw_heads(display="full")), the two arms alternating and checked
byte-equal on every repetition; then the chain detect_and_estimate_frames + draw_heads + encode_jpeg against
detect_and_estimate_frames + draw_heads.  Prints the card it ran on.  Usage: python tools/jpeg_bench.py [quality]"""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT]


def main(quality=95, reps=20):
    import cv2
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline, video
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
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
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 95)
