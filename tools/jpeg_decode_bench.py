"""JPEG decoding on the GPU: video.decode_jpeg against cv2.imdecode + upload per frame, on 8 synthetic annotated 1080p frames
encoded at quality 95 (as tools/jpeg_bench.py makes them), the two arms alternating and checked equal on every repetition;
then the whole MJPG AVI -> annotated AVI loop (read, decode, detect + estimate, draw, encode, write) with GPU decoding against
the same loop with cv2.imdecode + upload.  Prints the card it ran on.  Usage: python tools/jpeg_decode_bench.py [reps]"""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT]


def main(reps=20):
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
    files = video.encode_jpeg(wn, dev, 95)
    torch.cuda.synchronize()

    t_gpu, t_host = [], []
    for r in range(reps + 2):
        t0 = time.perf_counter()
        got = video.decode_jpeg(wn, files)
        t1 = time.perf_counter()
        ref = [torch.from_numpy(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)).cuda() for f in files]
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), "decode_jpeg differs from cv2.imdecode"
        if r >= 2:
            t_gpu.append(t1 - t0); t_host.append(t2 - t1)
    g, h = np.median(t_gpu) * 1e3 / n, np.median(t_host) * 1e3 / n
    print("quality 95, %d x %dx%d frames, %.2f MB of JPEG per frame" % (n, W, H, sum(map(len, files)) / n / 1e6))
    print("decode_jpeg          %.3f ms per frame (median of %d calls of %d files, equal to cv2 every time)" % (g, reps, n))
    print("imdecode+upload      %.3f ms per frame" % h)
    print("speed-up             %.1fx%s" % (h / g, "" if h / g >= 10 else "  (below the 10x aim)"))

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        video.decode_jpeg(wn, files)
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=14))

    yolo = whenet_b200.YOLO(None, max_frames=8)
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "src.avi")
        with video.MJPGWriter(src, 25, (W, H)) as w:
            for _ in range(4):
                w.write(files)

        def loop(gpu):
            t0 = time.perf_counter()
            with video.MJPGReader(src) as r, video.MJPGWriter(os.path.join(tmp, "dst.avi"), r.fps, r.frame_size) as w:
                while True:
                    if gpu:
                        batch = r.read_frames(wn, 8)
                        if batch is None:
                            break
                    else:
                        chunk = r.read(8)
                        if not chunk:
                            break
                        batch = torch.from_numpy(np.stack([cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) for f in chunk])).cuda()
                    out = pipeline.detect_and_estimate_frames(yolo, wn, batch)
                    overlay.draw_heads(wn, batch, out, display="full")
                    w.write(video.encode_jpeg(wn, batch))
                k = len(r)
            return (time.perf_counter() - t0) * 1e3 / k

        loop(True); loop(False)
        a = [loop(True) for _ in range(3)]
        b = [loop(False) for _ in range(3)]
    print("AVI loop, GPU decode     %.3f ms per frame" % np.median(a))
    print("AVI loop, host decode    %.3f ms per frame" % np.median(b))


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 20)
