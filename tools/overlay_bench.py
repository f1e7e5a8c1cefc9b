"""Head overlay on device frames: overlay.draw_heads against download + reference-typed cv2 drawing + upload, on 8
synthetic 1080p frames with about 20 heads each, the two arms alternating and checked bit-equal; the same with
display="full" (labels, DESIGN.md section 8.8): draw_heads(display="full"), display="simple" and the host round trip with
the labels, alternating, full checked bit-equal to the host; then the chain detect_and_estimate_frames + draw_heads against
detect_and_estimate_frames alone.  Prints the card it ran on."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]


def main(reps=20):
    import torch
    import whenet_b200
    from whenet_b200 import overlay, pipeline
    import cv2
    import overlay_oracle as O

    def ref_draw(img, box, ang):
        """process_detection_ref's drawing calls (every bench head is valid and has finite angles)"""
        y_min, x_min, y_max, x_max = box
        y_min = max(0, y_min - abs(y_min - y_max) / 10)
        y_max = min(H, y_max + abs(y_min - y_max) / 10)
        x_min = max(0, x_min - abs(x_min - x_max) / 5)
        x_max = min(W, x_max + abs(x_min - x_max) / 5)
        cv2.rectangle(img, (int(x_min), int(y_min)), (int(x_max), int(y_max)), (0, 0, 0), 2)
        O.draw_axis_ref(img, ang[0], ang[1], ang[2], tdx=(x_min + x_max) / 2, tdy=(y_min + y_max) / 2, size=abs(x_max - x_min) // 2)
        return int(x_min), int(y_min)

    def ref_draw_full(img, box, ang):
        x, y = ref_draw(img, box, ang)
        for k, name in enumerate(("yaw", "pitch", "roll")):
            cv2.putText(img, "%s: {}".format(np.round(ang[k])) % name, (x, y - 15 * k), cv2.FONT_HERSHEY_SIMPLEX, 0.4, (100, 255, 0), 1)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    n, H, W = 8, 1080, 1920
    rng = np.random.default_rng(0)
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    res = []
    for _ in range(n):
        y0, x0 = rng.uniform(0, H - 120, 20), rng.uniform(0, W - 120, 20)
        s = rng.uniform(40, 160, 20)
        b = np.stack([y0, x0, y0 + s, x0 + s * 0.8], 1).astype(np.float32)
        res.append((b, np.ones(20, np.float32), rng.uniform(-90, 90, (20, 3)).astype(np.float32)))
    wn = whenet_b200.WHENet(None, device=0, precision="bf16", max_batch=32)
    dev = torch.from_numpy(frames).cuda()

    t_gpu, t_host = [], []
    for r in range(reps + 2):
        dev.copy_(torch.from_numpy(frames)); torch.cuda.synchronize()
        t0 = time.perf_counter(); overlay.draw_heads(wn, dev, res); t1 = time.perf_counter()
        got = dev.cpu().numpy()
        dev.copy_(torch.from_numpy(frames)); torch.cuda.synchronize()
        t2 = time.perf_counter()
        host = dev.cpu().numpy()
        for f in range(n):
            for i in range(20):
                ref_draw(host[f], res[f][0][i], res[f][2][i])
        dev.copy_(torch.from_numpy(host)); torch.cuda.synchronize()
        t3 = time.perf_counter()
        assert np.array_equal(got, host)
        if r >= 2:
            t_gpu.append(t1 - t0); t_host.append(t3 - t2)
    print("draw_heads        %.3f ms per frame (median of %d calls of %d frames)" % (np.median(t_gpu) * 1e3 / n, reps, n))
    print("download+cv2+up   %.3f ms per frame" % (np.median(t_host) * 1e3 / n))

    t_full, t_simple, t_hfull = [], [], []
    for r in range(reps + 2):
        dev.copy_(torch.from_numpy(frames)); torch.cuda.synchronize()
        t0 = time.perf_counter(); overlay.draw_heads(wn, dev, res, display="full"); t1 = time.perf_counter()
        got = dev.cpu().numpy()
        dev.copy_(torch.from_numpy(frames)); torch.cuda.synchronize()
        t2 = time.perf_counter(); overlay.draw_heads(wn, dev, res, display="simple"); t3 = time.perf_counter()
        dev.copy_(torch.from_numpy(frames)); torch.cuda.synchronize()
        t4 = time.perf_counter()
        host = dev.cpu().numpy()
        for f in range(n):
            for i in range(20):
                ref_draw_full(host[f], res[f][0][i], res[f][2][i])
        dev.copy_(torch.from_numpy(host)); torch.cuda.synchronize()
        t5 = time.perf_counter()
        assert np.array_equal(got, host)
        if r >= 2:
            t_full.append(t1 - t0); t_simple.append(t3 - t2); t_hfull.append(t5 - t4)
    print("draw_heads full   %.3f ms per frame" % (np.median(t_full) * 1e3 / n))
    print("draw_heads simple %.3f ms per frame" % (np.median(t_simple) * 1e3 / n))
    print("download+cv2 full+up %.3f ms per frame" % (np.median(t_hfull) * 1e3 / n))
    yolo = whenet_b200.YOLO(None, max_frames=8)
    for _ in range(3):
        pipeline.detect_and_estimate_frames(yolo, wn, dev)
    a, b = [], []
    for r in range(reps):
        t0 = time.perf_counter(); pipeline.detect_and_estimate_frames(yolo, wn, dev); t1 = time.perf_counter()
        out = pipeline.detect_and_estimate_frames(yolo, wn, dev)
        overlay.draw_heads(wn, dev, out)
        t2 = time.perf_counter()
        a.append(t1 - t0); b.append(t2 - t1)
    print("chain detect+estimate        %.3f ms per frame" % (np.median(a) * 1e3 / n))
    print("chain detect+estimate+draw   %.3f ms per frame (%d heads drawn per call)" % (np.median(b) * 1e3 / n,
                                                                                     sum(int(d.sum()) for d in overlay.draw_heads(wn, dev, out))))


if __name__ == "__main__":
    main()
