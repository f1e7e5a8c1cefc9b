#!/usr/bin/env python
"""Per-layer time of the fused expand + depthwise kernels of blocks 2-6 (profile rows bNN.k1), for both routes in one process:

  python tools/k1_profile.py [--batch 512] [--steps 20]

k1x=0 is K1 (k1_expand_dw_kernel), k1x=1 its TMA-fed sibling (k1x_kernel).  Times are CUDA events recorded inside the library
around each launch, one stream (streams=1, as bench.py's kernel table); GB/s is over the layer's algorithmic bytes (block
input + depthwise output).  The card and its power limit are printed with the table: the numbers mean nothing without them.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def profile(net, ins, ang, steps):
    for i in range(3):
        net.forward_device(ins[i % len(ins)], ang)
    net.enable_profile(True)
    for i in range(steps):
        net.forward_device(ins[i % len(ins)], ang)
    net.synchronize()
    rows = {s["name"]: s for s in net.read_profile() if s["name"].endswith(".k1")}
    net.enable_profile(False)
    return {k: (v["ms"] / steps, v["bytes"] / v["ms"] / 1e6) for k, v in rows.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import whenet_b200
    if not torch.cuda.is_available():
        raise SystemExit("k1_profile needs a GPU")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    B = args.batch
    net = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=B)
    net.set_option("chunk", B)
    net.set_option("streams", 1)
    g = torch.Generator(device="cuda").manual_seed(1000)
    ins = [torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(3)]
    ang = torch.empty((B, 3), dtype=torch.float32, device="cuda")
    res = {}
    for route in (0, 1, 0, 1):                       # alternated: the second pair shows the run-to-run spread
        net.set_option("k1x", route)
        res.setdefault(route, []).append(profile(net, ins, ang, args.steps))
    print("%d crops, one stream; ms per step (GB/s on algorithmic bytes), two runs per route" % B)
    print("%-8s %-32s %-32s" % ("layer", "k1x=0", "k1x=1"))
    tot = {0: [0.0, 0.0], 1: [0.0, 0.0]}
    for name in sorted(res[0][0]):
        cells = []
        for route in (0, 1):
            cells.append("  ".join("%.4f (%4.0f)" % res[route][i][name] for i in range(2)))
            for i in range(2):
                tot[route][i] += res[route][i][name][0]
        print("%-8s %-32s %-32s" % (name, cells[0], cells[1]))
    print("%-8s %-32s %-32s" % ("sum", "  ".join("%.4f       " % t for t in tot[0]), "  ".join("%.4f       " % t for t in tot[1])))
    net.close()


if __name__ == "__main__":
    main()
