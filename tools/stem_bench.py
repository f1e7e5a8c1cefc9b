#!/usr/bin/env python
"""Time of the stem alone (profile row ``stem``), bf16 route, one stream, device-resident uint8 crops:

  python tools/stem_bench.py [--batch 512] [--steps 20]

Times are CUDA events recorded inside the library around each stem launch (streams=1, as bench.py's kernel table).  The
achieved FFMA rate and GB/s are over the algorithmic work (27 x 32 FFMA per output pixel; uint8 in, fp16 out), set against
the two floors computed from the H100 SXM data sheet: 128 FFMA/clk/SM at the card's max SM clock, and 3.35 TB/s HBM3.
The card, its power limit and max SM clock are read in the same process: the numbers mean nothing without them.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import whenet_b200
    if not torch.cuda.is_available():
        raise SystemExit("stem_bench needs a GPU")
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                          capture_output=True, text=True).stdout.strip()
    name, power, max_mhz = [s.strip() for s in card.split(",")]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = args.batch
    net = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision="bf16", max_batch=B)
    net.set_option("chunk", B)
    net.set_option("streams", 1)
    g = torch.Generator(device="cuda").manual_seed(1000)
    ins = [torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(3)]
    ang = torch.empty((B, 3), dtype=torch.float32, device="cuda")
    for i in range(3):
        net.forward_device(ins[i % len(ins)], ang)
    net.enable_profile(True)
    for i in range(args.steps):
        net.forward_device(ins[i % len(ins)], ang)
    net.synchronize()
    row = next(s for s in net.read_profile() if s["name"] == "stem")
    net.enable_profile(False)
    net.close()
    ms = row["ms"] / args.steps
    ffma = B * 112 * 112 * 27 * 32
    nbytes = B * (224 * 224 * 3 + 112 * 112 * 32 * 2)
    ffma_peak = 128 * sms * float(max_mhz) * 1e6
    print("%s, power limit %s W, max SM clock %s MHz, %d SMs" % (name, power, max_mhz, sms))
    print("stem, %d crops, one stream, %d passes: %.4f ms per pass" % (B, args.steps, ms))
    print("  FFMA: %.2f TFFMA/s achieved; floor %.4f ms (%.2f G FFMA at %.2f TFFMA/s)" %
          (ffma / ms / 1e9, ffma / ffma_peak * 1e3, ffma / 1e9, ffma_peak / 1e12))
    print("  HBM : %.0f GB/s achieved; floor %.4f ms (%.0f MB at %.2f TB/s)" %
          (nbytes / ms / 1e6, nbytes / HBM_BPS * 1e3, nbytes / 1e6, HBM_BPS / 1e12))


if __name__ == "__main__":
    main()
