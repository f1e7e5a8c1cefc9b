#!/usr/bin/env python
"""bench.py - WHENet per-crop forward throughput on H100 (see DESIGN.md).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--batch B] [--precision bf16] [--impl ours|reference] [--dump-outputs DIR]

A "step" is one pass of the hot path (reference whenet.py:22-34) over one batch of B synthetic
224x224x3 uint8 crops per GPU (default B=512: BASELINE.json configs[2]; at N GPUs the global batch
is N*B = configs[3] for N=8), followed - when N>1 - by the all-gather of the angles.

value  : crops/s, inputs already resident in HBM, CUDA events on the launching stream, max over ranks
e2e    : crops/s through WHENet.forward_host(): pinned host uint8 in, H2D + forward + D2H of the angles
         inside the timed region
roofline: dominant kernel family (per-kernel CUDA events recorded inside the library on its stream)
cpu_baseline: the torch-CPU port of the oracle on this box's host cores, bounded sample
--impl reference: the CPU port timed through the same surface (the reference's Keras/TF-1.12 stack
         cannot be installed: requirements.txt:3-5 pins are Python<=3.6 era and absent offline)
--dump-outputs DIR: after the timed steps, DIR/angles.npy holds the [B, 3] float32 angles (yaw, pitch, roll) of the last
         timed step; the inputs are seeded, so two builds run with the same arguments can be compared output for output
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

ALGO_ELEMS_PER_CROP = 6_938_112      # activation elements moved by the <=2-kernels-per-block plan (SURVEY.md 8d)
FLOP_PER_CROP = 2 * 389_533_088      # SURVEY.md 8a
IMG_BYTES = 224 * 224 * 3
METRIC = "head-crops/sec @224x224 bf16"   # BASELINE.json's metric; BOTH arms print this exact string (dtype says what ran)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return {"hbm_gbs": float(d["hbm_gbs"]), "bf16_tflops": float(d.get("bf16_tflops_sustained", d["bf16_tflops"])),
                "source": "measured (MEASURED_PEAKS.json; sustained bf16)"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet (dense bf16, HBM3), not measured"}


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag, self.proc = index, [], False, None

    def run(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                if self.stop_flag:
                    break
                self.rows.append([c.strip() for c in line.split(",")])
        except Exception:
            pass

    def finish(self):
        self.stop_flag = True
        if self.proc:
            self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 2 + i and r[2 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


def cpu_port(threads=None):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from whenet_oracle import TorchCpuPort
    import whenet_b200
    names, w = whenet_b200.weights.load_snapshot(whenet_b200.weights.DEFAULT_NPZ)
    return TorchCpuPort(names, w, threads=threads)


def best_cpu_port(sample_crops):
    """torch-CPU conv kernels on tiny per-layer work get SLOWER with too many threads (128-core hosts);
    probe a few thread counts and keep the fastest, so the baseline is the strongest one.  Each candidate is scored by
    the MEDIAN of five 8-crop calls after a warm-up call (a single timing picked 8 vs 16 threads at random in round 1)."""
    import torch
    cores = os.cpu_count() or 1
    port = cpu_port(threads=cores)
    best = (None, 0.0)
    probe = {}
    for th in sorted({cores, min(cores, 64), min(cores, 32), min(cores, 16), min(cores, 8)}, reverse=True):
        torch.set_num_threads(th)
        port.get_angle(sample_crops[:8])
        ts = []
        for _ in range(5):
            t = time.perf_counter()
            port.get_angle(sample_crops[:8])
            ts.append(time.perf_counter() - t)
        rate = 8 / statistics.median(ts)
        probe[th] = round(rate, 1)
        if rate > best[1]:
            best = (th, rate)
    torch.set_num_threads(best[0])
    port.thread_probe = probe
    return port, best[0]


def time_cpu(port, crops, reps):
    port.get_angle(crops[:8])
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        port.get_angle(crops)
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def run_reference(args):
    """The reference arm: CPU port of whenet.py:22-34 (batch_size=8 chunking) on all host cores."""
    import torch
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    sample = 32                                    # crops per step: a bounded sample of the B-crop batch
    rng = np.random.default_rng(0)
    crops = rng.integers(0, 256, (sample, 224, 224, 3), dtype=np.uint8)
    port, _th = best_cpu_port(crops)
    for _ in range(max(args.warmup, 1)):
        port.get_angle(crops)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        port.get_angle(crops)
    dt = time.perf_counter() - t0
    v = sample * args.steps / dt
    line = {"impl": "reference", "metric": METRIC, "value": v, "unit": "crops/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": "batch=%d synthetic 224x224x3 uint8 crops per GPU (configs[2]); CPU arm times a %d-crop "
                                   "sample per step" % (args.batch, sample)},
            "cpu_baseline": {"value": v, "unit": "crops/s", "cores": torch.get_num_threads(), "kind": "port",
                             "sample": "%d crops/step x %d steps, torch-CPU fp32 port of the oracle (Keras/TF-1.12 not installable); thread probe crops/s %s"
                                       % (sample, args.steps, getattr(port, "thread_probe", {}))},
            "e2e": {"value": v, "unit": "crops/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=512, help="crops per GPU per step")
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg")
    ap.add_argument("--chunk", type=int, default=0)
    ap.add_argument("--opt", action="append", default=[], help="library option key=value (repeatable)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the angles of the last timed step to DIR/angles.npy (float32)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)

    import torch
    import torch.distributed as dist
    import whenet_b200

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run --nproc-per-node %d" % args.gpus)
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B, K, W = args.batch, args.steps, max(args.warmup, 3)

    net = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=local, precision=args.precision, max_batch=B)
    net.set_option("chunk", args.chunk if args.chunk else B)      # one pass per step: every layer sees the whole batch
    for kv in args.opt:
        k, v = kv.split("=")
        net.set_option(k, int(v))
    # ---- self-check before timing anything: the configuration being measured (fused tensor-core kernels, two streams) must
    #      agree with the plain CUDA-core kernel family on the committed Sample/jitter crops.  A fast wrong kernel is
    #      not a result; the oracle comparison proper lives in tests/ and __graft_entry__.smoke().
    chk = np.concatenate([np.load(os.path.join(ROOT, "tests", "golden", "sample_crops.npy")),
                          np.load(os.path.join(ROOT, "tests", "golden", "jitter_crops.npy"))] * 8)
    got = np.stack(net.get_angle(chk), axis=1)
    net.set_option("fused", 0); net.set_option("tensor_cores", 0); net.set_option("streams", 1)
    ref = np.stack(net.get_angle(chk), axis=1)
    net.set_option("fused", 1); net.set_option("tensor_cores", 0 if args.precision == "fp32" else 1); net.set_option("streams", 2)
    for kv in args.opt:                                           # the self-check reset three switches: re-apply the overrides
        k, v = kv.split("=")
        net.set_option(k, int(v))
    tol = 0.02 if args.precision == "fp32" else (1.5 if args.precision == "bf16" else 0.3)
    self_check = float(np.abs(got - ref).max())
    if not (self_check <= tol):
        raise SystemExit("bench self-check failed: measured configuration differs from the CUDA-core path by %.3f deg" % self_check)

    stream = torch.cuda.Stream()          # a real (non-default) stream shared by the library, NCCL and the timing events
    torch.cuda.set_stream(stream)
    net.set_stream(stream.cuda_stream)

    # ---- synthetic inputs: NBUF different resident batches rotate so inputs are never L2-hot (NBUF*B*150 KB > 50 MB)
    NBUF = max(2, -(-(160 << 20) // (B * IMG_BYTES)))
    g = torch.Generator(device="cuda").manual_seed(1000 + rank)
    dev_in = [torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(NBUF)]
    angles = torch.empty((B, 3), dtype=torch.float32, device="cuda")
    gathered = torch.empty((world * B, 3), dtype=torch.float32, device="cuda") if world > 1 else None

    def step(i):
        net.forward_device(dev_in[i % NBUF], angles)
        if world > 1:
            dist.all_gather_into_tensor(gathered, angles)

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    for i in range(W):
        step(i)
    sync_all()
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
        time.sleep(0.3)
    l0 = net.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync_all()
    e0.record(stream)
    for i in range(K):
        step(W + i)
    e1.record(stream)
    sync_all()
    net.synchronize()          # also surfaces an mbarrier timeout of any kernel of the timed loop (raises)
    ms = e0.elapsed_time(e1)
    launches = net.launch_count() - l0
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "angles.npy"), angles.float().cpu().numpy())
    clocks = sampler.finish() if sampler else None
    t = torch.tensor([ms], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_max = float(t.item())
    value = world * B * K / (ms_max * 1e-3)

    # ---- e2e: pinned host uint8 -> H2D -> forward (-> all-gather) -> D2H of the angles, through the public API.
    #      Every step copies its own input up and its own result down inside the timed region; as a serving loop
    #      would, two steps are kept in flight (double-buffered pinned buffers) so step i+1 uploads while step i computes.
    h_in = [torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    h_out = [torch.empty((world * B, 3), dtype=torch.float32).pin_memory() for _ in range(2)]
    d_ang = [torch.empty((B, 3), dtype=torch.float32, device="cuda") for _ in range(2)]
    d_gat = [torch.empty((world * B, 3), dtype=torch.float32, device="cuda") for _ in range(2)] if world > 1 else d_ang
    done = [None, None]

    def e2e_step(i):
        s = i & 1
        if done[s] is not None:
            done[s].synchronize()                       # buffers of step i-2 are free again
        net.forward_host_to_device(h_in[s], d_ang[s])
        if world > 1:
            dist.all_gather_into_tensor(d_gat[s], d_ang[s])
        h_out[s].copy_(d_gat[s], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(stream)
        done[s] = ev

    KE = max(6, K // 2)
    for i in range(4):
        e2e_step(i)
    sync_all()
    e0.record(stream)
    for i in range(KE):
        e2e_step(i)
    e1.record(stream)
    sync_all()
    net.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_value = world * B * KE / (float(t.item()) * 1e-3)

    # ---- e2e through the reference's own call: WHENet.get_angle(np.ndarray) with a PAGEABLE uint8 array (what
    #      demo.py:12-14 / demo_video.py:24-28 pass), synchronous, wall clock, returns three fresh numpy arrays
    np_in = [h.numpy().copy() for h in h_in]
    for i in range(2):
        net.get_angle(np_in[i & 1])
    sync_all()
    KG = max(4, K // 4)
    t0 = time.perf_counter()
    for i in range(KG):
        net.get_angle(np_in[i & 1])
    dt_ga = time.perf_counter() - t0
    tg = torch.tensor([dt_ga], device="cuda")
    if world > 1:
        dist.all_reduce(tg, op=dist.ReduceOp.MAX)
    e2e_get_angle = world * B * KG / float(tg.item())

    # ---- per-kernel CUDA-event profile (recorded inside the library on the launching stream)
    # the per-kernel table is taken with the two half-batch streams serialised (streams=1): with both streams active
    # every kernel's event pair also spans the kernels it shares the GPU with and the per-kernel GB/s would be meaningless
    net.set_option("streams", 1)
    for i in range(2):
        net.forward_device(dev_in[i % NBUF], angles)
    net.enable_profile(True)
    KP = min(K, 10)
    for i in range(KP):
        net.forward_device(dev_in[i % NBUF], angles)
    torch.cuda.synchronize()
    stats = net.read_profile()
    net.enable_profile(False)
    net.set_option("streams", 2)

    if rank == 0:
        pk = peaks()
        fam = {}
        for s in stats:
            nm = s["name"]
            f = "pw_conv(1x1)" if (nm.endswith(".expand") or nm.endswith(".project") or nm == "head.conv") else \
                "k1_expand_dw(fused)" if nm.endswith(".k1") else \
                "kd_dw_se(late blocks)" if nm.endswith(".kd") else \
                "dw_conv" if nm.endswith(".dw") else "se_gate" if nm.endswith(".se") else nm
            a = fam.setdefault(f, {"ms": 0.0, "bytes": 0.0, "flops": 0.0, "launches": 0})
            for k in ("ms", "bytes", "flops", "launches"):
                a[k] += s[k]
        tot_ms = sum(a["ms"] for a in fam.values())
        dom = max(fam.items(), key=lambda kv: kv[1]["ms"])
        dname, d = dom
        achieved = d["bytes"] / (d["ms"] * 1e-3) / 1e9
        es = 4 if args.precision == "fp32" else 2
        roof = {"kernel": dname, "bound": "hbm", "achieved": achieved, "peak": pk["hbm_gbs"], "unit": "GB/s",
                "frac": achieved / pk["hbm_gbs"], "peak_source": pk["source"],
                "share_of_step": d["ms"] / tot_ms, "launches_per_step": d["launches"] / KP,
                "per_kernel_note": "kernel table measured with streams=1 (%.3f ms/step serialised); the timed `value` runs the default "
                                   "two-stream mode, where the halves overlap" % (tot_ms / KP),
                "ms_per_launch_avg": d["ms"] / d["launches"],
                "tflops": d["flops"] / (d["ms"] * 1e-3) / 1e12,
                "families": {k: {"ms_per_step": v["ms"] / KP, "GBps": v["bytes"] / (v["ms"] * 1e-3) / 1e9,
                                 "TFLOPs": v["flops"] / (v["ms"] * 1e-3) / 1e12} for k, v in fam.items()},
                "whole_net": {"algorithmic_bytes_per_crop": ALGO_ELEMS_PER_CROP * es,
                              "achieved_GBps": ALGO_ELEMS_PER_CROP * es * value / world / 1e9,
                              "frac_of_hbm_peak": ALGO_ELEMS_PER_CROP * es * value / world / 1e9 / pk["hbm_gbs"],
                              "achieved_TFLOPs": FLOP_PER_CROP * value / world / 1e12}}
        cpu = None
        if not args.no_cpu and world == 1:
            import torch as _t
            sample = 32
            crops = np.random.default_rng(0).integers(0, 256, (sample, 224, 224, 3), dtype=np.uint8)
            port, _th = best_cpu_port(crops)
            dt = time_cpu(port, crops, 3)
            cpu = {"value": sample / dt, "unit": "crops/s", "cores": _t.get_num_threads(), "kind": "port",
                   "sample": "%d crops, median of 3, best thread count of a probe over {all,64,32,16,8}, torch-CPU fp32 port of the oracle with the reference's batch_size=8 chunking "
                             "(Keras/TF-1.12 not installable)" % sample}
        line = {"metric": METRIC, "value": value, "unit": "crops/s", "n_gpus": world,
                "steps": K, "warmup": W, "ms_per_step": ms_max / K, "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": args.precision, "data": "synthetic",
                "config": {"workload": "batch=%d synthetic 224x224x3 uint8 crops per GPU (BASELINE configs[2]; global batch %d%s)"
                                       % (B, world * B, ", NCCL all-gather of angles" if world > 1 else ""),
                           "global_batch": world * B, "parallelism": "dp%d" % world, "weights": "WHENet.h5 (converted npz)",
                           "l2": "inputs rotate over %d resident batches (%d MB > 50 MB L2)" % (NBUF, NBUF * B * IMG_BYTES >> 20)},
                "clocks": clocks,
                "e2e": {"value": e2e_value, "unit": "crops/s", "h2d_bytes_per_step": B * IMG_BYTES, "d2h_bytes_per_step": B * 12,
                        "api": "WHENet.forward_host_to_device + D2H of the angles, two steps in flight (pinned uint8 in, pinned angles out)",
                        "get_angle_value": e2e_get_angle,
                        "get_angle_api": "WHENet.get_angle(np.ndarray): pageable uint8 in, synchronous, numpy out (reference whenet.py:22-34 call shape), wall clock"},
                "gpu_launches": int(launches * world),
                "self_check_max_deg_vs_simt_path": self_check,
                "roofline": roof, "cpu_baseline": cpu}
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
