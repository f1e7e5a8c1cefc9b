"""Record the GPU work of the WHENet forward, stream by stream, for a list of configurations and batch sizes.

  python tools/launch_trace.py --root DIR --out trace.json

imports ``whenet_b200`` from the package root DIR, so that two trees (say, a change and its parent) can be traced by the same
script and their outputs compared byte for byte.  Each configuration gets a fresh context; at each batch size one warm-up
forward runs, then one forward under torch.profiler with CUDA activities (three captures, keeping the most complete).  For each
stream (numbered by its first launch) the trace lists, in launch order, every kernel as [name, grid, block, shared memory]
(static + dynamic bytes, as CUPTI reports it) and every memcpy / memset as [kind, bytes].  Identical traces mean the same
kernels with the same launch shapes, in the same order on each stream.  A capture that lost records shows up as a stream whose
list is a tail of the complete one.

The batch sizes are the route switches of DESIGN.md section 4.2; the configurations cover every precision, stream count and
forward option whose route the batch size alone does not choose.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

NS = [1, 3, 8, 30, 32, 34, 64, 68, 128, 172, 240, 272, 456, 512]
BF16_OPTIONS = [("kd_from", 0), ("k1x", 0), ("fused", 0), ("pw_variant", 2), ("pw_variant", 3), ("pw3", 0), ("kd_tail", 1),
                ("se_fused", 1), ("se_tail", 0), ("se_scale_out", 0), ("dw1_kd", 0), ("stem_variant", 0), ("dw_variant", 0),
                ("se_wide", 1), ("se_batch", 0), ("head_batch", 0), ("k1_split_ctas", 0)]


def configs():
    """(name, precision, options, taps mode, input kind, batch sizes)"""
    out = [("bf16", "bf16", {}, 0, "device", NS)]
    out += [("bf16_streams%d" % s, "bf16", {"streams": s}, 0, "device", NS) for s in (1, 3, 4)]
    out += [("fp16", "fp16", {}, 0, "device", NS),
            ("fp32_tc0", "fp32", {"tensor_cores": 0}, 0, "device", NS),
            ("fp32_tc1", "fp32", {"tensor_cores": 1}, 0, "device", NS)]
    out += [("bf16_%s%d" % (k, v), "bf16", {k: v}, 0, "device", NS) for k, v in BF16_OPTIONS]
    out += [("bf16_taps1", "bf16", {}, 1, "device", NS), ("bf16_taps2", "bf16", {}, 2, "device", NS),
            ("bf16_graph", "bf16", {"graph": 1}, 0, "device", NS)]
    out += [("bf16_host_pinned", "bf16", {}, 0, "pinned", [128, 512]),
            ("bf16_host_pageable", "bf16", {}, 0, "pageable", [128, 512]),
            ("bf16_chunk100", "bf16", {"chunk": 100}, 0, "device", [250])]
    return out


def per_stream(trace_path):
    """The profiled GPU activities, grouped by stream, in launch order (the CUDA API call that issued them, then start time
    for the kernels of one graph launch).  Streams are numbered by their first launch: concurrent streams start in any order."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    gpu = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    gpu.sort(key=lambda e: (e["args"].get("correlation", 0), e["ts"]))
    streams = {}
    for e in gpu:
        a = e["args"]
        rows = streams.setdefault(a.get("stream"), [])
        if e["cat"] == "kernel":
            rows.append([e["name"], a.get("grid"), a.get("block"), a.get("shared memory")])
        else:
            rows.append([e["name"], a.get("bytes")])
    return list(streams.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", required=True, help="package root to import whenet_b200 from")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)
    import torch
    from torch.profiler import ProfilerActivity, profile
    import whenet_b200
    assert os.path.abspath(whenet_b200.__file__).startswith(root + os.sep), whenet_b200.__file__

    crops = np.random.default_rng(7).integers(0, 256, (512, 224, 224, 3), dtype=np.uint8)
    d_crops = torch.from_numpy(crops).cuda()
    p_crops = torch.from_numpy(crops).pin_memory()
    result = {}
    tmp = tempfile.mkdtemp(prefix="launch_trace_")
    for name, prec, opts, taps, kind, ns in configs():
        m = whenet_b200.WHENet(whenet_b200.weights.DEFAULT_NPZ, device=0, precision=prec, max_batch=512)
        for k, v in opts.items():
            m.set_option(k, v)
        result[name] = {}
        for n in ns:
            if taps:
                m.enable_taps(True, faithful=taps == 2, crops=sorted({0, n - 1}) if taps == 2 else None)
            if kind == "device":
                ang = torch.empty((n, 3), dtype=torch.float32, device="cuda")
                log = torch.empty((n, 252), dtype=torch.float32, device="cuda")
                run = lambda: m.forward_device(d_crops[:n], ang, log)     # noqa: E731
            else:
                src = p_crops[:n] if kind == "pinned" else crops[:n].copy()
                ang = np.empty((n, 3), dtype=np.float32)
                log = np.empty((n, 252), dtype=np.float32)
                run = lambda: m.forward_host(src, ang, log)               # noqa: E731
            run()
            m.synchronize()
            torch.cuda.synchronize()
            # the profiler now and then loses activity records, sometimes in two captures in a row: of three captures of the
            # same forward, keep the one with the most records
            best = None
            for _ in range(3):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run()
                    m.synchronize()
                    torch.cuda.synchronize()
                path = os.path.join(tmp, "trace.json")
                prof.export_chrome_trace(path)
                cur = per_stream(path)
                os.remove(path)
                if best is None or sum(map(len, cur)) > sum(map(len, best)):
                    best = cur
            result[name][str(n)] = best
        m.close()
        print("%-24s %s" % (name, " ".join("%s:%d" % (n, sum(map(len, r))) for n, r in result[name].items())), flush=True)
    os.rmdir(tmp)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=0)


if __name__ == "__main__":
    main()
