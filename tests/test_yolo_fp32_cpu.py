"""The detector's fp32 parity mode, everything that runs without a GPU: the ABI's precision argument, the Python keyword,
the fp32 tile plans at every legal model input size (tools/yolo_plan_dump.cu runs the library's own plan_igemm32), that the
GPU tests (test_gpu_yolo_fp32.py) reach every fp32 conv configuration a 132-SM H100 can choose, and how ptxas compiles the
new kernels (no spills, wgmma neither serialised nor fenced, registers that fit the CTAs per SM the plans assume)."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest

import yolo_cases as YC
import yolo_tiny_cases as TC
from conftest import ROOT
from whenet_b200 import yolo_arch as Y

EXE = os.path.join(ROOT, "build_tmp", "yolo_plan_dump32")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SMEM_OPTIN = 227 * 1024          # dynamic shared memory one CTA may opt in to on sm_90
SMEM_PER_SM = 228 * 1024         # shared memory per SM, 1 KB of it reserved per resident CTA
REGS_PER_SM = 65536
GPU_SMS = 132                    # H100 SXM, the GPU the tests run on
CLASSES = (1, 2, 80)

_LINE = re.compile(r"(?:(net32|tiny32) (\d+) (\d+) conv (\d+) mode (\w+) stride (\d+) |conv32 )Ho (\d+) Wo (\d+) N (\d+) Cin (\d+) "
                   r"k (\d+) n_tile (\d+) un (\d+) n_stages (\d+) ctas (\d+) smem (\d+) n_tail (\d+) m_tail (\d+)")
_KEYS = "Ho Wo N Cin k n_tile un n_stages ctas smem n_tail m_tail".split()


# ----------------------------------------------------------------------------------------------- ABI and Python argument checks
def test_create_ex_refuses_other_precisions():
    from whenet_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    for p in (-1, 2, 3, 99):
        assert L.whenet_det_create_ex(C.byref(h), 0, 416, 416, 1, p) == -1, p
        assert b"precision" in L.whenet_last_error()
    assert L.whenet_det_create_ex(None, 0, 416, 416, 1, 0) == -1
    assert L.whenet_det_create_ex(C.byref(h), 0, 400, 416, 1, 0) == -1 and b"multiples of 32" in L.whenet_last_error()
    assert L.whenet_det_create_ex(C.byref(h), 0, 416, 416, 0, 0) == -1 and b"max_frames" in L.whenet_last_error()
    assert L.whenet_det_precision(None) == -1
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        for p in (0, 1):
            assert L.whenet_det_create_ex(C.byref(h), 0, 416, 416, 1, p) == -2


def test_yolo_refuses_other_precisions_before_the_library():
    import whenet_b200
    for p in ("fp16", "tf32", "FP32", None, 0):
        with pytest.raises(ValueError, match="precision"):
            whenet_b200.YOLO(precision=p)
    with pytest.raises(TypeError):
        whenet_b200.YOLO(None, None, None, 0.3, 0.45, (416, 416), 1, "fp32")      # keyword only


# ----------------------------------------------------------------------------------------------- plans
@pytest.fixture(scope="module")
def dump():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run([NVCC, "-std=c++17", "-arch=sm_90a", "-o", EXE, os.path.join(ROOT, "tools", "yolo_plan_dump.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(*args):
        out = subprocess.run([EXE] + [str(a) for a in args], capture_output=True, text=True, check=True).stdout
        rows = []
        for m in _LINE.finditer(out):
            g = m.groups()
            r = dict(zip(_KEYS, (int(v) for v in g[6:])))
            if g[0] is not None:
                r.update(net=g[0], h=int(g[1]), w=int(g[2]), conv=int(g[3]), mode=g[4], stride=int(g[5]))
            rows.append(r)
        return rows
    return run


@pytest.fixture(scope="module")
def nets(dump):
    """(network, classes, sm_count) -> the fp32 plan rows of every conv but the first at every legal input size"""
    return {(net, c, sm): dump(net, c, sm) for net in ("net32", "tiny32") for c in CLASSES for sm in (GPU_SMS, 114)}


def config(r):
    return (r["mode"], r["k"], r["stride"], r["un"], r["n_tile"], r["n_stages"])


def test_every_fp32_plan_fits(nets):
    for (net, c, sm), rows in nets.items():
        tiny = net == "tiny32"
        assert len(rows) == 19 * 19 * (Y.TINY_N_CONV - 1 if tiny else Y.N_CONV - 1)
        for r in rows:
            what = (net, c, sm, r["h"], r["w"], r["conv"])
            L = Y.table(tiny)[r["conv"]]
            assert r["un"] in (32, 64, 128) and r["n_tile"] % 16 == 0 and r["n_tile"] <= r["un"], what
            assert 2 <= r["n_stages"] <= 4 and r["ctas"] in (1, 2), what
            stage = 2 * 128 * 64 * 2 + 2 * r["un"] * 64 * 2
            assert r["smem"] >= r["n_stages"] * stage + 1024 and r["smem"] >= r["un"] * 132 * 4 + 1024, what
            assert r["smem"] <= SMEM_OPTIN and r["ctas"] * (r["smem"] + 1024) <= SMEM_PER_SM, what
            assert 0 < r["n_tail"] <= r["n_tile"], what
            if r["mode"] != "f32":
                assert r["n_tail"] % 8 == 0, what
            assert r["N"] == (Y.head_channels(c) if L.head is not None else L.cout) and r["Cin"] == L.cin and r["k"] == L.k, what
            assert (r["Ho"], r["Wo"]) == Y.out_hw(r["h"], r["w"], tiny=tiny)[r["conv"]], what


def test_fp32_plans_take_the_bf16_tiles(dump):
    """The fp32 plan keeps plan_igemm's tile, which depends on the per-frame shape only (batch invariance)."""
    bf = re.compile(r"net (\d+) (\d+) conv (\d+) .*? n_tile (\d+) un (\d+)")
    exe_out = subprocess.run([EXE, "net", "1", str(GPU_SMS)], capture_output=True, text=True, check=True).stdout
    tiles = {(int(a), int(b), int(c)): (int(d), int(e)) for a, b, c, d, e in bf.findall(exe_out)}
    rows = dump("net32", 1, GPU_SMS)
    assert len(tiles) == len(rows)
    for r in rows:
        assert tiles[r["h"], r["w"], r["conv"]] == (r["n_tile"], r["un"]), r


def _debug_rows(dump, cases):
    args = []
    for (n, H, W, cin, c_up, cout, k, stride, mode, un) in cases:
        args += [H // stride, W // stride, cout, cin, k]
    rows = dump("conv32", GPU_SMS, *args)
    assert len(rows) == len(cases)
    for r, case in zip(rows, cases):
        r.update(mode=case[8], stride=case[7])
    return rows


def test_gpu_tests_reach_every_fp32_conv_configuration(dump, nets):
    """test_gpu_yolo_fp32.py checks every conv of both networks at MODEL_SIZES (one class) and the debug-conv cases of
    yolo_cases.DEBUG_CONVS and yolo_tiny_cases.DEBUG_CONVS; together they must reach every (mode, k, stride, tile width,
    columns, ring depth) the fp32 planner can choose for 1, 2 or 80 classes on 132 SMs."""
    reachable = {}
    for (net, c, sm), rows in nets.items():
        if sm == GPU_SMS:
            for r in rows:
                reachable.setdefault(config(r), (net, c, r["h"], r["w"], r["conv"]))
    covered = {config(r) for net in ("net32", "tiny32") for r in nets[net, 1, GPU_SMS] if (r["h"], r["w"]) in YC.MODEL_SIZES}
    covered |= {config(r) for r in _debug_rows(dump, YC.DEBUG_CONVS + TC.DEBUG_CONVS)}
    print("%d reachable fp32 configurations (mode, k, stride, un, n_tile, n_stages):" % len(reachable))
    for cfg in sorted(reachable):
        print("  ", cfg)
    missing = {cfg: reachable[cfg] for cfg in reachable if cfg not in covered}
    assert not missing, "reachable but never checked on the GPU (network, classes, h, w, conv): %s" % missing


# ----------------------------------------------------------------------------------------------- how ptxas compiles the new kernels
@pytest.fixture(scope="module")
def ptxas_log():
    from whenet_b200 import build
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas=-v", "-c", "-o", os.path.join(tmp, "inst_yolo32.o"),
                            os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc", "inst_yolo32.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout + r.stderr


def _entries(log):
    """kernel name -> (registers, spill store bytes, spill load bytes)"""
    out = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads.*?Used (\d+) registers", log, re.S):
        out[m.group(1)] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    return out


def test_ptxas_does_not_serialise_or_fence_the_fp32_kernels(ptxas_log):
    assert not re.findall(r"\(C7520\)", ptxas_log), "wgmma serialised"
    assert not re.findall(r"\(C7519\)", ptxas_log), "ptxas injected warpgroup arrives"


def test_fp32_kernels_do_not_spill_and_fit_their_ctas(ptxas_log, nets):
    ents = {k: v for k, v in _entries(ptxas_log).items() if re.search(r"conv_igemm32_kernel|yolo_conv0_32_kernel|yolo_maxpool32_kernel", k)}
    assert len(ents) == 12 + 2 + 1, sorted(ents)
    ctas = {}
    for rows in nets.values():
        for r in rows:
            ctas[r["un"]] = max(ctas.get(r["un"], 0), r["ctas"])
    for name, (regs, st, ld) in ents.items():
        assert st == 0 and ld == 0, (name, st, ld)
        m = re.search(r"conv_igemm32_kernelILi(\d)ELi(\d+)E", name)
        if m:
            assert regs * 128 * ctas.get(int(m.group(2)), 1) <= REGS_PER_SM, (name, regs)
