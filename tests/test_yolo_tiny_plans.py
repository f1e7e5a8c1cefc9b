"""Host-side checks of tiny YOLOv3's implicit-GEMM tile plans (no GPU), as test_yolo_plans.py does for the full model:
tools/yolo_plan_dump.cu runs the library's own plan_igemm over its own tiny conv table at every legal model input size.
Every plan must fit the kernel, and the tiny GPU tests (yolo_tiny_cases.py) must reach every conv configuration the planner
can choose for the tiny network, the 3x3 concat conv included."""
import os
import re
import subprocess

import pytest

import yolo_tiny_cases as TC
from whenet_b200 import yolo_arch as Y

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build_tmp", "yolo_plan_dump_tiny")
SMEM_OPTIN = 227 * 1024          # dynamic shared memory one CTA may opt in to on sm_90
SMEM_PER_SM = 228 * 1024         # shared memory per SM, 1 KB of it reserved per resident CTA
GPU_SMS = 132                    # H100 SXM, the GPU the tests run on
CLASSES = (1, 2, 80)

_LINE = re.compile(r"(?:tiny (\d+) (\d+) conv (\d+) mode (\w+) stride (\d+) |conv )Ho (\d+) Wo (\d+) N (\d+) Cin (\d+) k (\d+) "
                   r"n_tile (\d+) un (\d+) n_stages (\d+) smem (\d+) n_tail (\d+) m_tail (\d+)")
_KEYS = "Ho Wo N Cin k n_tile un n_stages smem n_tail m_tail".split()


@pytest.fixture(scope="module")
def dump():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    r = subprocess.run([nvcc, "-std=c++17", "-arch=sm_90a", "-o", EXE, os.path.join(ROOT, "tools", "yolo_plan_dump.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(*args):
        out = subprocess.run([EXE] + [str(a) for a in args], capture_output=True, text=True, check=True).stdout
        consts = dict(zip(("per", "threads", "max_boxes"), map(int, re.match(r"nms per (\d+) threads (\d+) max_boxes (\d+)", out).groups())))
        rows = []
        for m in _LINE.finditer(out):
            g = m.groups()
            r = dict(zip(_KEYS, (int(v) for v in g[5:])))
            if g[0] is not None:
                r.update(h=int(g[0]), w=int(g[1]), conv=int(g[2]), mode=g[3], stride=int(g[4]))
            rows.append(r)
        return consts, rows
    return run


@pytest.fixture(scope="module")
def nets(dump):
    """(classes, sm_count) -> the plan rows of tiny convs 1..12 at every legal input size"""
    return {(c, sm): dump("tiny", c, sm)[1] for sm in (GPU_SMS, 114) for c in CLASSES}


def config(r):
    return (r["mode"], r["k"], r["stride"], r["un"], r["n_tile"], r["n_stages"])


def _debug_rows(dump):
    args = []
    for (n, H, W, cin, c_up, cout, k, stride, mode, un) in TC.DEBUG_CONVS:
        args += [H // stride, W // stride, cout, cin, k]
    _, rows = dump("conv", GPU_SMS, *args)
    assert len(rows) == len(TC.DEBUG_CONVS)
    for r, case in zip(rows, TC.DEBUG_CONVS):
        r.update(mode=case[8], stride=case[7])
    return rows


def test_every_tiny_plan_fits_the_kernel(nets):
    modes = {L.idx: ("f32" if L.head is not None else "cat" if L.up is not None else "leaky") for L in Y.TINY_LAYERS}
    for (c, sm), rows in nets.items():
        assert len(rows) == 19 * 19 * 12
        for r in rows:
            what = (c, sm, r["h"], r["w"], r["conv"])
            assert r["un"] in (32, 64, 128) and r["n_tile"] % 16 == 0 and r["n_tile"] <= r["un"], what
            assert 2 <= r["n_stages"] <= 4, what
            assert r["smem"] <= SMEM_OPTIN and 2 * (r["smem"] + 1024) <= SMEM_PER_SM, what        # two CTAs per SM
            assert 0 < r["n_tail"] <= r["n_tile"], what
            if r["mode"] != "f32":
                assert r["n_tail"] % 8 == 0, what               # the bf16 epilogue stores 8-channel chunks
            L = Y.TINY_LAYERS[r["conv"]]
            assert r["mode"] == modes[L.idx] and r["stride"] == 1 and r["k"] == L.k and r["Cin"] == L.cin, what
            assert r["N"] == (Y.head_channels(c) if r["mode"] == "f32" else L.cout), what
            assert (r["Ho"], r["Wo"]) == Y.out_hw(r["h"], r["w"], tiny=True)[r["conv"]], what


def test_the_nms_block_holds_every_tiny_candidate(dump):
    consts, _ = dump("tiny", 1, GPU_SMS, 32, 32)
    assert Y.num_candidates(608, 608, tiny=True) <= consts["per"] * consts["threads"]


def test_tiny_debug_conv_cases_plan_as_stated(dump):
    for r, case in zip(_debug_rows(dump), TC.DEBUG_CONVS):
        assert r["un"] == case[9], (case, r)


def test_tiny_debug_conv_cases_include_conv10_at_32_416_608(dump, nets):
    """The concat cases include the exact tile plan the library runs tiny conv 10 with at 32^2, 416^2 and 608^2."""
    cases = {(case[1], case[2]): r for r, case in zip(_debug_rows(dump), TC.DEBUG_CONVS) if case[0] == 1}
    for s in (32, 416, 608):
        (r10,) = [r for r in nets[1, GPU_SMS] if (r["h"], r["w"], r["conv"]) == (s, s, 10)]
        assert config(cases[r10["Ho"], r10["Wo"]]) == config(r10), s


def test_tiny_gpu_tests_reach_every_conv_configuration(dump, nets):
    reachable = {}
    for c in CLASSES:
        for r in nets[c, GPU_SMS]:
            reachable.setdefault(config(r), (c, r["h"], r["w"], r["conv"]))
    covered = {config(r) for r in nets[1, GPU_SMS] if (r["h"], r["w"]) in TC.MODEL_SIZES}
    for c, sizes in TC.CLASS_SIZES.items():
        covered |= {config(r) for r in nets[c, GPU_SMS] if (r["h"], r["w"]) in sizes and r["mode"] == "f32"}
    covered |= {config(r) for r in _debug_rows(dump)}
    missing = {cfg: reachable[cfg] for cfg in reachable if cfg not in covered}
    print("%d reachable tiny configurations (mode, k, stride, un, n_tile, n_stages):" % len(reachable))
    for cfg in sorted(reachable):
        print("  ", cfg)
    assert not missing, "reachable but never checked on the GPU (classes, h, w, conv): %s" % missing
    assert ("cat", 3, 1, 32, 32, 4) in reachable
