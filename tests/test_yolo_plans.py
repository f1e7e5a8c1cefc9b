"""Host-side checks of the YOLOv3 detector's implicit-GEMM tile plans (no GPU): tools/yolo_plan_dump.cu runs the library's own
plan_igemm over its own conv table at every legal model input size.  Every plan must fit the kernel (tile width, ring depth,
shared memory for two CTAs per SM), the decode/NMS CTA must hold every candidate, and the GPU tests (yolo_cases.py) must
reach every conv configuration the planner can choose, so that no conv_igemm_kernel instance runs unchecked."""
import os
import re
import subprocess

import pytest

import yolo_cases as YC
from whenet_b200 import yolo_arch as Y

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build_tmp", "yolo_plan_dump")
SMEM_OPTIN = 227 * 1024          # dynamic shared memory one CTA may opt in to on sm_90
SMEM_PER_SM = 228 * 1024         # shared memory per SM, 1 KB of it reserved per resident CTA
GPU_SMS = 132                    # H100 SXM, the GPU the tests run on
CLASSES = (1, 2, 80)

_LINE = re.compile(r"(?:net (\d+) (\d+) conv (\d+) mode (\w+) stride (\d+) |conv )Ho (\d+) Wo (\d+) N (\d+) Cin (\d+) k (\d+) "
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
    """(classes, sm_count) -> the plan rows of convs 1..74 at every legal input size"""
    out = {}
    for sm in (GPU_SMS, 114):
        for c in CLASSES:
            out[c, sm] = dump("net", c, sm)[1]
    return out


def config(r):
    return (r["mode"], r["k"], r["stride"], r["un"], r["n_tile"], r["n_stages"])


def _debug_rows(dump):
    args = []
    for (n, H, W, cin, c_up, cout, k, stride, mode, un) in YC.DEBUG_CONVS:
        args += [H // stride, W // stride, cout, cin, k]
    _, rows = dump("conv", GPU_SMS, *args)
    assert len(rows) == len(YC.DEBUG_CONVS)
    for r, case in zip(rows, YC.DEBUG_CONVS):
        r.update(mode=case[8], stride=case[7])
    return rows


def test_every_plan_fits_the_kernel(nets):
    for (c, sm), rows in nets.items():
        assert len(rows) == 19 * 19 * 74
        for r in rows:
            what = (c, sm, r["h"], r["w"], r["conv"])
            assert r["un"] in (32, 64, 128) and r["n_tile"] % 16 == 0 and r["n_tile"] <= r["un"], what
            assert 2 <= r["n_stages"] <= 4, what
            assert r["smem"] <= SMEM_OPTIN and 2 * (r["smem"] + 1024) <= SMEM_PER_SM, what        # two CTAs per SM
            assert 0 < r["n_tail"] <= r["n_tile"], what
            if r["mode"] != "f32":
                assert r["n_tail"] % 8 == 0, what               # the bf16 epilogue stores 8-channel chunks
            assert r["N"] == (Y.head_channels(c) if r["mode"] == "f32" else Y.LAYERS[r["conv"]].cout), what
            assert (r["Ho"], r["Wo"]) == Y.out_hw(r["h"], r["w"])[r["conv"]], what


def test_the_nms_block_holds_every_candidate(dump):
    consts, _ = dump("net", 1, GPU_SMS, 32, 32)
    assert consts["max_boxes"] == 256 and consts["threads"] == 1024
    assert max(Y.num_candidates(h, w) for h in range(32, 609, 32) for w in range(32, 609, 32)) <= consts["per"] * consts["threads"]
    assert consts["per"] <= 32                          # one alive bit per candidate in a 32-bit mask


def test_debug_conv_cases_plan_as_stated(dump):
    for r, case in zip(_debug_rows(dump), YC.DEBUG_CONVS):
        assert r["un"] == case[9], (case, r)


def test_gpu_tests_reach_every_conv_configuration(dump, nets):
    """The per-layer test checks every conv at MODEL_SIZES (one class); the class-count tests check the output convs at
    CLASS_SIZES; debug_conv checks DEBUG_CONVS.  A plan change that leaves a reachable configuration unchecked names it."""
    reachable = {}
    for c in CLASSES:
        for r in nets[c, GPU_SMS]:
            reachable.setdefault(config(r), (c, r["h"], r["w"], r["conv"]))
    covered = set()
    for r in nets[1, GPU_SMS]:
        if (r["h"], r["w"]) in YC.MODEL_SIZES:
            covered.add(config(r))
    for c, sizes in YC.CLASS_SIZES.items():
        for r in nets[c, GPU_SMS]:
            if (r["h"], r["w"]) in sizes and r["mode"] == "f32":
                covered.add(config(r))
    covered |= {config(r) for r in _debug_rows(dump)}
    missing = {cfg: reachable[cfg] for cfg in reachable if cfg not in covered}
    print("%d reachable configurations (mode, k, stride, un, n_tile, n_stages), all covered:" % len(reachable))
    for cfg in sorted(reachable):
        print("  ", cfg)
    assert not missing, "reachable but never checked on the GPU (classes, h, w, conv): %s" % missing
    # every template instance the library can launch is among them
    assert {(m, u) for (m, _k, _s, u, _n, _st) in reachable} == {("leaky", 32), ("leaky", 64), ("leaky", 128), ("res", 32), ("res", 64),
                                                                  ("res", 128), ("cat", 32), ("f32", 32), ("f32", 64)}
