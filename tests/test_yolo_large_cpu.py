"""Model inputs above 608 without a GPU: whenet_det_create_large's argument checks, the Python size and max_boxes checks, the
tile plans tools/yolo_plan_dump.cu prints for sizes from 640 to 4096, the frame groups of the conv launch split and the
capacity of the second decode + NMS route (DESIGN.md 8.6)."""
import ctypes as C
import os
import re
import subprocess

import pytest

import test_yolo_fp32_cpu as F32
from test_gpu_yolo_large import CONV_RUNS
from test_yolo_plans import _LINE, _KEYS, SMEM_OPTIN, SMEM_PER_SM, config
from whenet_b200 import yolo_arch as Y

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build_tmp", "yolo_plan_dump_large")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SIZES = [(640, 640), (1088, 1920), (1056, 1920), (2176, 3840), (4096, 4096), (32, 4096), (4096, 32), (704, 1280), (2144, 3840),
         (1920, 1088)]
GRID_Y = 65535


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_create_large_argument_checks():
    from whenet_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    assert L.whenet_det_create_large(None, 0, 640, 640, 1, 1) == -1
    for hw in ((4128, 640), (640, 4128), (0, 640), (640, 0), (1080, 1920), (1088, 1900), (16, 32)):
        assert L.whenet_det_create_large(C.byref(h), 0, hw[0], hw[1], 1, 1) == -1, hw
        assert b"multiples of 32 in [32, 4096]" in L.whenet_last_error()
    assert L.whenet_det_create_large(C.byref(h), 0, 640, 640, 0, 1) == -1 and b"max_frames" in L.whenet_last_error()
    assert L.whenet_det_create_large(C.byref(h), 0, 640, 640, 1, 7) == -1 and b"precision" in L.whenet_last_error()
    # the 608 contract of whenet_det_create(_ex) is unchanged
    assert L.whenet_det_create_ex(C.byref(h), 0, 640, 640, 1, 1) == -1 and b"[32, 608]" in L.whenet_last_error()
    assert L.whenet_det_debug_force_large_decode(None, 1) == -1
    if not _has_gpu():
        for hw in ((640, 640), (4096, 4096), (1088, 1920), (32, 4096)):
            for p in (0, 1):
                assert L.whenet_det_create_large(C.byref(h), 0, hw[0], hw[1], 1, p) == -2, (hw, p)


def test_python_size_and_max_boxes_checks():
    import whenet_b200
    for size in ((4128, 640), (1080, 1920), (0, 640)):
        with pytest.raises(ValueError, match=r"multiples of 32 in \[32, 4096\]"):
            whenet_b200.YOLO(model_image_size=size)
    for mb in (0, 257, 2.5, True, "20"):
        with pytest.raises(ValueError, match="max_boxes"):
            whenet_b200.YOLO(max_boxes=mb)
    assert Y.MIN_SIZE == 32 and Y.MAX_SIZE == 608 and Y.LARGE_MAX_SIZE == 4096
    Y.check_size(4096, 32, max_size=Y.LARGE_MAX_SIZE)
    with pytest.raises(ValueError):
        Y.check_size(640, 640)
    if not _has_gpu():          # past every argument check to the device: the library reports no GPU
        from whenet_b200._lib import WhenetError
        for size in ((640, 640), (1088, 1920)):
            with pytest.raises(WhenetError) as e:
                whenet_b200.YOLO(model_image_size=size, max_boxes=256)
            assert e.value.code == -2


@pytest.fixture(scope="module")
def dump():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run([NVCC, "-std=c++17", "-arch=sm_90a", "-o", EXE, os.path.join(ROOT, "tools", "yolo_plan_dump.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(*args):
        return subprocess.run([EXE] + [str(a) for a in args], capture_output=True, text=True, check=True).stdout
    return run


def _rows(out, prefix):
    """The plan rows of `prefix` (net, tiny, net32, tiny32) lines, with the conv's index, mode and stride"""
    fp32 = prefix.endswith("32")
    line_re, keys = (F32._LINE, F32._KEYS) if fp32 else (_LINE, _KEYS)
    rows = []
    for line in out.splitlines():
        if not line.startswith(prefix + " "):
            continue
        g = re.search(r"conv (\d+) mode (\w+) stride (\d+) ", line)
        m = line_re.search(("net32 0 0 " if fp32 else "net 0 0 ") + line[line.index("conv "):])
        r = dict(zip(keys, (int(v) for v in m.groups()[6 if fp32 else 5:])))
        r.update(conv=int(g.group(1)), mode=g.group(2), stride=int(g.group(3)))
        rows.append(r)
    return rows


@pytest.mark.parametrize("tiny", [False, True], ids=["yolov3", "tiny"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_plans_fit_at_large_sizes(dump, tiny, precision):
    """plan_igemm (bf16) and plan_igemm32 (fp32) plans of both networks, with 1, 2 and 80 classes on 132 and 114 SMs, fit their
    kernel at every size, and the GPU tests run every configuration they choose: the per-layer tests at every size up to 608
    with one class, and test_gpu_yolo_large's CONV_RUNS above it."""
    fp32 = precision == "fp32"
    cmd = ("tiny" if tiny else "net") + ("32" if fp32 else "")
    table = Y.table(tiny)
    reachable = {}
    for sm in (132, 114):
        for c in (1, 2, 80):
            for h, w in SIZES:
                rows = _rows(dump(cmd, c, sm, h, w), cmd)
                assert len(rows) == len(table) - 1
                for r in rows:
                    what = (cmd, c, sm, h, w, r["conv"])
                    assert r["un"] in (32, 64, 128) and r["n_tile"] % 16 == 0 and r["n_tile"] <= r["un"], what
                    assert 2 <= r["n_stages"] <= 4, what
                    ctas = r["ctas"] if fp32 else 2
                    assert (not fp32 or ctas in (1, 2)) and r["smem"] <= SMEM_OPTIN and ctas * (r["smem"] + 1024) <= SMEM_PER_SM, what
                    assert 0 < r["n_tail"] <= r["n_tile"] and (r["mode"] == "f32" or r["n_tail"] % 8 == 0), what
                    assert (r["Ho"], r["Wo"]) == Y.out_hw(h, w, tiny)[r["conv"]], what
                    if sm == 132:
                        reachable.setdefault(config(r), what)
    covered = {config(r) for r in _rows(dump(cmd, 1, 132), cmd)}                  # every size 32..608, one class
    for (t, c, h, w, p) in CONV_RUNS:
        if t == tiny and p == precision:
            covered |= {config(r) for r in _rows(dump(cmd, c, 132, h, w), cmd)}
    missing = {k: v for k, v in reachable.items() if k not in covered}
    print("%d %s configurations at large sizes" % (len(reachable), cmd))
    assert not missing, "reachable at large sizes but never run on the GPU (net, classes, sm, h, w, conv): %s" % missing


def _groups(out):
    res = []
    for line in out.splitlines():
        if line.startswith("split "):
            head, *parts = line.split(" | ")
            hw = [int(v) for v in re.findall(r"\d+", head)]
            res.append((hw, [tuple(int(v) for v in re.match(r"f0 (\d+) nf (\d+) tiles (\d+)", p).groups()) for p in parts]))
    return res


def test_frame_groups_of_the_conv_launch_split(dump):
    """Every conv's M tiles at the new sizes, for 1..64 frames: no launch over 65,535 tiles, every frame exactly once, in
    order; one launch whenever the whole call fits."""
    shapes = set()
    for tiny in (False, True):
        for h, w in SIZES:
            shapes |= set(Y.out_hw(h, w, tiny)[1:])
    args = []
    for Ho, Wo in sorted(shapes):
        for n in (1, 2, 3, 16, 17, 33, 64):
            args += [Ho, Wo, n]
    got = _groups(dump("split", *args))
    assert len(got) == len(args) // 3
    for (Ho, Wo, n), groups in got:
        hw = Ho * Wo
        assert all(t <= GRID_Y for _f0, _nf, t in groups), (Ho, Wo, n)
        assert [f0 for f0, _nf, _t in groups] == [sum(g[1] for g in groups[:i]) for i in range(len(groups))]
        assert sum(nf for _f0, nf, _t in groups) == n
        assert all(t == -(-nf * hw // 128) for _f0, nf, t in groups)
        if -(-n * hw // 128) <= GRID_Y:
            assert len(groups) == 1
    assert max(-(-hw[0] * hw[1] // 128) for hw in shapes) == 32768          # conv 1 at 4096 x 4096: one frame always fits
    tiny17 = [g for (hw, g) in got if hw == [544, 960, 17]]
    assert tiny17 == [[(0, 16, 65280), (16, 1, 4080)]]


def test_large_route_capacity(dump):
    out = dump("net", 1, 132, 640, 640)
    m = re.search(r"large nms above (\d+) candidates max_candidates (\d+) alive_bytes (\d+) max_side (\d+) grid_y (\d+)", out)
    above, cap, alive, side, grid_y = (int(v) for v in m.groups())
    assert re.match(r"nms per (\d+) threads (\d+) max_boxes (\d+)", out)
    assert above == 24576 and side == Y.LARGE_MAX_SIZE and grid_y == GRID_Y
    assert cap == Y.num_candidates(4096, 4096) == 1032192
    assert max(Y.num_candidates(h, w, t) for h in range(32, 4097, 32) for w in (32, 4096) for t in (False, True)) <= cap
    assert alive == cap // 8 <= 227 * 1024 - 1024                       # one bit per candidate, in one CTA's shared memory
    assert Y.num_candidates(608, 608) <= above < Y.num_candidates(640, 640)
