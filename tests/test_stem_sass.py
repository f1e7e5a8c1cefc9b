"""What the compiler made of the register-blocked stem (no GPU needed: resource usage and SASS of the built library).

Every stem_tile_kernel instance (u8 / float input x fp16 / bf16 / fp32 storage) must fit two 224-thread CTAs per SM by
registers without spilling, and issue at least 4 FFMAs (one per pixel of the thread's quad) per instruction that can load
a weight: constant-bank loads and 16-byte shared-memory loads.  The one-pixel-per-thread kernel it replaced issued about 2
FFMAs per weight load.
"""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

NVCC_DIR = "/usr/local/cuda/bin"
INSTANCES = {(t, u8) for t in ("6__half", "13__nv_bfloat16", "f") for u8 in (0, 1)}
THREADS, CTAS_PER_SM = 224, 2
PIXELS_PER_THREAD = 4


def _cuobjdump(*args):
    from whenet_b200 import build
    cu = shutil.which("cuobjdump") or os.path.join(NVCC_DIR, "cuobjdump")
    if not os.path.exists(cu):
        pytest.skip("cuobjdump not available")
    return subprocess.run([cu, *args, build.build_lib()], capture_output=True, text=True, check=True).stdout


def _instance(name):
    m = re.search(r"stem_tile_kernelI(6__half|13__nv_bfloat16|f)Lb([01])ELb[01]E", name)
    return (m.group(1), int(m.group(2))) if m else None


def test_stem_registers_and_no_spills():
    seen = set()
    budget = (65536 // (THREADS * CTAS_PER_SM)) // 8 * 8         # registers are allocated in steps of 8 per thread
    for name, res in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("-res-usage")):
        inst = _instance(name)
        if inst is None:
            continue
        seen.add(inst)
        fields = dict(re.findall(r"(\w+):(\d+)", res))
        assert int(fields["REG"]) <= budget, "%s: %s registers > %d (%d CTAs of %d threads per SM)" % (
            name, fields["REG"], budget, CTAS_PER_SM, THREADS)
        assert int(fields["STACK"]) == 0 and int(fields["LOCAL"]) == 0, "%s spills: %s" % (name, res)
    assert seen == INSTANCES, seen


def test_stem_ffma_per_weight_load():
    seen = set()
    sass = _cuobjdump("-sass")
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        inst = _instance(name.strip())
        if inst is None:
            continue
        seen.add(inst)
        ops = Counter(m.split(".")[0] for m in re.findall(r"\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", body))
        assert ops["STL"] == 0 and ops["LDL"] == 0, name
        # weights reach the FFMAs from the constant bank (ULDC, LDC) or from shared memory as broadcast 16-byte loads; the
        # count includes the input and output-stage loads, so it is an upper bound on the weight loads
        loads = ops["ULDC"] + ops["LDC"] + len(re.findall(r"LDS\.128", body))
        assert ops["FFMA"] >= 27 * 32 * 2 * 2, "%s: %d FFMA" % (name, ops["FFMA"])    # 2 halves x 27 x 16 x 4 pixels
        assert ops["FFMA"] >= PIXELS_PER_THREAD * loads, "%s: %d FFMA for %d weight loads" % (name, ops["FFMA"], loads)
    assert seen == INSTANCES, seen
