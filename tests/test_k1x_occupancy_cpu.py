"""Host-side checks (no GPU) that K1X's instances fit the CTAs per SM they are compiled for: blocks 2-4 (64-byte A / W rows)
three, block 6 (128-byte rows) two, by shared memory (route_plan_dump's sizes) and by registers (the built library)."""
import os
import re
import subprocess

import pytest

from conftest import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
EXE = os.path.join(ROOT, "build_tmp", "route_plan_dump_k1x_occ")
WANT = {2: (3, 64), 3: (3, 64), 4: (3, 64), 6: (2, 128)}     # block -> (CTAs per SM, bytes per A / W row)
SMEM_PER_SM, SMEM_RESERVED, STATIC = 228 * 1024, 1024, 256    # per SM; reserved per CTA; the kernel's barriers, rounded up
REGS_PER_SM, THREADS = 65536, 256


@pytest.fixture(scope="module")
def k1x():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run([NVCC, "-std=c++17", "-arch=sm_90a", "-o", EXE, os.path.join(ROOT, "tools", "route_plan_dump.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([EXE, "256"], capture_output=True, text=True, check=True).stdout
    rows = {}
    for line in out.splitlines():
        m = re.search(r"k1x b(\d+) .* cin (\d+) .* smem (\d+) chunks \d+ ctas_per_sm (\d+) row_bytes (\d+)", line)
        if m:
            rows[int(m.group(1))] = dict(zip(("cin", "smem", "ctas", "rowb"), (int(v) for v in m.groups()[1:])))
    return rows


def test_row_width_and_ctas_per_sm(k1x):
    assert sorted(k1x) == sorted(WANT)
    for b, r in k1x.items():
        assert (r["ctas"], r["rowb"]) == WANT[b], b
        assert (r["rowb"] == 64) == (r["cin"] + 8 <= 32), b            # 64-byte rows exactly where K = Cin + 8 fits in 32


def test_shared_memory_fits(k1x):
    for b, r in k1x.items():
        assert r["ctas"] * (r["smem"] + SMEM_RESERVED + STATIC) <= SMEM_PER_SM, (b, r)


def test_registers_fit():
    from whenet_b200 import build
    cu = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    if not os.path.exists(cu):
        pytest.skip("cuobjdump not available")
    res = subprocess.run([cu, "-res-usage", build.build_lib()], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    regs, name = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Function (\S*k1x_kernelILi(\d+)ELi(\d+)ELi(\d+)E\S*):", line)
        if m:
            name = (int(m.group(2)), int(m.group(3)), int(m.group(4)))          # (KS, S, HIN)
            continue
        m = re.search(r"REG:(\d+)", line)
        if m and name:
            regs[name] = int(m.group(1))
            name = None
    block = {(3, 2, 112): 2, (3, 1, 56): 3, (5, 2, 56): 4, (3, 2, 28): 6}
    assert sorted(regs) == sorted(block)
    for key, n in regs.items():
        b = block[key]
        alloc = -(-n // 8) * 8                                                # registers are allocated 8 per thread at a time
        assert alloc * THREADS * WANT[b][0] <= REGS_PER_SM, (b, n)
