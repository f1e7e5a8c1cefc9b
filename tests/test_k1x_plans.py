"""Host-side checks (no GPU) of K1X (k1x_kernel, blocks 2, 3, 4 and 6 in bf16; block 5 stays on K1, where it is faster): the
instances tools/route_plan_dump.cu prints against K1's tile plans, and what ptxas and the SASS show for them in
inst_k1_bf16.cu."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc")
EXE = os.path.join(ROOT, "build_tmp", "route_plan_dump_k1x")
K1_EXE = os.path.join(ROOT, "build_tmp", "k1_plan_dump_k1x")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CEXP = {2: 96, 3: 144, 4: 144, 6: 240}
CIN = {2: 16, 3: 24, 4: 24, 6: 40}


def _build_and_run(src, exe, *args):
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    r = subprocess.run([NVCC, "-std=c++17", "-arch=sm_90a", "-o", exe, os.path.join(ROOT, "tools", src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return subprocess.run([exe] + list(args), capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def k1x():
    rows = {}
    for line in _build_and_run("route_plan_dump.cu", EXE, "256").splitlines():
        m = re.search(r"k1x b(\d+) th (\d+) r (\d+) cc (\d+) cin (\d+) tiles (\d+) pix (\d+) halves (\d+) ksteps (\d+) lanes (\d+) smem (\d+) chunks (\d+)", line)
        if m:
            rows[int(m.group(1))] = dict(zip("th r cc cin tiles pix halves ksteps lanes smem chunks".split(), (int(v) for v in m.groups()[1:])))
    return rows


def test_instances_follow_the_k1_plans(k1x):
    assert sorted(k1x) == [2, 3, 4, 6]
    k1 = {}
    for line in _build_and_run("k1_plan_dump.cu", K1_EXE).splitlines():
        m = re.match(r"\s*b(\d+)\s.*:\s*(\d+)x(\d+)\s+r(\d) cc(\d+)\s+nt(\d+) nb(\d)", line)
        if m and int(m.group(1)) in k1x:
            k1[int(m.group(1))] = tuple(int(v) for v in m.groups()[1:])
    for b, r in k1x.items():
        assert k1[b] == (r["th"], r["th"], r["r"], r["cc"], 256, 1), b           # same tiles, strips and chunks as K1
        assert r["cin"] == CIN[b] and r["chunks"] * r["cc"] == CEXP[b], b
        assert r["halves"] == -(-r["pix"] // 64) and r["ksteps"] == ((r["cin"] // 8 + 2) & ~1) // 2, b
        assert r["lanes"] * (r["cc"] // 4) <= 256, b
        # two CTAs per SM: 228 KB, 1 KB reserved per CTA, + the kernel's static barriers
        assert 2 * (r["smem"] + 256 + 1024) <= 228 * 1024, b


@pytest.fixture(scope="module")
def ptxas_and_sass(tmp_path_factory):
    d = tmp_path_factory.mktemp("k1x")
    obj = str(d / "inst_k1_bf16.o")
    r = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", "-o", obj,
                        os.path.join(CSRC, "inst_k1_bf16.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True)
    assert sass.returncode == 0, sass.stderr
    return r.stderr, sass.stdout


def _per_function(text, start_pat):
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(start_pat, line)
        if m:
            cur = m.group(1)
            out.setdefault(cur, [])
        if cur:
            out[cur].append(line)
    return out


def test_ptxas_clean(ptxas_and_sass):
    log, _ = ptxas_and_sass
    funcs = {k: "\n".join(v) for k, v in _per_function(log, r"Compiling entry function '(\w+)'").items() if "k1x_kernel" in k}
    assert len(funcs) == 4
    for name, body in funcs.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in body, name
        regs = int(re.search(r"Used (\d+) registers", body).group(1))
        assert regs * 256 * 2 <= 65536, (name, regs)              # the register file holds the two CTAs the shared memory allows
    for line in log.splitlines():
        if re.search(r"C75(17|19|20)", line):
            assert "k1x_kernel" not in line, line


def test_sass_hgmma(ptxas_and_sass):
    _, sass = ptxas_and_sass
    funcs = {k: "\n".join(v) for k, v in _per_function(sass, r"Function : (\w+)").items() if "k1x_kernel" in k}
    assert len(funcs) == 4
    for name, body in funcs.items():
        cc = int(re.search(r"ILi\d+ELi\d+ELi\d+ELi\d+ELi\d+ELi(\d+)ELi\d+E", name).group(1))
        assert set(re.findall(r"HGMMA\.64x(\d+)x16\.F32\.BF16", body)) == {str(cc)}, name
