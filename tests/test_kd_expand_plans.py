"""Host-side checks (no GPU) of KD with the on-chip expand conv (dwse_x_kernel): the instances tools/route_plan_dump.cu prints,
and what ptxas and the SASS show for them in inst_dwse.cu."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc")
EXE = os.path.join(ROOT, "build_tmp", "route_plan_dump_kdx")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SMEM_OPTIN = 227 * 1024          # dynamic + static shared memory one CTA may use on sm_90
CEXP = {7: 480, 9: 480, 10: 672, 12: 672, 13: 1152, 16: 1152}
CIN = {7: 80, 9: 80, 10: 112, 12: 112, 13: 192, 16: 192}


@pytest.fixture(scope="module")
def kdx():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run([NVCC, "-std=c++17", "-arch=sm_90a", "-o", EXE, os.path.join(ROOT, "tools", "route_plan_dump.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([EXE, "256"], capture_output=True, text=True, check=True).stdout
    rows = {}
    for line in out.splitlines():
        m = re.search(r"kdx b(\d+) cc (\d+) cin (\d+) threads (\d+) halves (\d+) nwg (\d+) smem (\d+) chunks (\d+) ctas_per_sm (\d+)", line)
        if m:
            rows[int(m.group(1))] = dict(zip("cc cin threads halves nwg smem chunks ctas".split(), (int(v) for v in m.groups()[1:])))
    return rows


def test_instances(kdx):
    assert sorted(kdx) == sorted(CEXP)                     # one line per distinct late-block shape
    for b, r in kdx.items():
        assert CEXP[b] % r["cc"] == 0 and r["chunks"] == CEXP[b] // r["cc"], b
        assert r["cin"] == CIN[b] and r["threads"] == 256, b
        assert r["smem"] + 256 <= SMEM_OPTIN, b             # + the kernel's static barriers
        assert r["nwg"] % 16 == 0 and r["nwg"] <= 128, b
    assert kdx[7]["halves"] == 4 and kdx[13]["halves"] == 1
    # CTAs per SM the instances are compiled for: their shared memory fits that many (1 KB reserved per CTA); two only for the
    # 14x14 / 3x3 instance (blocks 7-8), whose registers test_ptxas_clean checks
    for b, r in kdx.items():
        assert r["ctas"] * (r["smem"] + 256 + 1024) <= 228 * 1024, b
    assert {b: r["ctas"] for b, r in kdx.items()} == {7: 2, 9: 1, 10: 1, 12: 1, 13: 1, 16: 1}


@pytest.fixture(scope="module")
def ptxas_and_sass(tmp_path_factory):
    d = tmp_path_factory.mktemp("kdx")
    obj = str(d / "inst_dwse.o")
    r = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", "-o", obj,
                        os.path.join(CSRC, "inst_dwse.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True)
    assert sass.returncode == 0, sass.stderr
    return r.stderr, sass.stdout


def _per_function(text, start_pat):
    """Split ptxas / cuobjdump output into {mangled function name: its lines}."""
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
    funcs = _per_function(log, r"Compiling entry function '(\w+)'")
    kdx = {k: v for k, v in funcs.items() if "dwse_x_kernel" in k}
    assert len(kdx) == 6
    for name, lines in kdx.items():
        body = "\n".join(lines)
        assert "0 bytes spill stores, 0 bytes spill loads" in body, name
        regs = int(re.search(r"Used (\d+) registers", body).group(1))
        # the register file (64 K per SM) holds the CTAs per SM the shared memory allows: two for <3,1,14,32,80>, else one
        ctas = 2 if "ILi3ELi1ELi14ELi32ELi80E" in name else 1
        assert regs * 256 * ctas <= 65536, (name, regs)
    # wgmma serialisation warnings are printed outside the per-function blocks: none may name a fused instance
    for line in log.splitlines():
        if re.search(r"C75(17|19|20)", line):
            assert "dwse_x_kernel" not in line, line


def test_sass_hgmma(ptxas_and_sass):
    _, sass = ptxas_and_sass
    funcs = _per_function(sass, r"Function : (\w+)")
    kdx = {k: "\n".join(v) for k, v in funcs.items() if "dwse_x_kernel" in k}
    assert len(kdx) == 6
    for name, body in kdx.items():
        m = re.search(r"ILi(\d)ELi(\d)ELi(\d+)ELi(\d+)ELi(\d+)E", name)
        hin, cc = int(m.group(3)), int(m.group(4))
        nwg = cc if hin == 14 else cc // 2
        assert re.search(r"HGMMA\.64x%dx16\.F32\.BF16" % nwg, body), (name, nwg)
