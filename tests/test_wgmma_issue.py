"""How the tensor-core units issue their warpgroup MMAs (no GPU needed: ptxas diagnostics and the SASS of the library).

Every tile issues ONE wgmma.m64nNk16 per 64-row half and K step for its full width N, in straight runs that ptxas neither
fences with injected warpgroup arrives (C7519) nor serialises (C7520).  Narrow 16-column pieces behind runtime guards
brought both back, and with them one WARPGROUP.DEPBAR per HGMMA in the warp-specialised K2 kernel.
"""
import os
import re
import shutil
import subprocess
import tempfile
from collections import Counter

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# the units that carry wgmma: the 1x1 kernels (pw_tc2, pw_tc3, K2) and the one with the fp32 parity kernel and the stem
TC_UNITS = ["inst_pw.cu", "whenet_api.cu"]


def _ptxas_log():
    from whenet_b200 import build
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        procs = [subprocess.Popen([NVCC] + build.NVCC_FLAGS + ["-Xptxas=-v", "-c", "-o", os.path.join(tmp, u + ".o"), os.path.join(CSRC, u)],
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for u in TC_UNITS]
        logs = []
        for u, p in zip(TC_UNITS, procs):
            out, err = p.communicate()
            assert p.returncode == 0, "nvcc failed on %s:\n%s" % (u, err[-2000:])
            logs.append(out + err)
    return "\n".join(logs)


def test_ptxas_does_not_serialise_or_fence_wgmma():
    log = _ptxas_log()
    serialised = sorted(set(re.findall(r"\(C7520\).*?'(\w+)'", log)))
    assert not serialised, "wgmma serialised (C7520) in %s" % serialised
    fenced = Counter(re.search(r"(pw_tc2_kernel|pw_tc3_kernel|k2_kernel)", f).group(1)
                     for f in re.findall(r"\(C7519\).*?'(\w+)'", log) if re.search(r"pw_tc2_kernel|pw_tc3_kernel|k2_kernel", f))
    assert not fenced, "ptxas injected warpgroup arrives in the 1x1 kernels: %s" % dict(fenced)


def _sass_functions():
    from whenet_b200 import build
    cu = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cu):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cu, "-sass", build.build_lib()], capture_output=True, text=True).stdout
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        yield name.strip(), body


@pytest.mark.parametrize("kernel", ["k2_kernel", "pw_tc2_kernel"])
def test_sass_issues_full_width_hgmma(kernel):
    seen = Counter()
    for name, body in _sass_functions():
        if kernel not in name:
            continue
        m = re.search(r"Li(\d+)EEEv", name)                          # last template argument: the tile's MMA width
        assert m, "%s: the MMA width is not a template argument" % name
        width = int(m.group(1))
        shapes = Counter(re.findall(r"HGMMA\.64x(\d+)x16", body))
        assert set(shapes) == {str(width)}, "%s: HGMMA shapes %s" % (name, dict(shapes))
        if kernel == "k2_kernel":
            depbars = len(re.findall(r"WARPGROUP\.DEPBAR", body))
            assert depbars < sum(shapes.values()) // 4, "%s: %d DEPBAR for %d HGMMA" % (name, depbars, sum(shapes.values()))
        seen[width] += 1
    assert kernel != "k2_kernel" or set(seen) == {16, 32, 48, 64}, dict(seen)
    assert kernel != "pw_tc2_kernel" or set(seen) == {16, 32, 48, 64, 96, 128}, dict(seen)
