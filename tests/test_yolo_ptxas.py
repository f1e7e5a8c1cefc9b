"""The detector's kernels as ptxas builds them (no GPU needed): no spills, and wgmma neither fenced by injected warpgroup
arrives (C7519) nor serialised (C7520) in the first conv and the implicit-GEMM conv."""
import os
import re
import subprocess
import tempfile

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "headposeestimation-whenet_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_yolo_kernels_do_not_spill_or_serialise_wgmma():
    from whenet_b200 import build
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas=-v", "-c", "-o", os.path.join(tmp, "y.o"), os.path.join(CSRC, "inst_yolo.cu")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert not re.search(r"C75(19|20)", log), [l for l in log.splitlines() if "C75" in l]
    entries = re.split(r"Compiling entry function '", log)[1:]
    seen = set()
    for e in entries:
        name = e.split("'", 1)[0]
        if "yolo" not in name:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.group(1) == "0" and m.group(2) == "0", "%s spills" % name
        seen.add(re.sub(r"I.*", "", name.split("yolo")[1]))
    kinds = {k for k in ("conv_igemm_kernel", "yolo_conv0_kernel", "yolo_decode_nms_kernel", "letterbox_h_kernel", "letterbox_v_kernel")
             if any(k in e.split("'", 1)[0] for e in entries)}
    assert len(kinds) == 5, kinds
