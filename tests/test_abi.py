"""The C-ABI library: loads, exports every symbol the header declares, and fails loudly without a GPU
(no CPU fallback anywhere on the product path)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT


def _declared():
    with open(os.path.join(ROOT, "include", "whenet_b200.h")) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(whenet_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_header_symbols():
    from whenet_b200 import _lib, build
    path = build.build_lib()
    assert os.path.exists(path)
    L = _lib.load()
    decl = _declared()
    assert len(decl) >= 17
    for name in decl:
        assert hasattr(L, name), "missing export %s" % name
    assert sorted(_lib.EXPORTS) == decl
    assert b"sm_90a" in L.whenet_version()


def test_sass_contains_wgmma():
    """The shipped binary really carries Hopper warpgroup tensor-core code (HGMMA = wgmma.mma_async)."""
    import shutil
    import subprocess
    from whenet_b200 import build
    cu = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cu):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cu, "-sass", build.build_lib()], capture_output=True, text=True).stdout
    assert "HGMMA" in sass
    assert "sm_90a" in sass


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="this is the no-GPU behaviour")
def test_no_gpu_means_error_not_fallback():
    import whenet_b200
    from whenet_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    rc = L.whenet_create(C.byref(h), 0, 8, 0)
    assert rc == -2 and len(L.whenet_last_error()) > 0
    with pytest.raises(whenet_b200.WhenetError):
        whenet_b200.WHENet(None)


def test_argument_validation_without_gpu():
    from whenet_b200 import _lib
    L = _lib.load()
    assert L.whenet_create(None, 0, 8, 0) == -1
    h = C.c_void_p()
    assert L.whenet_create(C.byref(h), 0, 0, 0) == -1 and b"max_batch" in L.whenet_last_error()
    assert L.whenet_create(C.byref(h), 0, 8, 7) == -1 and b"precision" in L.whenet_last_error()
    out = np.zeros(3, np.float32)
    assert L.whenet_forward_u8(None, None, 1, 0, out.ctypes.data, None, 0) == -1
    assert L.whenet_launch_count(None) == 0
    L.whenet_destroy(None)


def test_shape_errors_are_keras_like():
    from whenet_b200.whenet import WHENet
    with pytest.raises(ValueError, match="expected input_1 to have shape"):
        WHENet._check_shape(np.zeros((2, 224, 224), np.uint8))
    WHENet._check_shape(np.zeros((0, 224, 224, 3), np.uint8))


def test_drop_in_module_name():
    """`from whenet import WHENet` (reference demo.py:3) resolves to the native class."""
    import whenet
    import whenet_b200
    assert whenet.WHENet is whenet_b200.WHENet
