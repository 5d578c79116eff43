"""The C-ABI library loads on a CPU-only box, exports every symbol include/gp_bbmm.h declares, and refuses to
compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gp_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_loads():
    from gpytorch_b200 import build

    path = build.build()
    assert os.path.exists(path)
    from gpytorch_b200 import _lib

    lib = _lib.load()
    assert b"gpbbmm" in lib.gp_version()


def test_every_declared_symbol_is_exported_and_bound():
    from gpytorch_b200 import _lib

    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/gp_bbmm.h but not exported by libgpbbmm.so"
        assert s in _lib.PROTOTYPES, f"{s} has no ctypes prototype"
    for s in _lib.PROTOTYPES:
        assert s in syms, f"{s} bound but not declared in the header"


def test_sass_is_hopper_native():
    import shutil, subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = os.path.join(ROOT, "gpytorch_b200", "build", "kmv_tc.o")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "WARPGROUP.ARRIVE", "UBLKCP", "SYNCS.ARRIVE", "MUFU.EX2"):
        assert mnemonic in sass, f"{mnemonic} missing from the fused K.V kernel"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from gpytorch_b200 import _lib

    lib = _lib.load()
    h = C.c_void_p()
    st = lib.gp_plan_create(C.byref(h), 0, None)
    assert st == _lib.GP_E_CUDA
    assert "no CPU fallback" in _lib.last_error()
    from gpytorch_b200.engine import Plan

    with pytest.raises(RuntimeError, match="CUDA"):
        Plan(torch.rand(10, 2))


def test_null_plan_is_rejected_not_crashing():
    from gpytorch_b200 import _lib

    lib = _lib.load()
    assert lib.gp_plan_set_backend(None, 0) == _lib.GP_E_STATE
    assert lib.gp_plan_destroy(None) == _lib.GP_OK
