"""CPU check that the fused K.V kernels' wgmma chains are pipelined: ptxas must not serialise them (C7511 / C7512 / C7515:
"wgmma.mma_async instructions are serialized ..."), and in the SASS of every kmv_tc_kernel and product_tc_kernel instance (the
one pipeline of kmv_tc.cu, with one GEMM1 operand or two) the 16 HGMMAs of one tile's GEMM2 (8 x 64x32x8 + 8 x 64x16x8) must
not be separated by a WARPGROUP.DEPBAR (a wait for the previous wgmma)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
SRC = os.path.join(ROOT, "gpytorch_b200", "csrc", "kmv_tc.cu")
KERNELS = {"kmv_tc_kernel": 8, "product_tc_kernel": 4}   # instantiations of each entry in the library


def _tool(name):
    t = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return t if os.path.exists(t) else None


def test_ptxas_does_not_serialise_the_wgmma_chains(tmp_path):
    nvcc = os.environ.get("NVCC") or _tool("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v",
           "-c", SRC, "-o", str(tmp_path / "kmv_tc.o")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    for name in KERNELS:
        assert name in log, name
    bad = [line for line in log.splitlines() if re.search(r"\(C751[125]\)", line) and any(k in line for k in KERNELS)]
    assert not bad, "\n".join(bad)


def _kernel_bodies(sass_text):
    bodies, cur = [], None
    for line in sass_text.splitlines():
        if "Function :" in line:
            name = next((k for k in KERNELS if k in line), None)
            cur = [] if name else None
            if name:
                bodies.append((name, cur))
        elif cur is not None:
            cur.append(line)
    return bodies


def test_gemm2_hgmmas_are_issued_back_to_back():
    tool = _tool("cuobjdump")
    if not tool or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    bodies = _kernel_bodies(r.stdout)
    counts = {k: sum(1 for name, _ in bodies if name == k) for k in KERNELS}
    assert counts == KERNELS, counts
    for name, body in bodies:
        ops = [ln for ln in body if re.search(r"HGMMA\.64x(32|16)x8\.F32\.TF32|WARPGROUP\.DEPBAR", ln)]
        starts = [i for i, ln in enumerate(ops) if re.search(r"HGMMA\.64x32x8\.F32\.TF32 .*RZ, !UPT", ln)]
        assert starts, f"{name}: no GEMM2 chain start (64x32x8 with a zero accumulator) found"
        for i in starts:
            chain = ops[i:i + 16]
            assert len(chain) == 16 and all("HGMMA" in ln for ln in chain), f"{name}: GEMM2 HGMMAs separated by WARPGROUP.DEPBAR:\n" + \
                "\n".join(ln.strip() for ln in ops[i:i + 20])
