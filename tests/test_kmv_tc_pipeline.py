"""CPU check that the fused K.V kernel's wgmma chains are pipelined: ptxas must not serialise them (C7511 / C7512 / C7515:
"wgmma.mma_async instructions are serialized ..."), and in the SASS of every kmv_tc_kernel instance the 16 HGMMAs of one
tile's GEMM2 (8 x 64x32x8 + 8 x 64x16x8) must not be separated by a WARPGROUP.DEPBAR (a wait for the previous wgmma)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
SRC = os.path.join(ROOT, "gpytorch_b200", "csrc", "kmv_tc.cu")


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
    assert "kmv_tc_kernel" in log
    bad = [line for line in log.splitlines() if re.search(r"\(C751[125]\)", line) and "kmv_tc_kernel" in line]
    assert not bad, "\n".join(bad)


def _kernel_bodies(sass_text):
    bodies, cur = [], None
    for line in sass_text.splitlines():
        if "Function :" in line:
            cur = [] if "kmv_tc_kernel" in line else None
            if cur is not None:
                bodies.append(cur)
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
    assert len(bodies) == 8, len(bodies)
    for body in bodies:
        ops = [ln for ln in body if re.search(r"HGMMA\.64x(32|16)x8\.F32\.TF32|WARPGROUP\.DEPBAR", ln)]
        starts = [i for i, ln in enumerate(ops) if re.search(r"HGMMA\.64x32x8\.F32\.TF32 .*RZ, !UPT", ln)]
        assert starts, "no GEMM2 chain start (64x32x8 with a zero accumulator) found"
        for i in starts:
            chain = ops[i:i + 16]
            assert len(chain) == 16 and all("HGMMA" in ln for ln in chain), "GEMM2 HGMMAs separated by WARPGROUP.DEPBAR:\n" + \
                "\n".join(ln.strip() for ln in ops[i:i + 20])
