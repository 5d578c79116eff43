"""CPU check of the shipped library's machine code (cuobjdump works without a GPU): the hot path must really be wgmma / bulk-TMA /
mbarrier code for sm_90a (SASS HGMMA, UBLKCP, SYNCS) and must not have regressed to slow constructs (fp32 atomicAdd on shared
memory = an ATOMS.CAST compare-and-swap loop)."""
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpytorch_b200", "lib", "libgpbbmm.so")


@pytest.fixture(scope="module")
def sass():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(LIB):
        pytest.skip("libgpbbmm.so not built (python -m gpytorch_b200.build)")
    r = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def _function_bodies(sass_text, name_part):
    out, keep = [], False
    for line in sass_text.splitlines():
        if "Function :" in line:
            keep = name_part in line
        elif keep:
            out.append(line)
    return "\n".join(out)


def test_library_is_sm90a_wgmma_code(sass):
    assert "sm_90a" in sass
    counts = {m: len(re.findall(m, sass)) for m in ("HGMMA", "WARPGROUP.ARRIVE", "UBLKCP", r"SYNCS\.ARRIVE", r"MUFU\.EX2")}
    # wgmma.mma_async / wgmma.fence / cp.async.bulk / mbarrier.arrive / ex2.approx of the fused K.V kernels (8 instantiations)
    assert counts["HGMMA"] >= 8 * 18 and counts["WARPGROUP.ARRIVE"] >= 8, counts
    assert counts["UBLKCP"] > 20 and counts[r"SYNCS\.ARRIVE"] > 20 and counts[r"MUFU\.EX2"] > 200, counts


def test_fused_kernel_and_ski_kernels_have_the_expected_instructions(sass):
    kv = _function_bodies(sass, "kmv_tc_kernel")
    assert "UBLKCP" in kv and "MUFU.EX2" in kv
    # GEMM1 from shared memory, GEMM2 with the covariance tile as the register A operand (HGMMA R.., R.., gdesc)
    assert re.search(r"HGMMA\.64x64x8\.F32\.TF32 R\d+, gdesc", kv)
    assert re.search(r"HGMMA\.64x32x8\.F32\.TF32 R\d+, R\d+, gdesc", kv) and re.search(r"HGMMA\.64x16x8\.F32\.TF32 R\d+, R\d+, gdesc", kv)
    mode = _function_bodies(sass, "ski_mode_kernel")
    assert re.search(r"HMMA\.1688\.F32\.TF32", mode), "the SKI mode product must run as a 3xTF32 tensor-core product"
    for k in ("ski_scatter_tiled_kernel", "ski_gather_tiled_kernel"):
        body = _function_bodies(sass, k)
        assert body and "ATOMS.CAST" not in body, f"{k}: fp32 shared-memory atomics compile to a compare-and-swap loop"
    assert "REDG.E.ADD.F32x4" in _function_bodies(sass, "ski_scatter_tiled_kernel")


def test_hot_kernels_fit_their_register_budget_without_spills():
    """Resource usage of the hot kernels: the fused K.V kernel runs two 256-thread CTAs per SM (<= 128 registers per thread) and
    must not spill; the SKI scatter / mode kernels likewise (a local-memory array in a tiled scatter costs GBs of L2 traffic)."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = {"kmv_tc_kernel": 0, "ski_scatter_tiled_kernelILi3": 0, "ski_mode_kernel": 0, "cg_finishv_wtv_kernel": 0, "cg_update_precond_kernel": 0}
    for i, line in enumerate(lines):
        if "Function" not in line:
            continue
        for key in seen:
            if key in line:
                usage = lines[i + 1]
                reg = int(re.search(r"REG:(\d+)", usage).group(1))
                stack = int(re.search(r"STACK:(\d+)", usage).group(1))
                assert stack == 0, f"{line.strip()}: {stack} bytes of local memory"
                if key == "kmv_tc_kernel":
                    assert reg <= 128, f"{line.strip()}: {reg} registers x 2 x 256 threads do not fit one SM"
                seen[key] += 1
    assert all(v > 0 for v in seen.values()), seen
