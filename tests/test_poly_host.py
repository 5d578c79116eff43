"""CPU checks of the polynomial kernel: the reference's golden covariances against the fp64 oracle, mutants of the engine's
formula that must fall outside the K.V bound (a diagonal forced to c^p, centred inputs, a dropped offset, power p - 1), the class
surface and the wrappers that keep power and offset, the refusals, and the compiled kernels (no stack, no spills, wgmma chains
not serialised)."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import poly_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
GOLD = os.path.join(ROOT, "tests", "golden", "poly_golden.npz")


def test_golden_against_the_oracle():
    g = np.load(GOLD)
    for ci in range(int(g["ncases"])):
        p, d, n1, n2, B, cancel = (int(v) for v in g[f"c{ci}_meta"])
        x1, x2, off = (torch.from_numpy(g[f"c{ci}_{k}"]) for k in ("x1", "x2", "offset"))
        W = torch.from_numpy(g[f"c{ci}_W"])
        for b in range(max(B, 1)):
            sl = (lambda t: t[b]) if B else (lambda t: t)
            c = float(sl(off).reshape(-1)[0])
            K = po.kernel(sl(x1), sl(x2), p, c)
            assert torch.allclose(K, torch.from_numpy(sl(g[f"c{ci}_K"])), rtol=1e-12, atol=1e-12)
            assert torch.allclose(po.kernel(sl(x1), sl(x1), p, c), torch.from_numpy(sl(g[f"c{ci}_Kxx"])), rtol=1e-12, atol=1e-12)
            assert torch.allclose(po.diag(sl(x1), p, c), torch.from_numpy(sl(g[f"c{ci}_diag"])), rtol=1e-12, atol=1e-12)
            gc, _ = po.grads(sl(x1), sl(x2), p, c, sl(W))
            assert abs(float(gc) - float(sl(g[f"c{ci}_goffset"]).reshape(-1)[0])) <= 1e-9 * max(1.0, abs(float(gc)))
        if cancel:   # the base cancels at (0, 0): k is tiny there, the bound in m_ij is not
            pair, _ = po.entry_bound(torch.from_numpy(g[f"c{ci}_x1"]).reshape(-1, d)[:1], torch.from_numpy(g[f"c{ci}_x2"]).reshape(-1, d)[:1], p,
                                     float(off.reshape(-1)[0]), "tc")
            assert float(pair[0, 0]) > abs(float(g[f"c{ci}_K"].reshape(-1)[0]))


@pytest.mark.parametrize("path", ["tc", "simt"])
def test_mutants_fall_outside_the_bound(path):
    gen = torch.Generator().manual_seed(3)
    n, d, p, c = 200, 3, 3, 0.5
    x = (torch.rand(n, d, generator=gen) * 2 - 1) + 0.3
    V = torch.randn(n, 4, generator=gen)
    ref = po.kernel(x, x, p, c) @ V.double()
    bnd = po.kmv_bound(x, x, p, c, V, 1.0, path, 1, 4)
    K = po.kernel(x, x, p, c)
    diag_forced = K.clone()
    diag_forced.fill_diagonal_(c ** p)
    xc = x - x.mean(0)
    mutants = {"diag c^p": diag_forced, "centred": po.kernel(xc, xc, p, c), "no offset": po.kernel(x, x, p, 0.0),
               "power p-1": po.kernel(x, x, p - 1, c)}
    for name, Km in mutants.items():
        assert bool(((Km @ V.double() - ref).abs() > bnd).any()), name
    assert bool(((K @ V.double() - ref).abs() <= bnd).all())


def test_class_surface_and_wrapper_methods():
    import gpytorch_b200 as gp
    from gpytorch_b200.operators import PolynomialKernelLinearOperator, SumKernelLinearOperator

    k = gp.kernels.PolynomialKernel(2)
    assert k.power == 2 and tuple(k.raw_offset.shape) == (1,) and type(k.raw_offset_constraint).__name__ == "Positive"
    k.offset = 0.7
    assert abs(float(k.offset) - 0.7) < 1e-6
    assert gp.kernels.PolynomialKernel(3.0).power == 3 and gp.kernels.PolynomialKernel(torch.tensor([4])).power == 4
    for bad in (2.5, "2", torch.tensor([1, 2])):
        with pytest.raises(NotImplementedError):
            gp.kernels.PolynomialKernel(bad)
    with pytest.raises(NotImplementedError):
        gp.kernels.PolynomialKernel(2, offset_prior=object())
    assert not isinstance(k, gp.kernels._StationaryKernel)
    assert tuple(gp.kernels.PolynomialKernel(2, batch_shape=torch.Size([3])).raw_offset.shape) == (3, 1)
    with pytest.raises(NotImplementedError):
        gp.kernels.PolynomialKernel(2, batch_shape=torch.Size([2, 2]))
    x = torch.randn(6, 3)
    with pytest.raises(NotImplementedError, match="PolynomialKernel"):
        k.forward(x, x, last_dim_is_batch=True)
    op = gp.kernels.ScaleKernel(gp.kernels.ScaleKernel(k))(x)
    assert isinstance(op, PolynomialKernelLinearOperator) and op.power == 2 and abs(float(op.offset) - 0.7) < 1e-6
    ka = gp.kernels.PolynomialKernel(3, active_dims=[0, 2])
    assert ka(x).x1.shape[1] == 2
    s = (gp.kernels.ScaleKernel(gp.kernels.PolynomialKernel(2)) + gp.kernels.ScaleKernel(gp.kernels.RBFKernel()))(x)
    assert isinstance(s, SumKernelLinearOperator) and isinstance(s.ops[0], PolynomialKernelLinearOperator)
    s2 = gp.kernels.ScaleKernel(gp.kernels.PolynomialKernel(4) + gp.kernels.RBFKernel())(x)
    assert s2.ops[0].power == 4
    for o in (op.detach(), op._transpose_nonbatch(), op[1:4, :], op.with_outputscale(torch.tensor(2.0))):
        assert isinstance(o, PolynomialKernelLinearOperator) and o.power == 2 and abs(float(o.offset) - 0.7) < 1e-6
    assert gp.operators.LowRankUpdatedKernelLinearOperator.supports(op)
    with pytest.raises(NotImplementedError, match="PolynomialKernel"):
        op.mul(gp.operators.KernelLinearOperator(x, None, "rbf", torch.tensor(1.0)))
    with pytest.raises(NotImplementedError, match="ProductKernel factors"):
        gp.kernels.ProductKernel(gp.kernels.PolynomialKernel(2), gp.kernels.RBFKernel())
    with pytest.raises(NotImplementedError):
        gp.kernels.MultitaskKernel(gp.kernels.PolynomialKernel(2), num_tasks=2)(x)


def test_header_and_api_document_the_call():
    h = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert "GP_POLY = 5" in h
    assert re.search(r"int gp_plan_set_hypers_poly\(gp_plan\* plan, int power, float offset, float outputscale, float noise\);", h)
    api = open(os.path.join(ROOT, "gpytorch_b200", "csrc", "api.cu")).read()
    assert "call gp_plan_set_hypers_poly" in api


def _tool(name):
    t = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return t if os.path.exists(t) else None


def test_new_kv_kernels_have_no_local_memory():
    tool = _tool("cuobjdump")
    if not tool or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = {"poly_tc_kernel": 0, "poly_simt_kernel": 0}
    for i, line in enumerate(lines):
        if "Function" not in line:
            continue
        for key in seen:
            if key in line:
                seen[key] += 1
                local = int(re.search(r"LOCAL:(\d+)", lines[i + 1]).group(1))
                assert local == 0, line
                m = re.search(r"poly_simt_kernelILi(\d+)E", line)
                if key == "poly_tc_kernel" or (m and int(m.group(1)) <= 32):   # every width the tensor-core path leaves to SIMT
                    assert int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1)) == 0, line
    assert seen == {"poly_tc_kernel": 2, "poly_simt_kernel": 10}, seen


def test_poly_wgmma_chains_are_not_serialised(tmp_path):
    nvcc = os.environ.get("NVCC") or _tool("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "gpytorch_b200", "csrc", "kmv_tc.cu")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v",
           "-cubin", src, "-o", str(tmp_path / "kmv_tc.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert "poly_tc_kernel" in log
    assert not [ln for ln in log.splitlines() if re.search(r"\(C751[125]\)", ln)]
    sass = subprocess.run([_tool("cuobjdump"), "-sass", str(tmp_path / "kmv_tc.cubin")], capture_output=True, text=True, timeout=300).stdout
    bodies, cur = [], None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = [] if "poly_tc_kernel" in line else None
            if cur is not None:
                bodies.append(cur)
        elif cur is not None:
            cur.append(line)
    assert len(bodies) == 2
    for body in bodies:
        ops = [ln for ln in body if re.search(r"HGMMA\.64x(32|16)x8\.F32\.TF32|WARPGROUP\.DEPBAR", ln)]
        starts = [i for i, ln in enumerate(ops) if re.search(r"HGMMA\.64x32x8\.F32\.TF32 .*RZ, !UPT", ln)]
        assert starts
        for i in starts:
            assert all("HGMMA" in ln for ln in ops[i:i + 16]) and len(ops[i:i + 16]) == 16
        assert "MUFU" not in "\n".join(body)   # the epilogue is FMA-pipe only
