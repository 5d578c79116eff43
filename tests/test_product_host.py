"""Kernel products without a GPU: the kernel algebra (k1 * k2, flattening, parameter names, refusals, ScaleKernel over a product), the
oracle of tests/product_oracle.py against tests/golden/product_golden.npz (built from the reference's own covariance functions),
the host-side gradient bookkeeping of ProductKernelLinearOperator against fp64 autograd with the engine call replaced by the
oracle, the launch-geometry mirror, and the machine code of product_tc_kernel in the built library."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bilinear_oracle as bo
import product_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")


@pytest.fixture(scope="module")
def gp():
    import gpytorch_b200

    return gpytorch_b200


@pytest.fixture(scope="module")
def product_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "product_golden.npz"))


# ---- kernel algebra -----------------------------------------------------------------------------------------------------------------
def test_mul_builds_a_flat_product_kernel_with_the_reference_parameter_names(gp):
    k = gp.kernels
    a, b, c = k.RBFKernel(active_dims=[0, 1]), k.MaternKernel(nu=0.5, active_dims=[2]), k.ScaleKernel(k.MaternKernel(nu=2.5))
    p2 = a * b
    assert isinstance(p2, k.ProductKernel) and list(p2.kernels) == [a, b]
    p3 = p2 * c
    assert isinstance(p3, k.ProductKernel) and list(p3.kernels) == [a, b, c]                 # nested products are flattened
    assert list((c * p2).kernels) == [c, a, b]
    names = {n for n, _ in p3.named_parameters()}
    assert names == {"kernels.0.raw_lengthscale", "kernels.1.raw_lengthscale", "kernels.2.raw_outputscale",
                     "kernels.2.base_kernel.raw_lengthscale"}
    assert set(names) <= set(p3.state_dict())
    s = k.ScaleKernel(p2)
    assert {n for n, _ in s.named_parameters()} == {"raw_outputscale", "base_kernel.kernels.0.raw_lengthscale",
                                                    "base_kernel.kernels.1.raw_lengthscale"}


def test_product_kernel_refusals(gp):
    k = gp.kernels
    rbf, mat = k.RBFKernel(), k.MaternKernel(nu=1.5)
    with pytest.raises(NotImplementedError, match="sums that contain a ProductKernel"):
        rbf * mat + k.RBFKernel()
    with pytest.raises(NotImplementedError, match="sums that contain a ProductKernel"):
        k.RBFKernel() + k.ScaleKernel(rbf * mat)
    with pytest.raises(NotImplementedError, match="RBF / Matern kernels"):
        (rbf + mat) * k.RBFKernel()
    with pytest.raises(NotImplementedError, match="RBF / Matern kernels"):
        rbf * k.GridInterpolationKernel(k.RBFKernel(), grid_size=16, num_dims=1)
    with pytest.raises(NotImplementedError, match="RBF / Matern kernels"):
        rbf * k.MultitaskKernel(k.RBFKernel(), num_tasks=2)
    with pytest.raises(NotImplementedError, match="RBF / Matern kernels"):
        rbf * k.RBFKernelGrad()
    with pytest.raises(NotImplementedError, match="batched factors"):
        rbf * k.RBFKernel(batch_shape=torch.Size([2]))
    with pytest.raises(NotImplementedError, match="up to 4 factors"):
        rbf * mat * k.RBFKernel() * k.RBFKernel() * k.RBFKernel()
    with pytest.raises(NotImplementedError, match="batched inputs"):
        (rbf * mat)(torch.rand(2, 5, 3))


def test_operator_refusals_and_algebra(gp, monkeypatch):
    ops = gp.operators
    x = torch.rand(6, 3)
    mk = lambda kind, xs=x: ops.KernelLinearOperator(xs, None, kind, torch.tensor(0.5), torch.tensor(1.0))  # noqa: E731
    a, b = mk("rbf"), mk("matern12")
    p = a.mul(b)
    assert isinstance(p, ops.ProductKernelLinearOperator) and [o.kind for o in p.ops] == ["rbf", "matern12"]
    assert [o.kind for o in (p * mk("matern52")).ops] == ["rbf", "matern12", "matern52"]
    assert len({o._plan_slot for o in p.ops}) == 2 and p.input_tensors() == [] and p.solve_input_tensors() == []
    assert len(p.hyper_tensors()) == 4 and tuple(p.shape) == (6, 6)
    assert isinstance(p + ops.ConstantDiagLinearOperator(torch.tensor(0.1), 6), ops.AddedDiagLinearOperator)
    with pytest.raises(NotImplementedError, match="sums that contain products"):
        p + a
    with pytest.raises(NotImplementedError):
        a + p
    with pytest.raises(RuntimeError, match="cannot multiply kernels of shapes"):
        a.mul(mk("rbf", torch.rand(5, 3)))
    with pytest.raises(NotImplementedError, match="inputs of a kernel product"):
        a.mul(mk("rbf", torch.rand(6, 3, requires_grad=True)))
    with pytest.raises(NotImplementedError, match="2 to 4 factors"):
        ops.ProductKernelLinearOperator([a, b, a, b, a])
    assert not ops.LowRankUpdatedKernelLinearOperator.supports(p) and ops.LowRankUpdatedKernelLinearOperator.supports(a)
    pt = p.detach()
    assert isinstance(pt, ops.ProductKernelLinearOperator) and p.t() is p


# ---- oracle vs the reference's covariance functions -------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", sorted(po.GOLDEN_CASES))
def test_oracle_matches_golden_products_and_derivatives(product_golden, tag):
    n1, n2, d, factors = po.GOLDEN_CASES[tag]
    x1 = torch.from_numpy(product_golden[f"{tag}_x1"])
    x2 = torch.from_numpy(product_golden[f"{tag}_x2"]) if n2 else None
    K = po.dense(factors, x1, x2)
    assert torch.allclose(K, torch.from_numpy(product_golden[f"{tag}_K"]), rtol=1e-12, atol=1e-14)
    # dK/dl_f by fp64 autograd through the oracle, entry by entry, against the reference's backward
    for f in range(len(factors)):
        W = torch.from_numpy(product_golden[f"{tag}_dK{f}"])
        ls = [torch.tensor(fl[2], dtype=torch.float64, requires_grad=(i == f)) for i, fl in enumerate(factors)]
        Kf = po.dense([(k, dm, l, s) for (k, dm, _, s), l in zip(factors, ls)], x1, x2)
        probe = torch.randn(Kf.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(f))
        (g,) = torch.autograd.grad((probe * Kf).sum(), ls[f])
        assert g.item() == pytest.approx((probe * W).sum().item(), rel=1e-9, abs=1e-12)


# ---- host-side gradient bookkeeping ---------------------------------------------------------------------------------------------------
def test_gradient_split_matches_fp64_autograd(gp, monkeypatch):
    """ProductKernelLinearOperator._bilinear_derivative_list with the engine call replaced by the oracle: the flat (lengthscale
    gradients, dF/dS) result split per factor, dF/ds_f = S / s_f dF/dS."""
    ops = gp.operators
    n, m, s = 40, 30, 5
    g = torch.Generator().manual_seed(3)
    x1, x2 = torch.rand(n, 4, generator=g), torch.rand(m, 4, generator=g)
    factors = [("rbf", [0, 1], [0.5, 0.9], 1.3), ("matern12", [2], 0.7, 0.6), ("matern52", [1, 3], 1.1, 1.7)]
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    ref = po.bilinear_grads(factors, x1, x2, L, R)
    S = float(np.prod([float(bo.f32(f[3])) for f in factors]))
    # what gp_bilinear_grad returns on a product plan: the lengthscale gradients back to back and dF/dS = dF/ds_f s_f / S
    flat = [v for rl, _ in ref for v in rl.reshape(-1).tolist()]
    dS = ref[0][1].item() * float(bo.f32(factors[0][3])) / S
    for f, (_, rs) in zip(factors, ref):
        assert rs.item() * float(bo.f32(f[3])) / S == pytest.approx(dS, rel=1e-12)

    class FakePlan:
        def bilinear_grad(self, left, right):
            return flat, dS

    facs = [ops.KernelLinearOperator(x1[:, dm].contiguous(), x2[:, dm].contiguous(), k, torch.tensor(ls, dtype=torch.float32).reshape(1, -1),
                                     torch.tensor(os_, dtype=torch.float32)) for k, dm, ls, os_ in factors]
    op = ops.ProductKernelLinearOperator(facs)
    monkeypatch.setattr(op, "plan", lambda noise=0.0: FakePlan())
    out = op._bilinear_derivative_list(L, R)
    assert len(out) == 6
    for i, (f, (rl, rs)) in enumerate(zip(factors, ref)):
        assert out[2 * i].shape == facs[i].lengthscale.shape and out[2 * i + 1].shape == facs[i].outputscale.shape
        assert torch.allclose(out[2 * i].double().reshape(-1), rl.reshape(-1), rtol=1e-6)
        assert out[2 * i + 1].item() == pytest.approx(rs.item(), rel=1e-6)


def test_geometry_mirror_reaches_the_edges_of_the_gpu_tests():
    """The cases of test_gpu_product.py on 132 and 114 SMs: several splits, a ring wrap, KP = 128 on tensor cores, 136 not."""
    for n_sm in (132, 114):
        g = po.geometry(6000, 6000, [24, 2], ("tcgen05", "tcgen05"), n_sm)
        assert g["path"] == "tc" and g["KP"] == 96 and g["nsplit"] > 1 and g["T"] > po.ring_depth(96), g
        assert po.geometry(6000, 6000, [24, 2], ("simt", "simt"), n_sm)["nsplit"] > 1
        assert po.geometry(700, 900, [20, 20], ("tcgen05", "tcgen05"), n_sm)["KP"] == 128
        assert po.geometry(700, 700, [20, 21], ("tcgen05", "tcgen05"), n_sm)["path"] == "simt"
        assert po.geometry(500, 500, [2, 1, 4], ("auto",) * 3, n_sm)["path"] == "simt"


def test_oracle_bound_is_tight_enough_to_catch_a_dropped_factor():
    """The K.V bound is far below the change a wrong kernel makes: a product that forgets its second factor's polynomial."""
    x = torch.rand(200, 3, generator=torch.Generator().manual_seed(1))
    V = torch.randn(200, 4, generator=torch.Generator().manual_seed(2))
    factors = [("rbf", [0, 1], 0.6, 1.2), ("matern32", [2], 0.5, 0.8)]
    for path in ("tc", "simt"):
        ref, bnd = po.kv_and_bound(factors, x, None, V, path, 1, 4, noise=0.1)
        wrong, _ = po.kv_and_bound([factors[0], ("matern12", [2], 0.5, 0.8)], x, None, V, path, 1, 4, noise=0.1)
        assert float(((wrong - ref).abs() / bnd).median()) > 10


# ---- the built library -----------------------------------------------------------------------------------------------------------------
def _tool():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available (python -m gpytorch_b200.build)")
    return tool


def test_library_exports_the_product_entry_point(gp):
    from gpytorch_b200 import _lib

    assert "gp_plan_set_product" in _lib.PROTOTYPES and _lib.GP_BACKEND_PRODUCT == 7
    hdr = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert "int gp_plan_set_product(gp_plan* plan, gp_plan* const* factors, int n_factors);" in hdr and "GP_BACKEND_PRODUCT = 7" in hdr
    if os.path.exists(LIB):
        assert hasattr(_lib.load(), "gp_plan_set_product")


def test_product_tc_kernel_machine_code():
    """product_tc_kernel is wgmma / bulk-TMA code: GEMM1 from shared-memory descriptors, GEMM2 with the covariance tile as the
    register A operand; every instantiation has ONE MUFU.EX2 per covariance entry -- 32 per thread and tile, in the one epilogue the
    tile loop inlines twice (turn 0 and the loop body: 64 in the SASS) -- and one MUFU.SQRT per entry and Matern factor."""
    r = subprocess.run([_tool(), "-sass", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    bodies, name = {}, None
    for line in r.stdout.splitlines():
        if "Function :" in line:
            m = re.search(r"product_tc_kernelILb([01])ELb([01])E", line)
            name = (int(m.group(1)), int(m.group(2))) if m else None
            if name:
                bodies[name] = []
        elif name:
            bodies[name].append(line)
    assert sorted(bodies) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    for (ra, rb), lines in bodies.items():
        body = "\n".join(lines)
        assert "UBLKCP" in body
        assert re.search(r"HGMMA\.64x64x8\.F32\.TF32 R\d+, gdesc", body)
        assert re.search(r"HGMMA\.64x32x8\.F32\.TF32 R\d+, R\d+, gdesc", body) and re.search(r"HGMMA\.64x16x8\.F32\.TF32 R\d+, R\d+, gdesc", body)
        assert len(re.findall(r"MUFU\.EX2", body)) == 2 * 32, (ra, rb)
        assert len(re.findall(r"MUFU\.SQRT", body)) == 2 * 32 * ((not ra) + (not rb)), (ra, rb)


def test_product_kernels_resource_usage():
    """<= 128 registers per thread for product_tc_kernel (384-thread CTAs, one per SM, as kmv_tc_kernel) and no local memory in the
    instantiations with a Matern factor -- the products no other operator expresses; RBF x RBF (an ARD RBF) may spill a few
    bytes."""
    r = subprocess.run([_tool(), "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function" in line and "product_tc_kernel" in line:
            reg = int(re.search(r"REG:(\d+)", lines[i + 1]).group(1))
            stack = int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1))
            assert reg <= 128, (line, reg)
            assert stack == 0 or ("ILb1ELb1E" in line and stack <= 16), (line, stack)
            seen += 1
    assert seen == 4
