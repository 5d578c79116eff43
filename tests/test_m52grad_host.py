"""CPU checks of the Matern-5/2 derivative-observation layer (Matern52KernelGrad): the fp64 oracle against the reference's own
Matern52KernelGrad.forward and its known answer (tests/golden/m52grad_golden.npz) and against autograd second derivatives of the
Matern-5/2; the kernel class (parameters, diag, the refusals that need no device); and the machine code of its kernels in deriv.cu (no
stack or local memory in any instantiation serving d <= 16) next to the unchanged RBF derivative kernels and fused K.V register counts."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import m52grad_oracle as mo

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "gpytorch_b200", "lib", "libgpbbmm.so")
GOLD = np.load(os.path.join(HERE, "golden", "m52grad_golden.npz"))


@pytest.mark.parametrize("d", [1, 2, 5])
@pytest.mark.parametrize("ard", [False, True])
def test_oracle_matches_reference_golden(d, ard):
    tag = f"d{d}_{'ard' if ard else 'iso'}"
    ls = torch.tensor(GOLD[f"{tag}_ls"])
    x1, x2 = torch.tensor(GOLD[f"{tag}_x1"]), torch.tensor(GOLD[f"{tag}_x2"])
    assert torch.allclose(mo.m52grad_dense(x1, x1, ls), torch.tensor(GOLD[f"{tag}_square"]), rtol=0, atol=1e-12)
    assert torch.allclose(mo.m52grad_dense(x1, x2, ls), torch.tensor(GOLD[f"{tag}_cross"]), rtol=0, atol=1e-12)   # a coincident pair
    assert torch.allclose(mo.m52grad_diag(x1.size(0), ls, d), torch.tensor(GOLD[f"{tag}_diag"]), rtol=0, atol=1e-12)
    s = 1.7
    assert torch.allclose(mo.m52grad_dense(x1, x2, ls, s), s * torch.tensor(GOLD[f"{tag}_cross"]), rtol=0, atol=2e-12)


def test_oracle_matches_reference_known_answer():
    """test/kernels/test_matern52_kernel_grad.py::test_kernel at the default lengthscale ln 2: its fp32 matrix, and the reference's
    forward in fp64."""
    a, b, ls = torch.tensor(GOLD["ka_a"]), torch.tensor(GOLD["ka_b"]), torch.tensor(GOLD["ka_ls"])
    assert abs(float(ls) - math.log(2.0)) < 1e-15
    K = mo.m52grad_dense(a, b, ls)
    assert torch.allclose(K, torch.tensor(GOLD["ka_reference_fp64"]), rtol=0, atol=1e-12)
    assert float((K - torch.tensor(GOLD["ka_expected"])).abs().max()) <= 5e-7


@pytest.mark.parametrize("ard", [False, True])
def test_oracle_matches_autograd_derivatives(ard):
    """[a, 0] = dk/dx_a, [0, b] = dk/dx'_b, [a, b] = d2k / dx_a dx'_b of k = (1 + rho + rho^2 / 3) exp(-rho), rho = sqrt(5) |x - x'| / l
    (pairs at distance > 0: the Hessian of the autograd form is 0/0 at D = 0, where the table gives (5/3) / l_a^2)."""
    g = torch.Generator().manual_seed(5)
    d = 3
    ls = torch.tensor([0.4, 0.7, 1.1], dtype=torch.float64) if ard else torch.tensor(0.6, dtype=torch.float64)
    x1 = torch.rand(4, d, generator=g, dtype=torch.float64)
    x2 = torch.rand(3, d, generator=g, dtype=torch.float64)
    K = mo.m52grad_dense(x1, x2, ls)

    def k(a, b):
        rho = math.sqrt(5) * torch.sqrt((((a - b) / ls) ** 2).sum())
        return (1 + rho + rho ** 2 / 3) * torch.exp(-rho)

    for i in range(4):
        for j in range(3):
            a, b = x1[i].clone(), x2[j].clone()
            blk = K[i * (d + 1):(i + 1) * (d + 1), j * (d + 1):(j + 1) * (d + 1)]
            ga = torch.autograd.functional.jacobian(lambda u: k(u, b), a)
            gb = torch.autograd.functional.jacobian(lambda v: k(a, v), b)
            H = torch.autograd.functional.jacobian(lambda v: torch.autograd.functional.jacobian(lambda u: k(u, v), a, create_graph=True), b)
            assert torch.allclose(blk[0, 0], k(a, b), atol=1e-14)
            assert torch.allclose(blk[1:, 0], ga, atol=1e-12)
            assert torch.allclose(blk[0, 1:], gb, atol=1e-12)
            assert torch.allclose(blk[1:, 1:], H, atol=1e-12)
    # at D = 0 the table is the limit of the Hessian: (5/3) / l_a^2 on the diagonal, 0 elsewhere
    eps = 1e-4
    x = torch.rand(d, generator=g, dtype=torch.float64)
    near = mo.m52grad_dense(x[None], (x + eps)[None], ls)
    at = mo.m52grad_dense(x[None], x[None], ls)
    assert torch.allclose(at[1:, 1:], torch.diag((5.0 / 3.0) / (ls.expand(d) ** 2)), atol=1e-14)
    assert torch.allclose(near, at, atol=1e-2)


def test_oracle_lengthscale_gradient_is_finite_at_coincident_points():
    x1 = torch.rand(4, 2, dtype=torch.float64)
    x2 = x1[[1, 3]].clone()
    ls = torch.tensor([0.5, 0.8], dtype=torch.float64, requires_grad=True)
    mo.m52grad_dense(x1, x2, ls).sum().backward()
    assert torch.isfinite(ls.grad).all()


def test_matern52_kernel_grad_parameters_and_diag():
    from gpytorch_b200 import kernels

    k = kernels.Matern52KernelGrad(nu=0.5)   # nu is dropped: always 5/2, as in the reference
    assert k.nu == 2.5 and k.kind == "matern52" and isinstance(k, kernels.MaternKernel)
    assert k.raw_lengthscale.shape == (1, 1)
    assert type(k.raw_lengthscale_constraint).__name__ == "Positive"
    ka = kernels.Matern52KernelGrad(ard_num_dims=2)
    assert ka.raw_lengthscale.shape == (1, 2)
    assert ka.num_outputs_per_input(torch.zeros(5, 2), torch.zeros(4, 2)) == 3
    sk = kernels.ScaleKernel(ka)
    assert sorted(n for n, _ in sk.named_parameters()) == ["base_kernel.raw_lengthscale", "raw_outputscale"]
    with pytest.raises(RuntimeError, match="x1 == x2"):
        ka(torch.rand(5, 2), torch.rand(5, 2), diag=True)
    with pytest.raises(NotImplementedError, match="batched Matern52KernelGrad"):
        kernels.Matern52KernelGrad(batch_shape=torch.Size([2]))(torch.rand(5, 2))
    for kern in (kernels.Matern52KernelGrad(), kernels.ScaleKernel(kernels.Matern52KernelGrad(ard_num_dims=2))):
        with pytest.raises(NotImplementedError, match="batched Matern52KernelGrad"):
            kern(torch.rand(3, 5, 2))
    # the RBF kernel keeps its own message
    with pytest.raises(NotImplementedError, match="batched RBFKernelGrad"):
        kernels.ScaleKernel(kernels.RBFKernelGrad())(torch.rand(3, 5, 2))


def test_matern52_kernel_grad_refusals():
    from gpytorch_b200 import kernels

    m = kernels.Matern52KernelGrad()
    for bad in (lambda: kernels.ProductKernel(m, kernels.RBFKernel()), lambda: m * kernels.RBFKernel(),
                lambda: kernels.ProductKernel(kernels.ScaleKernel(kernels.Matern52KernelGrad()), kernels.RBFKernel())):
        with pytest.raises(NotImplementedError, match="derivative kernels inside a product"):
            bad()
    for bad in (lambda: kernels.AdditiveKernel(m, kernels.RBFKernel()), lambda: kernels.RBFKernel() + kernels.ScaleKernel(m)):
        with pytest.raises(NotImplementedError, match="Matern52KernelGrad"):
            bad()
    with pytest.raises(NotImplementedError, match="Matern52KernelGrad"):
        kernels.MultitaskKernel(kernels.ScaleKernel(kernels.Matern52KernelGrad()), num_tasks=2)(torch.rand(6, 2))
    with pytest.raises(NotImplementedError, match="Matern52KernelGrad"):
        kernels.GridInterpolationKernel(kernels.Matern52KernelGrad(), 16, num_dims=2)
    with pytest.raises(RuntimeError, match="Matern52KernelGrad.*inputs"):
        m(torch.rand(5, 2).requires_grad_(True))


def test_operator_carries_its_kind_without_device():
    from gpytorch_b200.operators import DerivKernelLinearOperator

    x = torch.rand(10, 3)
    ls, os_ = torch.tensor(0.5), torch.tensor(1.3)
    with pytest.raises(RuntimeError, match="Matern52KernelGrad on the accelerated path supports d <= 16"):
        DerivKernelLinearOperator(torch.rand(4, 17), None, ls, kind="matern52")
    with pytest.raises(ValueError, match="matern52"):
        DerivKernelLinearOperator(x, None, ls, kind="matern32")
    op = DerivKernelLinearOperator(x, torch.rand(6, 3), ls, os_, kind="matern52")
    assert op.kind == "matern52" and op._data_op.kind == "matern52" and op.shape == (40, 24)
    for o in (op.detach(), op._transpose_nonbatch(), op[0:20, 4:24]):
        assert type(o) is DerivKernelLinearOperator and o.kind == "matern52" and o._data_op.kind == "matern52"
    assert op._transpose_nonbatch().shape == (24, 40) and op[0:20, 4:24].shape == (20, 20)
    assert DerivKernelLinearOperator(x, None, ls).kind == "rbf"   # the default keeps the RBF operator
    from gpytorch_b200 import kernels
    sop = kernels.ScaleKernel(kernels.Matern52KernelGrad()).forward(x, x, _same=True)
    assert type(sop) is DerivKernelLinearOperator and sop.kind == "matern52"
    with pytest.raises(NotImplementedError, match="Matern52KernelGrad"):
        op.mul(op)


def test_c_entry_is_declared_and_bound():
    from gpytorch_b200 import _lib

    hdr = open(os.path.join(os.path.dirname(HERE), "include", "gp_bbmm.h")).read()
    assert "int gp_plan_set_deriv_kind(gp_plan* plan, gp_plan* data, int kind);" in hdr
    assert "gp_plan_set_deriv_kind" in _lib.PROTOTYPES and "gp_plan_set_deriv" in _lib.PROTOTYPES


def _res_usage():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(LIB):
        pytest.skip("libgpbbmm.so not built (python -m gpytorch_b200.build)")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4)))
            for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", r.stdout)}


# registers of the fused K.V kernels (CUDA 12.9, -O3, sm_90a), as pinned by tests/test_deriv_host.py: the Matern-5/2 derivative
# operator adds no code to them
_TC_REGS = {k: (126 if k == 0 else 124) for k in range(8)}
# registers of the Matern-5/2 derivative product and gradient kernels, {(job, DP): REG}, as built before they were folded into the
# RBF kernels over a per-kind table (CUDA 12.9, -O3, sm_90a)
_M52_REGS = {("kmv", 4): 168, ("kmv", 8): 126, ("kmv", 12): 168, ("kmv", 16): 236,
             ("grad", 4): 168, ("grad", 8): 224, ("grad", 12): 168, ("grad", 16): 254}


def test_matern52_table_kernels_have_no_local_memory_and_the_rbf_kernels_stay():
    res = _res_usage()
    m52 = {k: v for k, v in res.items() if "DerivTableILi3E" in k or "pc_persistent1_kernelILi69E" in k}
    assert sum("deriv_kmv_kernel" in k for k in m52) == 4 and sum("deriv_grad_kernel" in k for k in m52) == 4, sorted(m52)
    assert len(m52) == 4 + 4 + 2 + 1, sorted(m52)   # + rows, diagonal, pivoted-Cholesky source
    for k, (_, stack, local) in m52.items():
        assert stack == 0 and local == 0, (k, stack, local)
    regs = {(m.group(1), int(m.group(2))): v[0] for k, v in m52.items()
            for m in [re.search(r"deriv_(kmv|grad)_kernelINS_10DerivTableILi3EEELi(\d+)E", k)] if m}
    assert regs == _M52_REGS
    deriv = {k for k in res if ("deriv_" in k and "DerivTableILi3E" not in k) or "pc_persistent1_kernelILi67E" in k}
    assert len(deriv) == 13 and sum("deriv_kmv_kernel" in k for k in deriv) == 4, sorted(deriv)
    tc = {int(re.search(r"kmv_tc_kernelILi(\d+)E", k).group(1)): v[0] for k, v in res.items() if "kmv_tc_kernel" in k}
    assert tc == _TC_REGS
