"""CPU checks of the derivative-observation layer (RBFKernelGrad): the fp64 oracle against the reference's own RBFKernelGrad.forward
(tests/golden/deriv_golden.npz) and against autograd second derivatives of the RBF; the host classes (RBFKernelGrad parameters,
ConstantMeanGrad, confidence_region); the refusals that need no device; and the machine code of deriv.cu (no local memory in any
instantiation serving d <= 16) next to the unchanged register counts of the fused K.V kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import deriv_oracle as do

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "gpytorch_b200", "lib", "libgpbbmm.so")
GOLD = np.load(os.path.join(HERE, "golden", "deriv_golden.npz"))


@pytest.mark.parametrize("d", [1, 2, 5])
@pytest.mark.parametrize("ard", [False, True])
def test_oracle_matches_reference_golden(d, ard):
    tag = f"d{d}_{'ard' if ard else 'iso'}"
    ls = torch.tensor(GOLD[f"{tag}_ls"])
    x1, x2 = torch.tensor(GOLD[f"{tag}_x1"]), torch.tensor(GOLD[f"{tag}_x2"])
    assert torch.allclose(do.deriv_dense(x1, x1, ls), torch.tensor(GOLD[f"{tag}_square"]), rtol=0, atol=1e-12)
    assert torch.allclose(do.deriv_dense(x1, x2, ls), torch.tensor(GOLD[f"{tag}_cross"]), rtol=0, atol=1e-12)   # incl. a coincident pair
    assert torch.allclose(do.deriv_diag(x1.size(0), ls, d), torch.tensor(GOLD[f"{tag}_diag"]), rtol=0, atol=1e-14)
    s = 1.7
    assert torch.allclose(do.deriv_dense(x1, x2, ls, s), s * torch.tensor(GOLD[f"{tag}_cross"]), rtol=0, atol=2e-12)


@pytest.mark.parametrize("ard", [False, True])
def test_oracle_matches_autograd_derivatives(ard):
    """[a, 0] = dk/dx_a, [0, b] = dk/dx'_b, [a, b] = d2k / dx_a dx'_b of k = exp(-|x - x'|^2 / 2 l^2)."""
    g = torch.Generator().manual_seed(5)
    d = 3
    ls = torch.tensor([0.4, 0.7, 1.1], dtype=torch.float64) if ard else torch.tensor(0.6, dtype=torch.float64)
    x1 = torch.rand(4, d, generator=g, dtype=torch.float64)
    x2 = torch.rand(3, d, generator=g, dtype=torch.float64)
    x2[1] = x1[2]
    K = do.deriv_dense(x1, x2, ls)

    def k(a, b):
        return torch.exp(-0.5 * (((a - b) / ls) ** 2).sum())

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


def test_rbf_kernel_grad_parameters_and_diag():
    from gpytorch_b200 import kernels

    k = kernels.RBFKernelGrad()
    assert k.raw_lengthscale.shape == (1, 1)
    assert type(k.raw_lengthscale_constraint).__name__ == "Positive"
    ka = kernels.RBFKernelGrad(ard_num_dims=2)
    assert ka.raw_lengthscale.shape == (1, 2)
    assert ka.num_outputs_per_input(torch.zeros(5, 2), torch.zeros(4, 2)) == 3
    sk = kernels.ScaleKernel(ka)
    assert sorted(n for n, _ in sk.named_parameters()) == ["base_kernel.raw_lengthscale", "raw_outputscale"]
    with pytest.raises(RuntimeError, match="x1 == x2"):
        ka(torch.rand(5, 2), torch.rand(5, 2), diag=True)
    with pytest.raises(NotImplementedError, match="batched"):
        kernels.RBFKernelGrad(batch_shape=torch.Size([2]))(torch.rand(5, 2))
    # batched inputs on an unbatched kernel, alone and inside a ScaleKernel, are refused before any operator is built
    for kern in (kernels.RBFKernelGrad(), kernels.ScaleKernel(kernels.RBFKernelGrad(ard_num_dims=2))):
        with pytest.raises(NotImplementedError, match="batched RBFKernelGrad"):
            kern(torch.rand(3, 5, 2))


def test_constant_mean_grad_output_and_state_dict():
    from gpytorch_b200 import means

    m = means.ConstantMeanGrad()
    assert [n for n, _ in m.named_parameters()] == ["constant"] and m.constant.shape == (1,)
    with torch.no_grad():
        m.constant.fill_(0.7)
    out = m(torch.rand(6, 3))
    assert out.shape == (6, 4)
    assert torch.all(out[:, 0] == 0.7) and torch.all(out[:, 1:] == 0)
    m2 = means.ConstantMeanGrad()
    m2.load_state_dict({"constant": torch.tensor([-1.5])})
    assert float(m2.constant.detach()) == -1.5
    assert set(m.state_dict()) == {"constant"}
    mb = means.ConstantMeanGrad(batch_shape=torch.Size([2]))
    assert mb.constant.shape == (2, 1) and mb(torch.rand(2, 5, 3)).shape == (2, 5, 4)


def test_confidence_region_and_stddev():
    from gpytorch_b200.distributions import MultitaskMultivariateNormal, MultivariateNormal

    cov = torch.diag(torch.tensor([4.0, 1.0, 0.25]))
    mvn = MultivariateNormal(torch.tensor([1.0, 2.0, 3.0]), cov)
    assert torch.allclose(mvn.stddev, torch.tensor([2.0, 1.0, 0.5]))
    lo, hi = mvn.confidence_region()
    assert torch.allclose(lo, torch.tensor([-3.0, 0.0, 2.0])) and torch.allclose(hi, torch.tensor([5.0, 4.0, 4.0]))
    mt = MultitaskMultivariateNormal(torch.zeros(2, 3), torch.diag(torch.arange(1.0, 7.0)))
    lo, hi = mt.confidence_region()
    assert lo.shape == (2, 3) and torch.allclose(hi, 2 * torch.arange(1.0, 7.0).sqrt().reshape(2, 3))


def test_operator_refusals_without_device():
    from gpytorch_b200.operators import ConstantDiagLinearOperator, DerivKernelLinearOperator, KernelLinearOperator

    x = torch.rand(10, 3)
    ls = torch.tensor(0.5)
    with pytest.raises(RuntimeError, match="d <= 16"):
        DerivKernelLinearOperator(torch.rand(4, 17), None, ls)
    with pytest.raises(RuntimeError, match="inputs"):
        DerivKernelLinearOperator(x.clone().requires_grad_(True), None, ls)
    op = DerivKernelLinearOperator(x, None, ls)
    assert op.shape == (40, 40) and op.hyper_tensors()[0] is ls and op.input_tensors() == [] and op.solve_input_tensors() == []
    sub = op[0:20, 4:40]
    assert sub.shape == (20, 36)
    for bad in ((slice(0, 21), slice(None)), (slice(None), slice(2, 40)), (slice(0, 20, 2), slice(None))):
        with pytest.raises(NotImplementedError, match="multiples of d \\+ 1"):
            op[bad]
    with pytest.raises(NotImplementedError, match="DiagLinearOperator"):
        op + KernelLinearOperator(x, None, "rbf", ls)
    with pytest.raises(NotImplementedError):
        op.mul(op)
    assert type(op + ConstantDiagLinearOperator(torch.tensor(0.1), 40)).__name__ == "AddedDiagLinearOperator"
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator
    assert not LowRankUpdatedKernelLinearOperator.supports(op)


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


# registers of the fused K.V kernels as built at the parent of this change (CUDA 12.9, -O3, sm_90a): kmv_tc_kernel<kind> and
# kmv_simt_kernel<kind, DP>; the derivative operator adds no code to them
_TC_REGS = {k: (126 if k == 0 else 124) for k in range(8)}
_SIMT_REGS = {(0, 4): 60, (0, 8): 70, (0, 12): 66, (0, 16): 72, (0, 24): 80, (0, 32): 93, (0, 48): 113, (0, 64): 128, (0, 96): 166,
              (0, 128): 203, (1, 4): 59, (1, 8): 64, (1, 12): 65, (1, 16): 72, (1, 24): 80, (1, 32): 96, (1, 48): 104, (1, 64): 128,
              (1, 96): 164, (1, 128): 208, (2, 4): 59, (2, 8): 64, (2, 12): 70, (2, 16): 72, (2, 24): 78, (2, 32): 90, (2, 48): 104,
              (2, 64): 128, (2, 96): 163, (2, 128): 206, (3, 4): 56, (3, 8): 64, (3, 12): 70, (3, 16): 71, (3, 24): 80, (3, 32): 90,
              (3, 48): 106, (3, 64): 128, (3, 96): 167, (3, 128): 204}


# registers of the RBF derivative product and gradient kernels, {(job, DP): REG}, as built before their Matern-5/2 siblings were
# folded into the same kernels over a per-kind table (CUDA 12.9, -O3, sm_90a)
_DERIV_REGS = {("kmv", 4): 168, ("kmv", 8): 127, ("kmv", 12): 168, ("kmv", 16): 230,
               ("grad", 4): 160, ("grad", 8): 216, ("grad", 12): 204, ("grad", 16): 255}


def test_rbf_table_kernels_have_no_local_memory_and_fused_kernels_keep_their_registers():
    res = _res_usage()
    deriv = {k: v for k, v in res.items() if ("deriv_" in k and "DerivTableILi3E" not in k) or "pc_persistent1_kernelILi67E" in k}
    # the product and gradient kernels for DP = 4, 8, 12, 16 (every d <= 16), rows, diagonal, split sum, pivoted-Cholesky source + init
    assert sum("deriv_kmv_kernel" in k for k in deriv) == 4 and sum("deriv_grad_kernel" in k for k in deriv) == 4, sorted(deriv)
    assert len(deriv) == 4 + 4 + 3 + 2, sorted(deriv)   # + pc_init_deriv_kernel
    for k, (_, stack, local) in deriv.items():
        assert stack == 0 and local == 0, (k, stack, local)
    regs = {(m.group(1), int(m.group(2))): v[0] for k, v in deriv.items()
            for m in [re.search(r"deriv_(kmv|grad)_kernelINS_10DerivTableILi0EEELi(\d+)E", k)] if m}
    assert regs == _DERIV_REGS
    tc = {int(re.search(r"kmv_tc_kernelILi(\d+)E", k).group(1)): v[0] for k, v in res.items() if "kmv_tc_kernel" in k}
    simt = {(int(m.group(1)), int(m.group(2))): v[0] for k, v in res.items()
            for m in [re.search(r"kmv_simt_kernelILi(\d+)ELi(\d+)E", k)] if m}
    assert tc == _TC_REGS
    assert simt == _SIMT_REGS
