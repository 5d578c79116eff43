"""CPU checks of the lazy LOVE posterior (settings.fast_pred_samples): the fp64 restatement of why its CIQ noise floor is valid,
the precedence / fallback of the posterior branches, and the resources of the low-rank kernels in the built library."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import kernels as ok, linalg as ol

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpytorch_b200", "lib", "libgpbbmm.so")


@pytest.mark.parametrize("J", [1, 5, 20, 60])
def test_love_posterior_dominates_the_exact_posterior(J):
    """R R^T = Q (Q^T K_hat Q)^-1 Q^T <= K_hat^-1, so K** - K*x R R^T Kx* - (K** - K*x K_hat^-1 Kx*) >= 0: the LOVE covariance
    is at least the exact one, whose spectrum is >= 0, so sigma^2 bounds the observed LOVE posterior's spectrum from below."""
    g = torch.Generator().manual_seed(J)
    n, m = 300, 120
    x = torch.rand(n, 2, generator=g, dtype=torch.float64)
    xs = torch.rand(m, 2, generator=g, dtype=torch.float64)
    K = ok.kernel_matrix("rbf", x, x, 0.3, 1.4, True)
    Khat = K + 0.05 * torch.eye(n, dtype=torch.float64)
    Ksx = ok.kernel_matrix("rbf", xs, x, 0.3, 1.4)
    Kss = ok.kernel_matrix("rbf", xs, xs, 0.3, 1.4, True)
    R = ol.root_inv_decomposition(lambda v: Khat @ v, J, torch.randn(n, generator=g, dtype=torch.float64))
    love = ol.love_predictive_covar(Kss, Ksx, R)
    exact = Kss - Ksx @ torch.linalg.solve(Khat, Ksx.T)
    diff = love - exact
    scale = float(torch.linalg.matrix_norm(Kss, 2))
    assert float(torch.linalg.eigvalsh(0.5 * (diff + diff.T))[0]) >= -1e-10 * scale
    assert float(torch.linalg.eigvalsh(0.5 * (exact + exact.T))[0]) >= -1e-10 * scale


def test_posterior_branch_precedence_and_fallback():
    from gpytorch_b200 import operators, settings
    from gpytorch_b200.models import _posterior_covar_mode
    from gpytorch_b200.operators import (BatchLinearOperator, KernelLinearOperator, LowRankUpdatedKernelLinearOperator,
                                         SKIKernelLinearOperator, SumKernelLinearOperator)

    x = torch.rand(50, 2)
    ls, os_ = torch.tensor(0.5), torch.tensor(1.0)
    plain = KernelLinearOperator(x, x, "rbf", ls, os_)
    summed = SumKernelLinearOperator([plain, KernelLinearOperator(x, x, "matern52", ls, os_)])
    ski = SKIKernelLinearOperator(x, "rbf", ls, os_, (16, 16), (0.0, 0.0), (0.1, 0.1))
    batch = BatchLinearOperator([plain, plain])
    sharded = KernelLinearOperator(x, x, "rbf", ls, os_, row_begin=0, row_count=25)
    cross = KernelLinearOperator(x, torch.rand(30, 2), "rbf", ls, os_)
    assert _posterior_covar_mode(plain) == "exact"
    with settings.fast_pred_var(True):
        assert _posterior_covar_mode(plain) == "love"
    with settings.fast_pred_samples(True):
        for op in (plain, summed):
            assert _posterior_covar_mode(op) == "lazy_love"
        for op in (ski, batch, sharded, cross):               # not eligible: today's dense LOVE path
            assert _posterior_covar_mode(op) == "love"
        with settings.fast_pred_var(True):
            assert _posterior_covar_mode(plain) == "lazy_love"
        with settings.skip_posterior_variances(True):
            assert _posterior_covar_mode(plain) == "skip"
    assert settings.fast_pred_samples.off() and settings.fast_pred_samples in settings.snapshot()
    # the operator refuses what it cannot represent
    with pytest.raises(RuntimeError):
        LowRankUpdatedKernelLinearOperator(ski, torch.zeros(50, 3))
    with pytest.raises(RuntimeError):
        LowRankUpdatedKernelLinearOperator(plain, torch.zeros(50, 129))
    op = LowRankUpdatedKernelLinearOperator(plain, torch.zeros(50, 3))
    assert op.shape == (50, 50) and op.hyper_tensors() == [] and not op.requires_grad
    assert op.base._plan_slot == operators._slot("plain", "lowrank") != plain._plan_slot


def test_lowrank_kernels_are_spill_free():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = {k: 0 for k in ("lowrank_utv_kernel", "lowrank_apply_kernel", "lowrank_kdiag_kernel", "lowrank_krows_kernel")}
    for i, line in enumerate(lines):
        if "Function" not in line:
            continue
        for key in seen:
            if key in line:
                usage = lines[i + 1]
                assert int(re.search(r"STACK:(\d+)", usage).group(1)) == 0, f"{line.strip()}: local memory"
                assert int(re.search(r"REG:(\d+)", usage).group(1)) <= 64, f"{line.strip()}: {usage.strip()}"
                seen[key] += 1
    assert all(v > 0 for v in seen.values()), seen
