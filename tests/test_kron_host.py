"""Kronecker multitask GPs without a GPU: the fp64 oracle of tests/kron_oracle.py against a hand-built matrix and against the Hadamard
oracle on repeated inputs, the new classes' parameters and shapes (MultitaskKernel, MultitaskMean, MultitaskGaussianLikelihood,
MultitaskMultivariateNormal), every refusal, and the resource usage of the kron.cu kernels in the built library."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import hadamard_oracle as ho
import kron_oracle as ko
from oracle import kernels as ok

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _B(T, seed=0):
    g = torch.Generator().manual_seed(seed)
    return ko.index_covar(torch.randn(T, 2, generator=g, dtype=torch.float64), 0.1 + torch.rand(T, generator=g, dtype=torch.float64))


def test_oracle_matches_hand_built_matrix():
    g = torch.Generator().manual_seed(1)
    n, T = 5, 3
    x = torch.rand(n, 2, generator=g, dtype=torch.float64)
    B = _B(T)
    K = ok.kernel_matrix("rbf", x, x, 0.7, 1.3, True)
    A = ko.kron_matrix("rbf", x, x, 0.7, 1.3, B, True)
    for i in range(n):
        for a in range(T):
            for j in range(n):
                for b in range(T):
                    assert A[i * T + a, j * T + b] == K[i, j] * B[a, b]
    tn, sn = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64), 0.05
    D = torch.diagonal(ko.khat("rbf", x, 0.7, 1.3, B, tn, sn) - A)
    assert torch.allclose(D, torch.tensor([0.15, 0.25, 0.35] * n, dtype=torch.float64))


def test_oracle_equals_hadamard_over_repeated_inputs():
    g = torch.Generator().manual_seed(2)
    n, T = 7, 4
    x = torch.rand(n, 3, generator=g, dtype=torch.float64)
    B = _B(T, 3)
    xr = x.repeat_interleave(T, 0)
    t = torch.arange(n * T) % T
    A = ko.kron_matrix("matern52", x, x, 0.5, 0.8, B, True)
    H = ho.hadamard_matrix("matern52", xr, xr, t, t, 0.5, 0.8, B, True)
    assert torch.allclose(A, H, rtol=1e-12, atol=1e-14)
    y = torch.randn(n, T, generator=g, dtype=torch.float64)
    tn = torch.rand(T, generator=g, dtype=torch.float64) * 0.1 + 0.01
    m1 = ko.mll("matern52", x, y, 0.5, 0.8, B, tn, 0.02)
    m2 = ho.mll("matern52", xr, t, y.reshape(-1), 0.5, 0.8, B, tn + 0.02)
    assert abs(float(m1 - m2)) < 1e-10


def test_multitask_kernel_parameters_and_refusals():
    from gpytorch_b200 import kernels

    k = kernels.MultitaskKernel(kernels.ScaleKernel(kernels.RBFKernel()), num_tasks=3, rank=2)
    names = dict(k.named_parameters())
    assert names["task_covar_module.covar_factor"].shape == (3, 2)
    assert names["task_covar_module.raw_var"].shape == (3,)
    assert "data_covar_module.raw_outputscale" in names and "data_covar_module.base_kernel.raw_lengthscale" in names
    assert k.num_outputs_per_input(None, None) == 3
    with pytest.raises(NotImplementedError):
        kernels.MultitaskKernel(kernels.RBFKernel(), num_tasks=2, task_covar_prior=object())
    with pytest.raises(NotImplementedError):
        kernels.MultitaskKernel(kernels.RBFKernel(), num_tasks=2, batch_shape=torch.Size([2]))
    x = torch.rand(4, 2)
    bad = kernels.MultitaskKernel(kernels.AdditiveKernel(kernels.RBFKernel(), kernels.RBFKernel()), num_tasks=2)
    with pytest.raises(NotImplementedError):
        bad(x)


def test_kron_operator_shape_slices_and_refusals():
    from gpytorch_b200.operators import (ConstantDiagLinearOperator, KroneckerKernelLinearOperator,
                                         LowRankUpdatedKernelLinearOperator)

    x = torch.rand(6, 2)
    B = torch.eye(3)
    op = KroneckerKernelLinearOperator(x, None, "rbf", torch.tensor(0.5), torch.tensor(1.0), B)
    assert tuple(op.shape) == (18, 18)
    assert op.hyper_tensors()[2] is B and op.input_tensors() == []
    sub = op[9:, :9]
    assert tuple(sub.shape) == (9, 9) and torch.equal(sub.x1, x[3:]) and torch.equal(sub.x2, x[:3])
    assert tuple(op[9:, 9:].shape) == (9, 9) and op[9:, 9:].same
    with pytest.raises(NotImplementedError):
        op[1:, :]
    with pytest.raises(NotImplementedError):
        op[::2, :]
    assert not LowRankUpdatedKernelLinearOperator.supports(op)
    added = op + ConstantDiagLinearOperator(torch.tensor(0.1), 18)
    assert tuple(added.shape) == (18, 18)
    with pytest.raises(NotImplementedError):
        op + op
    with pytest.raises(RuntimeError):
        KroneckerKernelLinearOperator(x.clone().requires_grad_(), None, "rbf", torch.tensor(0.5), torch.tensor(1.0), B)
    with pytest.raises(RuntimeError):
        KroneckerKernelLinearOperator(x, None, "rbf", torch.tensor(0.5), torch.tensor(1.0), torch.eye(33))


def test_multitask_mean_interleaving():
    from gpytorch_b200 import means

    m = means.MultitaskMean(means.ConstantMean(), num_tasks=3)
    assert [n for n, _ in m.named_parameters()] == [f"base_means.{i}.raw_constant" for i in range(3)]
    with torch.no_grad():
        for i, bm in enumerate(m.base_means):
            bm.constant = float(i + 1)
    out = m(torch.rand(4, 2))
    assert out.shape == (4, 3)
    assert torch.equal(out.reshape(-1), torch.tensor([1.0, 2.0, 3.0] * 4))
    with pytest.raises(RuntimeError):
        means.MultitaskMean([means.ConstantMean(), means.ConstantMean()], num_tasks=3)


def test_likelihood_parameters_noise_diagonal_and_refusals():
    from gpytorch_b200 import likelihoods
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    lk = likelihoods.MultitaskGaussianLikelihood(num_tasks=3)
    params = dict(lk.named_parameters())
    assert params["raw_task_noises"].shape == (3,) and params["raw_noise"].shape == (1,)
    assert torch.all(params["raw_task_noises"] == 0) and torch.all(params["raw_noise"] == 0)
    assert lk.raw_noise_constraint.lower_bound.item() == pytest.approx(1e-4)
    with torch.no_grad():
        lk.task_noises = torch.tensor([0.1, 0.2, 0.3])
        lk.noise = torch.tensor([0.05])
    f = MultitaskMultivariateNormal(torch.zeros(4, 3), torch.eye(12))
    out = lk(f)
    assert isinstance(out, MultitaskMultivariateNormal)
    d = torch.diagonal(out.covariance_matrix) - 1.0
    assert torch.allclose(d, torch.tensor([0.15, 0.25, 0.35] * 4), atol=1e-6)
    with pytest.raises(ValueError):
        likelihoods.MultitaskGaussianLikelihood(num_tasks=2, has_global_noise=False, has_task_noise=False)
    with pytest.raises(NotImplementedError):
        likelihoods.MultitaskGaussianLikelihood(num_tasks=2, rank=1)
    only_task = likelihoods.MultitaskGaussianLikelihood(num_tasks=2, has_global_noise=False)
    assert "raw_noise" not in dict(only_task.named_parameters())


def test_multitask_mvn_shapes_and_refusals():
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    mean = torch.arange(8.0).reshape(4, 2)
    cov = torch.eye(8) * 2.0
    mvn = MultitaskMultivariateNormal(mean, cov)
    assert mvn.event_shape == torch.Size([4, 2]) and mvn.event_shape.numel() == 8
    assert mvn.mean.shape == (4, 2) and mvn.variance.shape == (4, 2) and torch.equal(mvn.loc, mean.reshape(-1))
    y = torch.randn(4, 2)
    ref = torch.distributions.MultivariateNormal(mean.reshape(-1), cov).log_prob(y.reshape(-1))
    assert torch.allclose(mvn.log_prob(y), ref)
    assert mvn.rsample(torch.Size([5])).shape == (5, 4, 2)
    assert mvn.rsample().shape == (4, 2)
    with pytest.raises(NotImplementedError):
        MultitaskMultivariateNormal(mean, cov, interleaved=False)
    with pytest.raises(RuntimeError):
        MultitaskMultivariateNormal(mean, torch.eye(6))


def test_kron_kernels_have_no_local_memory():
    """cuobjdump resource usage of the kron.cu kernels: no stack, no local memory."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
    if not os.path.exists(tool) or not os.path.exists(lib):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = set()
    for i, line in enumerate(lines):
        m = re.search(r"Function _ZN2gp\d+(kron_\w+?_kernel)", line)
        if not m:
            continue
        use = lines[i + 1]
        assert int(re.search(r"STACK:(\d+)", use).group(1)) == 0, line
        assert int(re.search(r"LOCAL:(\d+)", use).group(1)) == 0, line
        seen.add(m.group(1))
    assert seen == {"kron_mix_kernel", "kron_scatter_kernel", "kron_dB_kernel", "kron_point_idx_kernel", "kron_expand_rows_kernel",
                    "kron_expand_diag_kernel"}, seen
