"""CPU checks of the Hadamard multitask pieces: the fp64 oracle of tests/hadamard_oracle.py against a hand-built dense K o B with
per-task noise, its MLL and posterior against direct linear algebra, and the C ABI declarations of the three task calls."""
import math
import os
import re

import torch

import hadamard_oracle as ho
from oracle import kernels as ok

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _problem(seed=0, n=40, d=3, T=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    t = torch.randint(0, T, (n,), generator=g)
    F = torch.randn(T, 2, generator=g, dtype=torch.float64)
    v = 0.1 + torch.rand(T, generator=g, dtype=torch.float64)
    noise = 0.05 + 0.1 * torch.rand(T, generator=g, dtype=torch.float64)
    y = torch.randn(n, generator=g, dtype=torch.float64)
    return x, t, F, v, noise, y


def test_index_covar_is_factor_outer_product_plus_diag():
    _, _, F, v, _, _ = _problem()
    B = ho.index_covar(F, v)
    for a in range(3):
        for b in range(3):
            want = float((F[a] * F[b]).sum()) + (float(v[a]) if a == b else 0.0)
            assert math.isclose(float(B[a, b]), want, rel_tol=1e-14, abs_tol=1e-14)


def test_hadamard_matrix_matches_hand_built_entries():
    x, t, F, v, noise, _ = _problem(1)
    B = ho.index_covar(F, v)
    for kind in ("rbf", "matern12", "matern52"):
        K = ho.hadamard_matrix(kind, x, x, t, t, 0.4, 1.7, B, True)
        base = ok.kernel_matrix(kind, x, x, 0.4, 1.7, True)
        for i in range(0, 40, 7):
            for j in range(0, 40, 5):
                assert math.isclose(float(K[i, j]), float(base[i, j]) * float(B[t[i], t[j]]), rel_tol=1e-13, abs_tol=1e-15)
    A = ho.khat("rbf", x, t, 0.4, 1.7, B, noise)
    K = ho.hadamard_matrix("rbf", x, x, t, t, 0.4, 1.7, B, True)
    assert torch.allclose(torch.diagonal(A - K), noise[t])


def test_mll_and_posterior_match_direct_linear_algebra():
    x, t, F, v, noise, y = _problem(2)
    B = ho.index_covar(F, v)
    A = ho.khat("matern32", x, t, 0.5, 1.2, B, noise)
    n = y.numel()
    want = -0.5 * (float(y @ torch.linalg.solve(A, y)) + float(torch.linalg.slogdet(A)[1]) + n * math.log(2 * math.pi)) / n
    assert math.isclose(float(ho.mll("matern32", x, t, y, 0.5, 1.2, B, noise)), want, rel_tol=1e-10)
    g = torch.Generator().manual_seed(3)
    xs = torch.rand(7, 3, generator=g, dtype=torch.float64)
    ts = torch.randint(0, 3, (7,), generator=g)
    mean, cov = ho.posterior("matern32", x, t, y, xs, ts, 0.5, 1.2, B, noise)
    Ksx = ok.kernel_matrix("matern32", xs, x, 0.5, 1.2, False) * B[ts][:, t]
    Kss = ok.kernel_matrix("matern32", xs, xs, 0.5, 1.2, True) * B[ts][:, ts]
    assert torch.allclose(mean, Ksx @ torch.linalg.solve(A, y), atol=1e-10)
    assert torch.allclose(cov, Kss - Ksx @ torch.linalg.solve(A, Ksx.t()), atol=1e-10)


def test_oracle_gradients_reach_the_index_kernel_parameters():
    x, t, F, v, noise, y = _problem(4)
    F = F.clone().requires_grad_(True)
    v = v.clone().requires_grad_(True)
    noise = noise.clone().requires_grad_(True)
    ho.mll("rbf", x, t, y, 0.3, 1.0, ho.index_covar(F, v), noise).backward()
    for p in (F, v, noise):
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0


def test_c_abi_declares_the_task_calls():
    from gpytorch_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    for name in ("gp_plan_set_tasks", "gp_plan_set_task_covar", "gp_task_covar_grad"):
        assert re.search(r"\bint\s+" + name + r"\s*\(", hdr), name
        assert name in _lib.PROTOTYPES
    assert len(_lib.PROTOTYPES["gp_task_covar_grad"][1]) == 7


# ---- host layer: IndexKernel, HadamardGaussianLikelihood, operators, ExactGP with several inputs (no engine call) ---------------
def test_index_kernel_parameters_formula_and_constraints():
    import pytest
    from gpytorch_b200.kernels import IndexKernel

    torch.manual_seed(0)
    k = IndexKernel(num_tasks=4, rank=2)
    names = dict(k.named_parameters())
    assert set(names) == {"covar_factor", "raw_var"}
    assert tuple(k.covar_factor.shape) == (4, 2) and tuple(k.raw_var.shape) == (4,)
    assert "covar_factor" in k.state_dict() and "raw_var" in k.state_dict()
    assert torch.all(k.var > 0)
    B = k.covar_matrix
    assert torch.allclose(B, k.covar_factor @ k.covar_factor.t() + torch.diag(k.var))
    k.var = torch.tensor([0.5, 1.0, 1.5, 2.0])
    assert torch.allclose(k.var, torch.tensor([0.5, 1.0, 1.5, 2.0]), atol=1e-6)
    i = torch.tensor([[0], [3], [1]])
    op = k(i)
    assert tuple(op.shape) == (3, 3)
    assert torch.allclose(op.to_dense(), k.covar_matrix[i.reshape(-1)][:, i.reshape(-1)])
    with pytest.raises(RuntimeError, match="larger than the number of tasks"):
        IndexKernel(num_tasks=2, rank=3)
    with pytest.raises(NotImplementedError):
        IndexKernel(num_tasks=2, prior=object())


def test_hadamard_likelihood_names_and_diagonal():
    import pytest
    from gpytorch_b200.likelihoods import HadamardGaussianLikelihood

    lik = HadamardGaussianLikelihood(num_tasks=3)
    assert "noise_covar.raw_noise" in lik.state_dict()
    assert tuple(lik.raw_noise.shape) == (3,)
    lik.noise = torch.tensor([0.1, 0.2, 0.3])
    t = torch.tensor([[2], [0], [1], [2]])
    d = lik._shaped_noise_covar(torch.Size([4]), t)
    assert torch.allclose(d.diag_vec, torch.tensor([0.3, 0.1, 0.2, 0.3]), atol=1e-6)
    # the model's inputs as a tuple: the integer tensor is the task index
    d2 = lik._shaped_noise_covar(torch.Size([4]), (torch.rand(4, 2), t))
    assert torch.equal(d.diag_vec, d2.diag_vec)
    with pytest.raises(ValueError, match="Task indices must be provided"):
        lik._shaped_noise_covar(torch.Size([4]))
    # a state dict written by the model loads back
    lik2 = HadamardGaussianLikelihood(num_tasks=3)
    lik2.load_state_dict(lik.state_dict())
    assert torch.allclose(lik2.noise, lik.noise)


def _hadamard_model(x, i, y, T=3):
    from gpytorch_b200 import kernels, likelihoods, means, models

    class MultitaskGPModel(models.ExactGP):
        def __init__(self, train_x, train_i, train_y, likelihood):
            super().__init__((train_x, train_i), train_y, likelihood)
            self.mean_module = means.ConstantMean()
            self.covar_module = kernels.RBFKernel()
            self.task_covar_module = kernels.IndexKernel(num_tasks=T, rank=1)

        def forward(self, x, i):
            from gpytorch_b200.distributions import MultivariateNormal
            covar = self.covar_module(x).mul(self.task_covar_module(i))
            return MultivariateNormal(self.mean_module(x), covar)

    return MultitaskGPModel(x, i, y, likelihoods.HadamardGaussianLikelihood(T))


def test_exact_gp_tuple_inputs_in_train_mode():
    import pytest
    from gpytorch_b200.operators import HadamardKernelLinearOperator, LowRankUpdatedKernelLinearOperator

    x, i, y = torch.rand(20, 2), torch.randint(0, 3, (20, 1)), torch.randn(20)
    m = _hadamard_model(x, i, y)
    assert len(m.train_inputs) == 2
    out = m(x, i)
    op = out.lazy_covariance_matrix
    assert isinstance(op, HadamardKernelLinearOperator)
    assert [t is h for t, h in zip(op.hyper_tensors()[:2], [op.lengthscale, op.outputscale])] == [True, True]
    assert len(op.hyper_tensors()) == 3 and op.hyper_tensors()[2].requires_grad
    assert op.input_tensors() == [] and op.solve_input_tensors() == []
    assert not LowRankUpdatedKernelLinearOperator.supports(op)
    # slicing re-indexes the task ids with the inputs
    sub = op[3:9, 10:20]
    assert torch.equal(sub.t1, i.reshape(-1)[3:9]) and torch.equal(sub.t2, i.reshape(-1)[10:20])
    with pytest.raises(RuntimeError, match="training inputs"):
        m(x, (i + 1) % 3)
    # refusals: inputs that require grad, a second factor, other pairings
    with pytest.raises(RuntimeError, match="inputs of a Hadamard"):
        m.covar_module(x.clone().requires_grad_(True)).mul(m.task_covar_module(i))
    with pytest.raises(NotImplementedError):
        op.mul(m.task_covar_module(i))
    with pytest.raises(NotImplementedError):
        (m.covar_module(x) + m.covar_module(x)).mul(m.task_covar_module(i))
