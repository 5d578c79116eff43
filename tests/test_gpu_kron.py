"""Kronecker multitask operator (s K) (x) B on the engine (gp_plan_set_kron / gp_plan_set_task_covar / gp_task_covar_grad) against
the fp64 dense oracle of tests/kron_oracle.py: products entry by entry on the tensor-core and SIMT kernels (T t exactly 16, just over
16, T = 32 with t = 16, N off the 128-row tile, cross plans), bit-identity of T = 1, B = [[1]] with the plain plan, agreement with
the Hadamard plan over the repeated inputs, rows, diagonal and the pivoted Cholesky, mBCG solves and the MLL with per-task noise,
the hyper-parameter and task-covariance gradients, Lanczos and CIQ, NaN propagation, the refusals, and the reference's Kronecker
example through ExactGP.

Product tolerance: 1e-5 of the row's absolute product sum (|s K (x) B| |V|)_i, as for the Hadamard operator.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import hadamard_oracle as ho  # noqa: E402
import kron_oracle as ko  # noqa: E402

BACKENDS = ["tcgen05", "simt"]


def _plan(dev, x1, x2=None, backend="auto"):
    from gpytorch_b200.engine import Plan

    return Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)


def _kron(data, T, B, noise=0.0):
    from gpytorch_b200.engine import KronPlan

    p = KronPlan(data, T)
    p.set_noise(noise)
    p.set_task_covar(B.float())
    return p


def _random_B(T, g, rank=2):
    F = torch.randn(T, rank, generator=g, dtype=torch.float64)
    return ko.index_covar(F, 0.1 + torch.rand(T, generator=g, dtype=torch.float64))


# (n1, n2 or None, T, t): T t = 16, T t = 33 (T = 3, t = 11), T = 32 with t = 16, N off the tile, cross plans with N1 != N2
CASES = {"Tt16": (256, None, 4, 4), "T3t11": (300, None, 3, 11), "T32t16": (200, None, 32, 16), "odd_n": (333, None, 2, 7),
         "cross": (210, 333, 3, 5)}


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("kind", ["rbf", "matern32"])
def test_kmv_entrywise(cuda_dev, backend, case, kind):
    g = torch.Generator().manual_seed(7 * len(case) + len(kind))
    n1, n2, T, t = CASES[case]
    d = 5
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64).float().double()
    x2 = None if n2 is None else torch.rand(n2, d, generator=g, dtype=torch.float64).float().double()
    B = _random_B(T, g).float().double()
    ls, os_ = 0.4, 1.3
    data = _plan(cuda_dev, x1.float(), None if x2 is None else x2.float(), backend)
    data.set_hypers(kind, ls, os_, 0.0)
    p = _kron(data, T, B)
    assert p.info()["backend"] == "kron"
    V = torch.randn((n2 or n1) * T, t, generator=g, dtype=torch.float64)
    out = p.kmv(V.float().to(cuda_dev)).double().cpu()
    Kb = ko.kron_matrix(kind, x1, x1 if x2 is None else x2, ls, os_, B, x2 is None)
    ref = Kb @ V
    scale = Kb.abs() @ V.abs()
    err = (out - ref).abs()
    assert torch.all(err <= 1e-5 * scale + 1e-7), (err / scale).max().item()
    assert torch.equal(out, p.kmv(V.float().to(cuda_dev)).double().cpu())   # repeated products: identical bits


@pytest.mark.parametrize("backend", BACKENDS)
def test_single_task_identity_is_bit_identical(cuda_dev, backend):
    g = torch.Generator().manual_seed(5)
    n, d = 517, 6
    x = torch.rand(n, d, generator=g).to(cuda_dev)
    plain = _plan(cuda_dev, x, backend=backend)
    plain.set_hypers("rbf", 0.5, 1.2, 0.1)
    data = _plan(cuda_dev, x, backend=backend)
    data.set_hypers("rbf", 0.5, 1.2, 0.0)
    p = _kron(data, 1, torch.ones(1, 1), noise=0.1)
    for t in (16, 11):
        V = torch.randn(n, t, generator=g).to(cuda_dev)
        assert torch.equal(plain.kmv(V), p.kmv(V))
        assert torch.equal(plain.kmv(V, add_noise=True), p.kmv(V, add_noise=True))


@pytest.mark.parametrize("backend", BACKENDS)
def test_agrees_with_hadamard_over_repeated_inputs(cuda_dev, backend):
    g = torch.Generator().manual_seed(9)
    n, d, T = 150, 3, 4
    x = torch.rand(n, d, generator=g)
    B = _random_B(T, g).float()
    data = _plan(cuda_dev, x, backend=backend).set_hypers("matern52", 0.5, 0.9, 0.0)
    p = _kron(data, T, B)
    h = _plan(cuda_dev, x.repeat_interleave(T, 0), backend=backend).set_hypers("matern52", 0.5, 0.9, 0.0)
    h.set_tasks((torch.arange(n * T) % T).to(cuda_dev), None, T)
    h.set_task_covar(B)
    V = torch.randn(n * T, 9, generator=g).to(cuda_dev)
    a, b = p.kmv(V).double(), h.kmv(V).double()
    assert torch.all((a - b).abs() <= 2e-5 * (b.abs().max() + 1.0))


@pytest.mark.parametrize("backend", BACKENDS)
def test_rows_diag_and_pivoted_cholesky(cuda_dev, backend):
    g = torch.Generator().manual_seed(11)
    n, d, T, rank = 130, 3, 3, 12
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    B = (torch.diag(torch.tensor([0.5, 2.0, 1.0], dtype=torch.float64)) + 0.1).float().double()
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("rbf", 0.3, 1.1, 0.0)
    p = _kron(data, T, B, noise=0.1)
    Kb = ko.kron_matrix("rbf", x, x, 0.3, 1.1, B, True)
    N = n * T
    idx = torch.tensor([0, 5, N - 1, N, -1, 77])
    rows = p.rows(idx.to(cuda_dev)).double().cpu()
    for r, i in enumerate(idx.tolist()):
        if 0 <= i < N:
            assert torch.allclose(rows[r], Kb[i], rtol=1e-5, atol=1e-6)
        else:
            assert torch.isnan(rows[r]).all()
    assert torch.allclose(p.diag().double().cpu(), torch.diagonal(Kb), rtol=1e-6, atol=0)
    lt, piv, _ = p.pivoted_cholesky(rank, 1e-8)
    Lr, piv_ref = ko.pivoted_cholesky(Kb, rank)
    assert int(piv[0]) == int(torch.argmax(torch.diagonal(Kb)))   # first pivot: argmax of s B[a, a]
    assert piv.cpu().tolist() == piv_ref
    assert torch.allclose(lt.double().cpu(), Lr, atol=2e-4)


@pytest.mark.parametrize("backend", BACKENDS)
def test_mbcg_and_mll_with_task_noise(cuda_dev, backend):
    g = torch.Generator().manual_seed(13)
    n, d, T = 800, 3, 3     # N T = 2400 > 2000: the preconditioned MLL pivots the Kronecker operator
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    B = _random_B(T, g).float().double()
    task_noise = torch.tensor([0.05, 0.2, 0.1], dtype=torch.float64)
    y = torch.randn(n * T, generator=g, dtype=torch.float64)
    ls, os_ = 0.35, 1.2
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("rbf", ls, os_, 0.0)
    p = _kron(data, T, B)
    p.set_noise_diag(ko.noise_diag(n, task_noise, 0.0).float().to(cuda_dev))
    A = ko.khat("rbf", x, ls, os_, B, task_noise.float().double(), 0.0)
    rhs = torch.randn(n * T, 3, generator=g, dtype=torch.float64)
    sol, _, info = p.mbcg(rhs.float().to(cuda_dev), tolerance=1e-5, max_iter=2000)
    ref = torch.linalg.solve(A, rhs)
    assert torch.linalg.norm(sol.double().cpu() - ref) <= 1e-3 * torch.linalg.norm(ref), info
    tp = 10
    gg = torch.Generator().manual_seed(3)
    rad = (torch.randint(0, 2, (n * T, tp), generator=gg).float() * 2 - 1).to(cuda_dev)
    iq_ref = float(y @ torch.linalg.solve(A, y))
    ld_ref = float(torch.linalg.slogdet(A)[1])
    res, _ = p.mll(y.float().to(cuda_dev), None, None, rad, num_probes=tp, precond_rank=0, cg_tol=1e-4, max_tridiag_iter=60,
                   max_cg_iter=2000)
    assert abs(res.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0
    eps1 = torch.randn(100, tp, generator=gg).to(cuda_dev)
    eps2 = torch.randn(n * T, tp, generator=gg).to(cuda_dev)
    res2, _ = p.mll(y.float().to(cuda_dev), eps1, eps2, rad, num_probes=tp, precond_rank=100, cg_tol=1e-4, max_tridiag_iter=60,
                    max_cg_iter=2000)
    assert res2.precond_rank > 0
    assert abs(res2.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res2.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("cross", [False, True])
def test_hyper_and_task_covar_gradients(cuda_dev, backend, ard, cross):
    g = torch.Generator().manual_seed(17 + 2 * ard + cross)
    n1, n2, d, T, s = 150, 121, 4, 3, 5
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64).float().double()
    x2 = torch.rand(n2, d, generator=g, dtype=torch.float64).float().double() if cross else x1
    B = _random_B(T, g).float().double()
    L = torch.randn(n1 * T, s, generator=g, dtype=torch.float64).float().double()
    R = torch.randn(x2.size(0) * T, s, generator=g, dtype=torch.float64).float().double()
    ls0 = [0.4, 0.5, 0.6, 0.7] if ard else [0.5]
    os0 = 1.3
    data = _plan(cuda_dev, x1.float(), x2.float() if cross else None, backend)
    data.set_hypers("matern52", ls0 if ard else ls0[0], os0, 0.0)
    p = _kron(data, T, B)
    gl, go = p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    dB = p.task_covar_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    ls = torch.tensor(ls0, dtype=torch.float64, requires_grad=True)
    os_ = torch.tensor(os0, dtype=torch.float64, requires_grad=True)
    Bv = B.clone().requires_grad_(True)
    K = ko.kron_matrix("matern52", x1, x2, ls if ard else ls[0], os_, Bv, not cross)
    (L * (K @ R)).sum().backward()
    scale = float((K.detach().abs() @ R.abs() * L.abs()).sum())
    for a, b in zip(gl, ls.grad.tolist()):
        assert abs(a - b) <= 1e-3 * abs(b) + 2e-6 * scale / min(ls0), (gl, ls.grad)
    assert abs(go - float(os_.grad)) <= 1e-3 * abs(float(os_.grad)) + 2e-6 * scale / os0
    assert torch.all((dB - Bv.grad).abs() <= 1e-3 * Bv.grad.abs() + 2e-6 * scale / float(B.abs().min())), (dB, Bv.grad)
    assert torch.equal(dB, p.task_covar_grad(L.float().to(cuda_dev), R.float().to(cuda_dev)))


@pytest.mark.parametrize("backend", BACKENDS)
def test_ciq_and_lanczos_against_dense(cuda_dev, backend):
    g = torch.Generator().manual_seed(23)
    n, d, T = 150, 3, 3
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    B = _random_B(T, g).float().double()
    task_noise = torch.tensor([0.1, 0.3, 0.2], dtype=torch.float64)
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("rbf", 0.4, 1.0, 0.0)
    p = _kron(data, T, B)
    p.set_noise_diag(ko.noise_diag(n, task_noise, 0.0).float().to(cuda_dev))
    A = ko.khat("rbf", x, 0.4, 1.0, B, task_noise.float().double(), 0.0)
    N = n * T
    b = torch.randn(N, 4, generator=g, dtype=torch.float64)
    tau = [0.05 * 3 ** q for q in range(6)]
    w = [0.2, 0.1, 0.3, 0.15, 0.05, 0.2]
    out, _ = p.ciq_sqrt_matmul(b.float().to(cuda_dev), tau, w, tol=1e-6, max_iter=2000, warn=False)
    ref = A @ sum(wq * torch.linalg.solve(A + tq * torch.eye(N, dtype=torch.float64), b) for tq, wq in zip(tau, w))
    assert torch.linalg.norm(out.double().cpu() - ref) <= 2e-3 * torch.linalg.norm(ref)
    q, tm = p.lanczos(torch.randn(N, generator=g).to(cuda_dev), 20)
    Q = q.double().cpu()
    assert torch.allclose(Q.t() @ A @ Q, tm.double().cpu(), atol=2e-3 * float(torch.linalg.matrix_norm(A, 2)))


def test_nan_propagation(cuda_dev):
    g = torch.Generator().manual_seed(19)
    n, d, T = 200, 3, 2
    x = torch.rand(n, d, generator=g)
    x[17, 1] = float("nan")
    p = _kron(_plan(cuda_dev, x).set_hypers("rbf", 0.5, 1.0, 0.0), T, torch.eye(T), noise=0.1)
    V = torch.randn(n * T, 2, generator=g).to(cuda_dev)
    assert torch.isnan(p.kmv(V)).all()
    assert torch.isnan(p.task_covar_grad(V, V)).all()
    gl, go = p.bilinear_grad(V, V)
    assert math.isnan(go) and all(math.isnan(v) for v in gl)
    # a non-finite B
    q = _kron(_plan(cuda_dev, torch.rand(n, d, generator=g)).set_hypers("rbf", 0.5, 1.0, 0.0), T,
              torch.tensor([[1.0, float("nan")], [0.0, 1.0]]))
    assert torch.isnan(q.kmv(V)).all()
    gl, go = q.bilinear_grad(V, V)
    assert math.isnan(go) and all(math.isnan(v) for v in gl)


def test_refusals(cuda_dev):
    from gpytorch_b200.engine import KronPlan, Plan

    n = 64
    x = torch.rand(n, 2, device=cuda_dev)
    ski = Plan(x)
    ski.set_ski([8, 8], [-0.5, -0.5], [0.3, 0.3])
    ski.set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        KronPlan(ski, 2)
    sp = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    sp.set_sum([Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)])
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        KronPlan(sp, 2)
    tk = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    tk.set_tasks(torch.zeros(n, dtype=torch.int32, device=cuda_dev), None, 1)
    with pytest.raises(RuntimeError, match="task indices"):
        KronPlan(tk, 2)
    lr = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    lr.set_lowrank(torch.randn(n, 2, device=cuda_dev))
    with pytest.raises(RuntimeError, match="low-rank"):
        KronPlan(lr, 2)
    sh = Plan(x, row_begin=0, row_count=32).set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="row-sharded"):
        KronPlan(sh, 2)
    data = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    for T in (0, 33):
        with pytest.raises(RuntimeError, match="not in"):
            KronPlan(data, T)
    p = KronPlan(data, 2)
    p.set_noise(0.1)
    with pytest.raises(RuntimeError, match="task covariance not set"):
        p.kmv(torch.ones(2 * n, 1, device=cuda_dev))
    p.set_task_covar(torch.eye(2))
    g1 = torch.ones(2 * n, 1, device=cuda_dev)
    with pytest.raises(RuntimeError, match="Kronecker"):
        p.kmv_input_grad(g1, g1)
    with pytest.raises(RuntimeError, match="Kronecker"):
        p.dense_input_grad(torch.ones(2 * n, 2 * n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="Kronecker"):
        p.set_lowrank(torch.randn(2 * n, 2, device=cuda_dev))
    with pytest.raises(RuntimeError, match="Kronecker"):
        p.set_tasks(torch.zeros(2 * n, dtype=torch.int32, device=cuda_dev), None, 1)
    with pytest.raises(RuntimeError, match="task covariance"):
        p.set_task_covar(torch.eye(3))


# ---- the model layer: the reference's Kronecker example through ExactGP ----------------------------------------------------------
def _model(dev, n, T, seed, d=1, sigma=0.2):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g) if d > 1 else torch.linspace(0, 1, n).unsqueeze(-1)
    f = [torch.sin(x[:, 0] * (2 * math.pi)), torch.cos(x[:, 0] * (2 * math.pi))] + \
        [torch.sin(x[:, 0] * (a + 2)) for a in range(T - 2)]
    y = torch.stack(f[:T], -1) + sigma * torch.randn(n, T, generator=g)

    class MultitaskGPModel(models.ExactGP):
        def __init__(self, train_x, train_y, likelihood):
            super().__init__(train_x, train_y, likelihood)
            self.mean_module = means.MultitaskMean(means.ConstantMean(), num_tasks=T)
            self.covar_module = kernels.MultitaskKernel(kernels.RBFKernel(), num_tasks=T, rank=1)

        def forward(self, x):
            return MultitaskMultivariateNormal(self.mean_module(x), self.covar_module(x))

    torch.manual_seed(seed)
    lik = likelihoods.MultitaskGaussianLikelihood(num_tasks=T)
    m = MultitaskGPModel(x.to(dev), y.to(dev), lik).to(dev)
    return m, x.double(), y.double()


def _oracle_params(m, T):
    raw = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in m.named_parameters()}
    sp = torch.nn.functional.softplus
    ls = sp(raw["covar_module.data_covar_module.raw_lengthscale"]).reshape(())
    B = ko.index_covar(raw["covar_module.task_covar_module.covar_factor"], sp(raw["covar_module.task_covar_module.raw_var"]))
    tn = 1e-4 + sp(raw["likelihood.raw_task_noises"])
    noise = 1e-4 + sp(raw["likelihood.raw_noise"])
    mean = torch.stack([raw[f"mean_module.base_means.{a}.raw_constant"] for a in range(T)])
    return raw, ls, B, tn, noise, mean


def test_reference_example_trains(cuda_dev):
    """examples/03_Multitask_Exact_GPs/Multitask_GP_Regression.ipynb as written: 100 points, 2 tasks, 50 Adam steps (lr 0.1)."""
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, T = 100, 2
    m, x, y = _model(cuda_dev, n, T, 0, sigma=0.1)   # the notebook's N(0, 0.01) observation noise
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.1)
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    for _ in range(50):
        opt.zero_grad()
        loss = -mll(m(m.train_inputs[0]), m.train_targets)
        loss.backward()
        opt.step()
    m.eval()
    xs = torch.linspace(0, 1, 51).unsqueeze(-1)
    with torch.no_grad():
        pred = m.likelihood(m(xs.to(cuda_dev)))
        mu = pred.mean.cpu()
    truth = torch.stack([torch.sin(xs[:, 0] * 2 * math.pi), torch.cos(xs[:, 0] * 2 * math.pi)], -1)
    assert mu.shape == (51, 2) and pred.variance.shape == (51, 2)
    assert torch.all((mu - truth).abs().mean(0) < 0.05), (mu - truth).abs().mean(0)


def test_model_mll_and_gradients_on_the_cg_branch(cuda_dev):
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, T = 300, 3   # N T = 900 > 800: the CG branch
    m, x, y = _model(cuda_dev, n, T, 31, d=2)
    with torch.no_grad():
        m.covar_module.data_covar_module.lengthscale = 0.3
    m.train()
    raw, ls, B, tn, noise, mean = _oracle_params(m, T)
    with settings.cg_tolerance(1e-6), settings.max_cg_iterations(3000):
        out = m(m.train_inputs[0])
        khat = m.likelihood(out).lazy_covariance_matrix
        loss = khat.inv_quad((m.train_targets - out.mean).reshape(-1, 1))
    A = ko.khat("rbf", x, ls, 1.0, B, tn, noise)
    r = (y - mean).reshape(-1)
    ref = r @ torch.linalg.solve(A, r)
    loss.backward()
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-3 * abs(float(ref))
    for k, v in m.named_parameters():
        if raw[k].grad is None:
            continue
        got, want = v.grad.double().cpu(), raw[k].grad
        assert torch.linalg.norm(got - want) <= 5e-3 * torch.linalg.norm(want) + 1e-5, (k, got, want)
    # the MLL itself (stochastic log det) against the fp64 value
    m.zero_grad()
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    with settings.cg_tolerance(1e-4), settings.num_trace_samples(15), settings.max_lanczos_quadrature_iterations(60):
        val = float(mll(m(m.train_inputs[0]), m.train_targets))
    with torch.no_grad():
        ref_mll = float(ko.mll("rbf", x, y, ls, 1.0, B, tn, noise, mean))
    assert abs(val - ref_mll) <= 0.02 * abs(ref_mll) + 0.02


@pytest.mark.parametrize("fast", [False, True])
def test_model_posterior_against_fp64(cuda_dev, fast):
    from gpytorch_b200 import settings

    n, T = 150, 3
    m, x, y = _model(cuda_dev, n, T, 37, d=2)
    with torch.no_grad():
        m.covar_module.data_covar_module.lengthscale = 0.4
    _, ls, B, tn, noise, mean = _oracle_params(m, T)
    xs = torch.rand(20, 2, generator=torch.Generator().manual_seed(41))
    m.eval()
    with torch.no_grad(), settings.fast_pred_var(fast), settings.max_root_decomposition_size(450):
        post = m(xs.to(cuda_dev))
        mu, var = post.mean.double().cpu(), post.variance.double().cpu()
    with torch.no_grad():
        mu_ref, cov_ref = ko.posterior("rbf", x, y, xs.double(), ls, 1.0, B, tn, noise, mean, mean)
    assert mu.shape == (20, T) and var.shape == (20, T)
    assert torch.allclose(mu, mu_ref, atol=2e-3 * float(y.abs().max()))
    assert torch.allclose(var, torch.diagonal(cov_ref).reshape(-1, T), atol=2e-3 * float(B.diagonal().max()))


def test_model_ciq_rsample(cuda_dev):
    from gpytorch_b200 import settings

    n, T = 1000, 3
    m, _, _ = _model(cuda_dev, n, T, 43, d=2)
    m.train()
    with torch.no_grad(), settings.ciq_samples(True):
        out = m.likelihood(m(m.train_inputs[0]))
        s = out.rsample(torch.Size([3]))
    assert s.shape == (3, n, T) and torch.isfinite(s).all()
