"""Derivative-observation operator (gp_plan_set_deriv, RBFKernelGrad) on the engine against the fp64 dense oracle of
tests/deriv_oracle.py: products entry by entry over d in {1, 2, 5, 16}, N in {1, 63, 64, 65, 1000} points, t in {1, 11, 16, 33}
columns, scalar and ARD lengthscales, tensor-core and SIMT data plans, square and cross; the value block against the plain plan,
the adjoint identity, bit-identical repeats; rows, diagonal and the pivoted Cholesky; mBCG and the MLL with per-task noise with and
without the preconditioner; lengthscale and outputscale gradients; Lanczos and CIQ; NaN and the refusals; and, through the public
API, the reference's 2-d derivative notebook (training, posterior on its 2 500-point grid, confidence_region), a CG-branch model and
CIQ rsample.

Product tolerance (DESIGN 4.14): |out - ref| <= 1e-4 (M |V|) entrywise, M = deriv_oracle.deriv_majorant.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import deriv_oracle as do  # noqa: E402
import kron_oracle as ko  # noqa: E402

TOL = 1e-4


def _plan(dev, x1, x2=None, backend="auto"):
    from gpytorch_b200.engine import Plan

    return Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)


def _deriv(data, noise=0.0):
    from gpytorch_b200.engine import DerivPlan

    return DerivPlan(data).set_noise(noise)


def _ls0(d, ard, g):
    return (0.3 + 0.5 * torch.rand(d, generator=g, dtype=torch.float64)).float().double().tolist() if ard else [0.45]


# every d with every N; t, ARD, backend and square / cross rotate through them so that each value of each appears
DS = [1, 2, 5, 16]
NS = [1, 63, 64, 65, 1000]
TS = [1, 11, 16, 33]
CASES = [(d, n, TS[(i + j) % 4], (i + j) % 2 == 1, ["tcgen05", "simt"][(i + 2 * j) % 2], (i * 3 + j) % 3 == 2)
         for i, d in enumerate(DS) for j, n in enumerate(NS)]


@pytest.mark.parametrize("d,n,t,ard,backend,cross", CASES, ids=[f"d{c[0]}-n{c[1]}-t{c[2]}-{'ard' if c[3] else 'iso'}-{c[4]}-"
                                                                   f"{'cross' if c[5] else 'sq'}" for c in CASES])
def test_kmv_entrywise(cuda_dev, d, n, t, ard, backend, cross):
    g = torch.Generator().manual_seed(1000 * d + n + t)
    x1 = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    x2 = torch.rand(n + 7, d, generator=g, dtype=torch.float64).float().double() if cross else None
    ls = _ls0(d, ard, g)
    os_ = 1.3
    data = _plan(cuda_dev, x1.float(), None if x2 is None else x2.float(), backend).set_hypers("rbf", ls if ard else ls[0], os_, 0.0)
    p = _deriv(data)
    assert p.info()["backend"] == "deriv"
    xr = x1 if x2 is None else x2
    V = torch.randn(xr.size(0) * (d + 1), t, generator=g, dtype=torch.float64).float().double()
    out = p.kmv(V.float().to(cuda_dev)).double()
    ref, bound = _oracle_product(x1.to(cuda_dev), xr.to(cuda_dev), torch.tensor(ls, device=cuda_dev), os_, V.to(cuda_dev))
    err = (out - ref).abs()
    assert torch.all(err <= TOL * bound), float((err / bound).max())
    assert torch.equal(out, p.kmv(V.float().to(cuda_dev)).double())   # repeated products: identical bits


def _oracle_product(x1, x2, ls, os_, V, chunk=128):
    """(K V, M |V|) in fp64 on the device, 128 row points at a time (the d = 16, N = 1000 operator is 17 000 x 17 000)."""
    ref, bound = [], []
    for i0 in range(0, x1.size(0), chunk):
        xa = x1[i0:i0 + chunk]
        ref.append(do.deriv_dense(xa, x2, ls, os_) @ V)
        bound.append(do.deriv_majorant(xa, x2, ls, os_) @ V.abs())
    return torch.cat(ref), torch.cat(bound)


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_value_block_and_adjoint(cuda_dev, backend):
    g = torch.Generator().manual_seed(3)
    n, d = 700, 3
    x = torch.rand(n, d, generator=g).to(cuda_dev)
    plain = _plan(cuda_dev, x, backend=backend).set_hypers("rbf", 0.4, 1.2, 0.0)
    p = _deriv(_plan(cuda_dev, x, backend=backend).set_hypers("rbf", 0.4, 1.2, 0.0))
    v = torch.randn(n, 5, generator=g).to(cuda_dev)
    V = torch.zeros(n * (d + 1), 5, device=cuda_dev)
    V[0::d + 1] = v
    a = p.kmv(V)[0::d + 1].double()
    b = plain.kmv(v).double()
    assert torch.all((a - b).abs() <= 2e-5 * (plain.kmv(v.abs()).double() + 1e-3))
    L = torch.randn(n * (d + 1), 3, generator=g).to(cuda_dev)
    R = torch.randn(n * (d + 1), 3, generator=g).to(cuda_dev)
    lhs = float((L.double() * p.kmv(R).double()).sum())
    rhs = float((p.kmv(L).double() * R.double()).sum())
    assert abs(lhs - rhs) <= 1e-4 * float((L.double().abs() * p.kmv(R.abs()).double().abs()).sum())


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
@pytest.mark.parametrize("ard", [False, True])
def test_rows_diag_and_pivoted_cholesky(cuda_dev, backend, ard):
    g = torch.Generator().manual_seed(11 + ard)
    n, d, rank = 90, 3, 14
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    ls = [0.35, 0.5, 0.7] if ard else [0.45]
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("rbf", ls if ard else ls[0], 1.1, 0.0)
    p = _deriv(data, noise=0.1)
    K = do.deriv_dense(x, x, torch.tensor(ls), 1.1)
    N = n * (d + 1)
    idx = torch.tensor([0, 1, 5, N - 1, N, -1, 77])
    rows = p.rows(idx.to(cuda_dev)).double().cpu()
    M = do.deriv_majorant(x, x, torch.tensor(ls), 1.1)
    for r, i in enumerate(idx.tolist()):
        if 0 <= i < N:
            assert torch.all((rows[r] - K[i]).abs() <= 2e-5 * M[i]), i
        else:
            assert torch.isnan(rows[r]).all()
    assert torch.allclose(p.diag().double().cpu(), do.deriv_diag(n, torch.tensor(ls), d, 1.1), rtol=1e-6, atol=0)
    assert torch.allclose(p.diag().double().cpu(), torch.diagonal(K), rtol=1e-6, atol=0)
    lt, piv, _ = p.pivoted_cholesky(rank, 1e-8)
    Lr, piv_ref = ko.pivoted_cholesky(K, rank)
    assert int(piv[0]) == int(torch.argmax(torch.diagonal(K)))   # first pivot: argmax of the (non-constant) diagonal
    assert piv.cpu().tolist() == piv_ref
    assert torch.allclose(lt.double().cpu(), Lr, atol=2e-4 * math.sqrt(float(torch.diagonal(K).max())))


def _task_noise(d):
    return torch.tensor([0.05] + [0.02 + 0.01 * a for a in range(d)], dtype=torch.float64)


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_mbcg_and_mll_with_task_noise(cuda_dev, backend):
    g = torch.Generator().manual_seed(13)
    n, d = 600, 3    # N (d+1) = 2400 > 2000: the preconditioned MLL pivots the derivative operator
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    ls, os_ = 0.35, 1.2
    tn = _task_noise(d)
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("rbf", ls, os_, 0.0)
    p = _deriv(data)
    p.set_noise_diag(tn.repeat(n).float().to(cuda_dev))
    A = do.deriv_dense(x, x, ls, os_) + torch.diag(tn.float().double().repeat(n))
    N = n * (d + 1)
    rhs = torch.randn(N, 3, generator=g, dtype=torch.float64)
    sol, _, info = p.mbcg(rhs.float().to(cuda_dev), tolerance=1e-5, max_iter=3000)
    ref = torch.linalg.solve(A, rhs)
    assert torch.linalg.norm(sol.double().cpu() - ref) <= 1e-3 * torch.linalg.norm(ref), info
    y = torch.randn(N, generator=g, dtype=torch.float64)
    tp = 10
    gg = torch.Generator().manual_seed(3)
    rad = (torch.randint(0, 2, (N, tp), generator=gg).float() * 2 - 1).to(cuda_dev)
    iq_ref = float(y @ torch.linalg.solve(A, y))
    ld_ref = float(torch.linalg.slogdet(A)[1])
    res, _ = p.mll(y.float().to(cuda_dev), None, None, rad, num_probes=tp, precond_rank=0, cg_tol=1e-4, max_tridiag_iter=80,
                   max_cg_iter=3000)
    assert abs(res.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0
    eps1 = torch.randn(100, tp, generator=gg).to(cuda_dev)
    eps2 = torch.randn(N, tp, generator=gg).to(cuda_dev)
    res2, _ = p.mll(y.float().to(cuda_dev), eps1, eps2, rad, num_probes=tp, precond_rank=100, cg_tol=1e-4, max_tridiag_iter=80,
                    max_cg_iter=3000)
    assert res2.precond_rank > 0
    assert abs(res2.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res2.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("cross", [False, True])
def test_hyper_gradients(cuda_dev, backend, ard, cross):
    g = torch.Generator().manual_seed(17 + 2 * ard + cross)
    n1, n2, d, s = 130, 111, 4, 5
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64).float().double()
    x2 = torch.rand(n2, d, generator=g, dtype=torch.float64).float().double() if cross else x1
    L = torch.randn(n1 * (d + 1), s, generator=g, dtype=torch.float64).float().double()
    R = torch.randn(x2.size(0) * (d + 1), s, generator=g, dtype=torch.float64).float().double()
    ls0 = [0.4, 0.5, 0.6, 0.7] if ard else [0.5]
    os0 = 1.3
    data = _plan(cuda_dev, x1.float(), x2.float() if cross else None, backend).set_hypers("rbf", ls0 if ard else ls0[0], os0, 0.0)
    p = _deriv(data)
    gl, go = p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    ls = torch.tensor(ls0, dtype=torch.float64, requires_grad=True)
    os_ = torch.tensor(os0, dtype=torch.float64, requires_grad=True)
    K = do.deriv_dense(x1, x2, ls if ard else ls[0], os_)
    (L * (K @ R)).sum().backward()
    scale = float((do.deriv_majorant(x1, x2, torch.tensor(ls0), os0) @ R.abs() * L.abs()).sum())
    for a, b in zip(gl, ls.grad.tolist()):
        assert abs(a - b) <= 1e-3 * abs(b) + 1e-5 * scale / min(ls0), (gl, ls.grad)
    assert abs(go - float(os_.grad)) <= 1e-3 * abs(float(os_.grad)) + 1e-5 * scale / os0
    assert (gl, go) == p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))


def test_ciq_and_lanczos_against_dense(cuda_dev):
    g = torch.Generator().manual_seed(23)
    n, d = 120, 2
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    tn = _task_noise(d)
    p = _deriv(_plan(cuda_dev, x.float()).set_hypers("rbf", 0.4, 1.0, 0.0))
    p.set_noise_diag(tn.repeat(n).float().to(cuda_dev))
    A = do.deriv_dense(x, x, 0.4, 1.0) + torch.diag(tn.float().double().repeat(n))
    N = n * (d + 1)
    b = torch.randn(N, 4, generator=g, dtype=torch.float64)
    tau = [0.05 * 3 ** q for q in range(6)]
    w = [0.2, 0.1, 0.3, 0.15, 0.05, 0.2]
    out, _ = p.ciq_sqrt_matmul(b.float().to(cuda_dev), tau, w, tol=1e-6, max_iter=3000, warn=False)
    ref = A @ sum(wq * torch.linalg.solve(A + tq * torch.eye(N, dtype=torch.float64), b) for tq, wq in zip(tau, w))
    assert torch.linalg.norm(out.double().cpu() - ref) <= 2e-3 * torch.linalg.norm(ref)
    q, tm = p.lanczos(torch.randn(N, generator=g).to(cuda_dev), 20)
    Q = q.double().cpu()
    assert torch.allclose(Q.t() @ A @ Q, tm.double().cpu(), atol=2e-3 * float(torch.linalg.matrix_norm(A, 2)))


def test_nan_propagation(cuda_dev):
    g = torch.Generator().manual_seed(19)
    n, d = 200, 3
    x = torch.rand(n, d, generator=g)
    x[17, 1] = float("nan")
    p = _deriv(_plan(cuda_dev, x).set_hypers("rbf", 0.5, 1.0, 0.0), noise=0.1)
    V = torch.randn(n * (d + 1), 2, generator=g).to(cuda_dev)
    assert torch.isnan(p.kmv(V)).all()
    assert torch.isnan(p.rows(torch.tensor([0, 5], device=cuda_dev))).all()
    assert torch.isnan(p.diag()).all()
    gl, go = p.bilinear_grad(V, V)
    assert math.isnan(go) and all(math.isnan(v) for v in gl)


def test_refusals(cuda_dev):
    from gpytorch_b200.engine import DerivPlan, KronPlan, Plan

    n = 64
    x = torch.rand(n, 2, device=cuda_dev)
    with pytest.raises(RuntimeError, match="RBF kernel only"):
        DerivPlan(Plan(x).set_hypers("matern52", 0.5, 1.0, 0.0))
    ski = Plan(x)
    ski.set_ski([8, 8], [-0.5, -0.5], [0.3, 0.3])
    ski.set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        DerivPlan(ski)
    sp = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    sp.set_sum([Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)])
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        DerivPlan(sp)
    tk = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    tk.set_tasks(torch.zeros(n, dtype=torch.int32, device=cuda_dev), None, 1)
    with pytest.raises(RuntimeError, match="task indices"):
        DerivPlan(tk)
    kr = KronPlan(Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0), 2).set_noise(0.1)
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        DerivPlan(kr)
    lr = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    lr.set_lowrank(torch.randn(n, 2, device=cuda_dev))
    with pytest.raises(RuntimeError, match="low-rank"):
        DerivPlan(lr)
    sh = Plan(x, row_begin=0, row_count=32).set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="row-sharded"):
        DerivPlan(sh)
    with pytest.raises(RuntimeError, match="d <= 16"):
        DerivPlan(Plan(torch.rand(n, 17, device=cuda_dev)).set_hypers("rbf", 0.5, 1.0, 0.0))
    data = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    p = DerivPlan(data).set_noise(0.1)
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        DerivPlan(p)
    with pytest.raises(RuntimeError, match="Kronecker|derivative"):
        KronPlan(p, 2)
    g1 = torch.ones(3 * n, 1, device=cuda_dev)
    with pytest.raises(RuntimeError, match="derivative"):
        p.kmv_input_grad(g1, g1)
    with pytest.raises(RuntimeError, match="derivative"):
        p.dense_input_grad(torch.ones(3 * n, 3 * n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="derivative"):
        p.set_lowrank(torch.randn(3 * n, 2, device=cuda_dev))
    with pytest.raises(RuntimeError, match="derivative"):
        p.set_tasks(torch.zeros(3 * n, dtype=torch.int32, device=cuda_dev), None, 1)
    with pytest.raises(RuntimeError, match="no task covariance"):
        p.set_task_covar(torch.eye(3))
    with pytest.raises(RuntimeError, match="no task covariance"):
        p.task_covar_grad(g1, g1)
    data.set_hypers("matern32", 0.5, 1.0, 0.0)     # the data plan changed its kind: the next call refuses
    with pytest.raises(RuntimeError, match="RBF kernel only"):
        p.kmv(g1)
    # new data with the same N (d + 1) but other N and d (64 points at d = 2 -> 96 points at d = 1): refused, not re-split silently
    data.set_hypers("rbf", 0.5, 1.0, 0.0)
    p.kmv(g1)
    data.x1 = data.x2 = torch.rand(96, 1, device=cuda_dev)
    data.n1, data.n2, data.d, data.row_count = 96, 96, 1, 96
    data.refresh_data()
    with pytest.raises(RuntimeError, match="changed its size"):
        p.kmv(g1)


# ---- the model layer: the reference's derivative notebooks through ExactGP ----------------------------------------------------------
def _notebook_model(dev, train_x, train_y, ard):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    d = train_x.size(-1)

    class GPModelWithDerivatives(models.ExactGP):
        def __init__(self, train_x, train_y, likelihood):
            super().__init__(train_x, train_y, likelihood)
            self.mean_module = means.ConstantMeanGrad()
            self.base_kernel = kernels.RBFKernelGrad(ard_num_dims=d if ard else None)
            self.covar_module = kernels.ScaleKernel(self.base_kernel)

        def forward(self, x):
            return MultitaskMultivariateNormal(self.mean_module(x), self.covar_module(x))

    lik = likelihoods.MultitaskGaussianLikelihood(num_tasks=d + 1)
    return GPModelWithDerivatives(train_x.to(dev), train_y.to(dev), lik).to(dev)


def _franke_grid(n_side, noise, seed):
    xv, yv = torch.meshgrid(torch.linspace(0, 1, n_side), torch.linspace(0, 1, n_side), indexing="ij")
    train_x = torch.cat((xv.contiguous().view(xv.numel(), 1), yv.contiguous().view(yv.numel(), 1)), dim=1)
    f, dfx, dfy = do.franke(train_x[:, 0], train_x[:, 1])
    train_y = torch.stack([f, dfx, dfy], -1).float()
    g = torch.Generator().manual_seed(seed)
    return train_x, train_y + noise * torch.randn(train_y.shape, generator=g)


def _oracle_loss(raw, x, y):
    """-ExactMarginalLogLikelihood of the notebook model in fp64 (dense Cholesky)."""
    sp = torch.nn.functional.softplus
    ls = sp(raw["base_kernel.raw_lengthscale"]).reshape(-1)
    os_ = sp(raw["covar_module.raw_outputscale"])
    tn = 1e-4 + sp(raw["likelihood.raw_task_noises"])
    noise = 1e-4 + sp(raw["likelihood.raw_noise"])
    n, T = y.shape
    A = do.deriv_dense(x, x, ls, os_) + torch.diag((tn + noise).repeat(n))
    mean = torch.zeros(n, T, dtype=torch.float64)
    mean[:, 0] = raw["mean_module.constant"]
    r = (y - mean).reshape(-1, 1)
    L = torch.linalg.cholesky(A)
    a = torch.cholesky_solve(r, L)
    N = r.numel()
    return 0.5 * ((r * a).sum() + 2.0 * torch.log(torch.diagonal(L)).sum() + N * math.log(2 * math.pi)) / N


def _oracle_posterior(raw, x, y, xs):
    sp = torch.nn.functional.softplus
    ls = sp(raw["base_kernel.raw_lengthscale"]).reshape(-1)
    os_ = sp(raw["covar_module.raw_outputscale"])
    tn = 1e-4 + sp(raw["likelihood.raw_task_noises"])
    noise = 1e-4 + sp(raw["likelihood.raw_noise"])
    n, T = y.shape
    A = do.deriv_dense(x, x, ls, os_) + torch.diag((tn + noise).repeat(n))
    c = float(raw["mean_module.constant"])
    mean = torch.zeros(n, T, dtype=torch.float64)
    mean[:, 0] = c
    Ksx = do.deriv_dense(xs, x, ls, os_)
    mu = Ksx @ torch.linalg.solve(A, (y - mean).reshape(-1))
    mu = mu.reshape(-1, T)
    mu[:, 0] += c
    var = do.deriv_diag(xs.size(0), ls, x.size(1), os_) - (Ksx * torch.linalg.solve(A, Ksx.t()).t()).sum(-1)
    return mu, var.reshape(-1, T)


def test_notebook_2d_trains_like_the_fp64_oracle(cuda_dev):
    """Simple_GP_Regression_Derivative_Information_2d: 10 x 10 Franke grid (300 rows, Cholesky branch), 50 Adam steps at lr 0.05."""
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    train_x, train_y = _franke_grid(10, 0.05, 0)
    m = _notebook_model(cuda_dev, train_x, train_y, ard=True)
    raw = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in m.named_parameters()}
    x, y = train_x.double(), train_y.double()
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.05)
    opt_ref = torch.optim.Adam(list(raw.values()), lr=0.05)
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    worst = 0.0
    for _ in range(50):
        opt.zero_grad()
        loss = -mll(m(m.train_inputs[0]), m.train_targets)
        loss.backward()
        opt.step()
        opt_ref.zero_grad()
        ref = _oracle_loss(raw, x, y)
        ref.backward()
        opt_ref.step()
        worst = max(worst, abs(float(loss.detach()) - float(ref.detach())) / (abs(float(ref.detach())) + 0.1))
    assert worst <= 2e-3, worst
    for k, v in m.named_parameters():
        assert torch.allclose(v.detach().double().cpu(), raw[k].detach(), rtol=1e-2, atol=1e-2), (k, v, raw[k])


@pytest.mark.parametrize("fast", [False, True])
def test_notebook_2d_posterior_against_fp64(cuda_dev, fast):
    """Posterior mean and variance on the notebook's 50 x 50 test grid (7 500 rows), exact and fast_pred_var, and confidence_region."""
    from gpytorch_b200 import settings

    train_x, train_y = _franke_grid(10, 0.05, 1)
    m = _notebook_model(cuda_dev, train_x, train_y, ard=True)
    with torch.no_grad():
        m.base_kernel.lengthscale = torch.tensor([[0.25, 0.3]])
        m.covar_module.outputscale = 0.5
        m.likelihood.noise = 1e-3
    raw = {k: v.detach().double().cpu() for k, v in m.named_parameters()}
    xv, yv = torch.meshgrid(torch.linspace(0, 1, 50), torch.linspace(0, 1, 50), indexing="ij")
    test_x = torch.stack([xv.reshape(-1), yv.reshape(-1)], -1)
    m.eval()
    with torch.no_grad(), settings.fast_pred_var(fast), settings.max_root_decomposition_size(300):
        post = m.likelihood(m(test_x.to(cuda_dev)))
        mu, var = post.mean.double().cpu(), post.variance.double().cpu()
        lo, hi = post.confidence_region()
    mu_ref, var_ref = _oracle_posterior(raw, train_x.double(), train_y.double(), test_x.double())
    tn = 1e-4 + torch.nn.functional.softplus(raw["likelihood.raw_task_noises"])
    var_ref = var_ref + tn + 1e-4 + torch.nn.functional.softplus(raw["likelihood.raw_noise"])
    assert mu.shape == (2500, 3) and var.shape == (2500, 3) and lo.shape == (2500, 3)
    scale = train_y.abs().max(0).values.double()
    assert torch.all((mu - mu_ref).abs() <= 5e-3 * scale), ((mu - mu_ref).abs() / scale).max()
    assert torch.all((var - var_ref).abs() <= 5e-3 * var_ref.max(0).values), ((var - var_ref).abs() / var_ref.max(0).values).max()
    assert torch.allclose(lo.double().cpu(), mu - 2 * var.sqrt(), atol=1e-5 * float(scale.max()))
    assert torch.allclose(hi.double().cpu(), mu + 2 * var.sqrt(), atol=1e-5 * float(scale.max()))


def test_notebook_1d_runs(cuda_dev):
    """Simple_GP_Regression_Derivative_Information_1d: sin / cos data, scalar lengthscale, training, prediction, confidence_region."""
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    lb, ub, n = 0.0, 5 * math.pi, 50
    train_x = torch.linspace(lb, ub, n).unsqueeze(-1)
    g = torch.Generator().manual_seed(0)
    train_y = torch.stack([torch.sin(2 * train_x) + torch.cos(train_x), -torch.sin(train_x) + 2 * torch.cos(2 * train_x)], -1).squeeze(1)
    train_y = train_y + 0.05 * torch.randn(n, 2, generator=g)
    m = _notebook_model(cuda_dev, train_x, train_y, ard=False)
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.05)
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    for _ in range(100):
        opt.zero_grad()
        loss = -mll(m(m.train_inputs[0]), m.train_targets)
        loss.backward()
        opt.step()
    m.eval()
    xs = torch.linspace(lb, ub, 500).unsqueeze(-1)
    with torch.no_grad():
        pred = m.likelihood(m(xs.to(cuda_dev)))
        lo, hi = pred.confidence_region()
    truth = torch.stack([torch.sin(2 * xs) + torch.cos(xs), -torch.sin(xs) + 2 * torch.cos(2 * xs)], -1).squeeze(1)
    assert pred.mean.shape == (500, 2) and lo.shape == (500, 2)
    assert float((pred.mean.cpu() - truth).abs().mean()) < 0.1
    assert torch.all(lo <= hi)


def test_model_mll_and_gradients_on_the_cg_branch(cuda_dev):
    """N = 2 000 points, d = 5: 12 000 rows, preconditioned by default; the CG terms and every parameter's gradient against fp64."""
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, d = 2000, 5
    g = torch.Generator().manual_seed(31)
    train_x = torch.rand(n, d, generator=g)
    w = torch.randn(d, generator=g)
    f = torch.sin(train_x @ w)
    df = torch.cos(train_x @ w)[:, None] * w[None, :]
    train_y = torch.cat([f[:, None], df], -1) + 0.05 * torch.randn(n, d + 1, generator=g)
    m = _notebook_model(cuda_dev, train_x, train_y, ard=True)
    with torch.no_grad():
        m.base_kernel.lengthscale = torch.full((1, d), 0.6)
        m.mean_module.constant.fill_(0.1)
    m.train()
    raw = {k: v.detach().double().to(cuda_dev).clone().requires_grad_(True) for k, v in m.named_parameters()}
    xg, yg = train_x.double().to(cuda_dev), train_y.double().to(cuda_dev)
    with settings.cg_tolerance(1e-6), settings.max_cg_iterations(4000):
        out = m(m.train_inputs[0])
        khat = m.likelihood(out).lazy_covariance_matrix
        loss = khat.inv_quad((m.train_targets - out.mean).reshape(-1, 1))
    sp = torch.nn.functional.softplus
    ls = sp(raw["base_kernel.raw_lengthscale"]).reshape(-1)
    A = do.deriv_dense(xg, xg, ls, sp(raw["covar_module.raw_outputscale"])) + \
        torch.diag((1e-4 + sp(raw["likelihood.raw_task_noises"]) + 1e-4 + sp(raw["likelihood.raw_noise"])).repeat(n))
    mean = torch.zeros(n, d + 1, dtype=torch.float64, device=cuda_dev)
    mean[:, 0] = raw["mean_module.constant"]
    r = (yg - mean).reshape(-1)
    ref = r @ torch.linalg.solve(A, r)
    loss.backward()
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-3 * abs(float(ref.detach()))
    for k, v in m.named_parameters():
        got, want = v.grad.double().cpu(), raw[k].grad.cpu()
        assert torch.linalg.norm(got - want) <= 5e-3 * torch.linalg.norm(want) + 1e-5, (k, got, want)
    del A
    m.zero_grad()
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    val = mll(m(m.train_inputs[0]), m.train_targets)   # the default path: N (d+1) >= 2000 rows, preconditioned
    assert torch.isfinite(val)


def test_model_ciq_rsample(cuda_dev):
    from gpytorch_b200 import settings

    train_x, train_y = _franke_grid(20, 0.05, 2)
    m = _notebook_model(cuda_dev, train_x, train_y, ard=True)
    with torch.no_grad():
        m.base_kernel.lengthscale = torch.tensor([[0.3, 0.3]])
    m.train()
    torch.manual_seed(0)
    with torch.no_grad(), settings.ciq_samples(True):
        out = m.likelihood(m(m.train_inputs[0]))
        s = out.rsample(torch.Size([400]))
    assert s.shape == (400, 400, 3) and torch.isfinite(s).all()
    # moments: the sample covariance of the draws against the operator (value row 0 and derivative row 1 of point 0)
    cov = out.lazy_covariance_matrix
    flat = (s - out.mean.unsqueeze(0)).reshape(400, -1).double()
    emp = (flat[:, :3].t() @ flat[:, :3]) / 400
    dense = cov.to_dense()[:3, :3].double().cpu() if not torch.is_tensor(cov) else cov[:3, :3].double().cpu()
    assert torch.allclose(emp.cpu(), dense, atol=0.25 * float(dense.diagonal().max()))
