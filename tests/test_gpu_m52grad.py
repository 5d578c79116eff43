"""Matern-5/2 derivative-observation operator (gp_plan_set_deriv_kind, Matern52KernelGrad) on the engine against the fp64 dense
oracle of tests/m52grad_oracle.py: products entry by entry over d in {1, 2, 5, 16}, N in {1, 63, 64, 65, 1000} points, t in
{1, 11, 16, 33} columns, scalar and ARD lengthscales, tensor-core and SIMT data plans, square and cross; the value block against the
plain Matern-5/2 plan, the adjoint identity, bit-identical repeats; rows, diagonal and the pivoted Cholesky; mBCG and the MLL with
per-task noise with and without the preconditioner; lengthscale and outputscale gradients (also across coincident points); Lanczos
and CIQ; NaN, a data plan that changes kind, and, through the public API, the reference's 2-d derivative notebook with
ScaleKernel(Matern52KernelGrad(ard_num_dims=2)) (training, posterior on its 2 500-point grid, exact and fast_pred_var), a CG-branch
model and the reference's known answer.

Product tolerance (DESIGN 4.16): |out - ref| <= tol (M |V|) entrywise, M = m52grad_oracle.m52grad_majorant, with
    tol = 2^-24 (16 (rho_max + 4) + 2 n2 + 4 (d + 1)).
Per entry, relative to M: the packed difference dz carries an absolute error of a few 2^-24 |z| (|z| <= ~5 here), which moves u_a by
that much in units of 1 / l_a (the + 1 / l_a of M) and rho by about as much (absorbed by A' >= |dA / drho| and the 4 of rho_max + 4);
sqrt.approx and ex2.approx add a relative 2^-22 each, and ex2's argument -log2e rho a relative 2^-24 of rho, so e, [0, 0], A and B
are within (8 + 6 rho) 2^-24 of their values: 16 (rho_max + 4) covers both.  The sum over the other side rounds the accumulator twice
per pair (n2 pairs, split partials included) and h over d + 1 terms: 2 n2 + 4 (d + 1).  rho_max = sqrt(5 d) / min l bounds rho on the
unit cube.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import kron_oracle as ko  # noqa: E402
import m52grad_oracle as mo  # noqa: E402
from deriv_oracle import franke  # noqa: E402


def _plan(dev, x1, x2=None, backend="auto"):
    from gpytorch_b200.engine import Plan

    return Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)


def _deriv(data, noise=0.0):
    from gpytorch_b200.engine import DerivPlan

    return DerivPlan(data, "matern52").set_noise(noise)


def _ls0(d, ard, g):
    return (0.3 + 0.5 * torch.rand(d, generator=g, dtype=torch.float64)).float().double().tolist() if ard else [0.45]


def _tol(d, n2, ls):
    rho_max = math.sqrt(5 * d) / min(ls)
    return 2.0 ** -24 * (16 * (rho_max + 4) + 2 * n2 + 4 * (d + 1))


DS = [1, 2, 5, 16]
NS = [1, 63, 64, 65, 1000]
TS = [1, 11, 16, 33]
CASES = [(d, n, TS[(i + j) % 4], (i + j) % 2 == 1, ["tcgen05", "simt"][(i + 2 * j) % 2], (i * 3 + j) % 3 == 2)
         for i, d in enumerate(DS) for j, n in enumerate(NS)]


def _oracle_product(x1, x2, ls, os_, V, chunk=128):
    """(K V, M |V|) in fp64 on the device, 128 row points at a time."""
    ref, bound = [], []
    for i0 in range(0, x1.size(0), chunk):
        xa = x1[i0:i0 + chunk]
        ref.append(mo.m52grad_dense(xa, x2, ls, os_) @ V)
        bound.append(mo.m52grad_majorant(xa, x2, ls, os_) @ V.abs())
    return torch.cat(ref), torch.cat(bound)


@pytest.mark.parametrize("d,n,t,ard,backend,cross", CASES, ids=[f"d{c[0]}-n{c[1]}-t{c[2]}-{'ard' if c[3] else 'iso'}-{c[4]}-"
                                                                   f"{'cross' if c[5] else 'sq'}" for c in CASES])
def test_kmv_entrywise(cuda_dev, d, n, t, ard, backend, cross):
    g = torch.Generator().manual_seed(1000 * d + n + t)
    x1 = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    x2 = torch.rand(n + 7, d, generator=g, dtype=torch.float64).float().double() if cross else None
    ls = _ls0(d, ard, g)
    os_ = 1.3
    data = _plan(cuda_dev, x1.float(), None if x2 is None else x2.float(), backend).set_hypers("matern52", ls if ard else ls[0], os_, 0.0)
    p = _deriv(data)
    assert p.info()["backend"] == "deriv"
    xr = x1 if x2 is None else x2
    V = torch.randn(xr.size(0) * (d + 1), t, generator=g, dtype=torch.float64).float().double()
    out = p.kmv(V.float().to(cuda_dev)).double()
    ref, bound = _oracle_product(x1.to(cuda_dev), xr.to(cuda_dev), torch.tensor(ls, device=cuda_dev), os_, V.to(cuda_dev))
    err = (out - ref).abs()
    tol = _tol(d, xr.size(0), ls)
    assert torch.all(err <= tol * bound), (float((err / bound).max()), tol)
    assert torch.equal(out, p.kmv(V.float().to(cuda_dev)).double())   # repeated products: identical bits


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_value_block_and_adjoint(cuda_dev, backend):
    g = torch.Generator().manual_seed(3)
    n, d = 700, 3
    x = torch.rand(n, d, generator=g).to(cuda_dev)
    plain = _plan(cuda_dev, x, backend=backend).set_hypers("matern52", 0.4, 1.2, 0.0)
    p = _deriv(_plan(cuda_dev, x, backend=backend).set_hypers("matern52", 0.4, 1.2, 0.0))
    v = torch.randn(n, 5, generator=g).to(cuda_dev)
    V = torch.zeros(n * (d + 1), 5, device=cuda_dev)
    V[0::d + 1] = v
    a = p.kmv(V)[0::d + 1].double()
    b = plain.kmv(v).double()
    assert torch.all((a - b).abs() <= 5e-5 * (plain.kmv(v.abs()).double() + 1e-3))
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
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("matern52", ls if ard else ls[0], 1.1, 0.0)
    p = _deriv(data, noise=0.1)
    K = mo.m52grad_dense(x, x, torch.tensor(ls), 1.1)
    N = n * (d + 1)
    idx = torch.tensor([0, 1, 5, N - 1, N, -1, 77])
    rows = p.rows(idx.to(cuda_dev)).double().cpu()
    M = mo.m52grad_majorant(x, x, torch.tensor(ls), 1.1)
    tol = _tol(d, 1, ls)
    for r, i in enumerate(idx.tolist()):
        if 0 <= i < N:
            assert torch.all((rows[r] - K[i]).abs() <= tol * M[i]), i
        else:
            assert torch.isnan(rows[r]).all()
    assert torch.allclose(p.diag().double().cpu(), mo.m52grad_diag(n, torch.tensor(ls), d, 1.1), rtol=1e-6, atol=0)
    assert torch.allclose(p.diag().double().cpu(), torch.diagonal(K), rtol=1e-6, atol=0)
    lt, piv, _ = p.pivoted_cholesky(rank, 1e-8)
    Lr, piv_ref = ko.pivoted_cholesky(K, rank)
    assert int(piv[0]) == int(torch.argmax(torch.diagonal(K)))
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
    data = _plan(cuda_dev, x.float(), backend=backend).set_hypers("matern52", ls, os_, 0.0)
    p = _deriv(data)
    p.set_noise_diag(tn.repeat(n).float().to(cuda_dev))
    A = mo.m52grad_dense(x, x, ls, os_) + torch.diag(tn.float().double().repeat(n))
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
    if cross:
        x2[::10] = x1[:12]   # coincident pairs in a cross plan: rho = 0 there, the 5 B / rho guard
    L = torch.randn(n1 * (d + 1), s, generator=g, dtype=torch.float64).float().double()
    R = torch.randn(x2.size(0) * (d + 1), s, generator=g, dtype=torch.float64).float().double()
    ls0 = [0.4, 0.5, 0.6, 0.7] if ard else [0.5]
    os0 = 1.3
    data = _plan(cuda_dev, x1.float(), x2.float() if cross else None, backend).set_hypers("matern52", ls0 if ard else ls0[0], os0, 0.0)
    p = _deriv(data)
    gl, go = p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    assert all(math.isfinite(v) for v in gl) and math.isfinite(go)
    ls = torch.tensor(ls0, dtype=torch.float64, requires_grad=True)
    os_ = torch.tensor(os0, dtype=torch.float64, requires_grad=True)
    K = mo.m52grad_dense(x1, x2, ls if ard else ls[0], os_)
    (L * (K @ R)).sum().backward()
    scale = float((mo.m52grad_majorant(x1, x2, torch.tensor(ls0), os0) @ R.abs() * L.abs()).sum())
    for a, b in zip(gl, ls.grad.tolist()):
        assert abs(a - b) <= 1e-3 * abs(b) + 1e-5 * scale / min(ls0), (gl, ls.grad)
    assert abs(go - float(os_.grad)) <= 1e-3 * abs(float(os_.grad)) + 1e-5 * scale / os0
    assert (gl, go) == p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))


def test_ciq_and_lanczos_against_dense(cuda_dev):
    g = torch.Generator().manual_seed(23)
    n, d = 120, 2
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    tn = _task_noise(d)
    p = _deriv(_plan(cuda_dev, x.float()).set_hypers("matern52", 0.4, 1.0, 0.0))
    p.set_noise_diag(tn.repeat(n).float().to(cuda_dev))
    A = mo.m52grad_dense(x, x, 0.4, 1.0) + torch.diag(tn.float().double().repeat(n))
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
    p = _deriv(_plan(cuda_dev, x).set_hypers("matern52", 0.5, 1.0, 0.0), noise=0.1)
    V = torch.randn(n * (d + 1), 2, generator=g).to(cuda_dev)
    assert torch.isnan(p.kmv(V)).all()
    assert torch.isnan(p.rows(torch.tensor([0, 5], device=cuda_dev))).all()
    assert torch.isnan(p.diag()).all()
    gl, go = p.bilinear_grad(V, V)
    assert math.isnan(go) and all(math.isnan(v) for v in gl)


def test_kind_refusals_and_a_data_plan_that_changes_kind(cuda_dev):
    from gpytorch_b200.engine import DerivPlan, Plan

    n = 64
    x = torch.rand(n, 2, device=cuda_dev)
    with pytest.raises(RuntimeError, match="Matern-5/2 plan"):
        DerivPlan(Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0), "matern52")
    with pytest.raises(ValueError, match="matern52"):
        DerivPlan(Plan(x).set_hypers("matern32", 0.5, 1.0, 0.0), "matern32")
    with pytest.raises(RuntimeError, match="RBF kernel only"):   # the default stays the RBF operator
        DerivPlan(Plan(x).set_hypers("matern52", 0.5, 1.0, 0.0))
    data = Plan(x).set_hypers("matern52", 0.5, 1.0, 0.0)
    p = DerivPlan(data, "matern52").set_noise(0.1)
    g1 = torch.ones(3 * n, 1, device=cuda_dev)
    p.kmv(g1)
    data.set_hypers("rbf", 0.5, 1.0, 0.0)   # the data plan changed its kind: the next call refuses
    with pytest.raises(RuntimeError, match="Matern-5/2 plan"):
        p.kmv(g1)
    data.set_hypers("matern52", 0.5, 1.0, 0.0)
    p.kmv(g1)
    # the same data plan under an RBF parent, then back: each parent checks its own kind
    data_rbf = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    q = DerivPlan(data_rbf).set_noise(0.1)
    q.attach(data, "matern52")
    assert torch.equal(q.kmv(g1), p.kmv(g1))
    with pytest.raises(RuntimeError, match="RBF kernel only"):
        q.attach(data)
    assert torch.equal(q.kmv(g1), p.kmv(g1))   # a refused attach leaves the operator as it was


def test_operator_cache_keeps_kinds_apart(cuda_dev):
    """One RBF and one Matern-5/2 derivative operator over the same inputs: the plan cache gives each its own parent."""
    from gpytorch_b200.operators import DerivKernelLinearOperator

    g = torch.Generator().manual_seed(29)
    x = torch.rand(50, 2, generator=g).to(cuda_dev)
    ls = torch.tensor(0.4, device=cuda_dev)
    V = torch.randn(150, 3, generator=g).to(cuda_dev)
    ref_m = mo.m52grad_dense(x.double(), x.double(), 0.4) @ V.double()
    ref_r = __import__("deriv_oracle").deriv_dense(x.double(), x.double(), 0.4) @ V.double()
    for _ in range(2):
        om = DerivKernelLinearOperator(x, None, ls, kind="matern52")
        orb = DerivKernelLinearOperator(x, None, ls)
        assert torch.allclose(om.plan().kmv(V).double(), ref_m, atol=1e-4 * float(ref_m.abs().max()))
        assert torch.allclose(orb.plan().kmv(V).double(), ref_r, atol=1e-4 * float(ref_r.abs().max()))


# ---- the model layer: the reference's 2-d derivative notebook with a Matern-5/2 kernel --------------------------------------------
def _notebook_model(dev, train_x, train_y):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    d = train_x.size(-1)

    class GPModelWithDerivatives(models.ExactGP):
        def __init__(self, train_x, train_y, likelihood):
            super().__init__(train_x, train_y, likelihood)
            self.mean_module = means.ConstantMeanGrad()
            self.base_kernel = kernels.Matern52KernelGrad(ard_num_dims=d)
            self.covar_module = kernels.ScaleKernel(self.base_kernel)

        def forward(self, x):
            return MultitaskMultivariateNormal(self.mean_module(x), self.covar_module(x))

    lik = likelihoods.MultitaskGaussianLikelihood(num_tasks=d + 1)
    return GPModelWithDerivatives(train_x.to(dev), train_y.to(dev), lik).to(dev)


def _franke_grid(n_side, noise, seed):
    xv, yv = torch.meshgrid(torch.linspace(0, 1, n_side), torch.linspace(0, 1, n_side), indexing="ij")
    train_x = torch.cat((xv.contiguous().view(xv.numel(), 1), yv.contiguous().view(yv.numel(), 1)), dim=1)
    f, dfx, dfy = franke(train_x[:, 0], train_x[:, 1])
    train_y = torch.stack([f, dfx, dfy], -1).float()
    g = torch.Generator().manual_seed(seed)
    return train_x, train_y + noise * torch.randn(train_y.shape, generator=g)


def _khat(raw, x, n):
    sp = torch.nn.functional.softplus
    ls = sp(raw["base_kernel.raw_lengthscale"]).reshape(-1)
    os_ = sp(raw["covar_module.raw_outputscale"])
    tn = 1e-4 + sp(raw["likelihood.raw_task_noises"])
    noise = 1e-4 + sp(raw["likelihood.raw_noise"])
    return mo.m52grad_dense(x, x, ls, os_) + torch.diag((tn + noise).repeat(n)), ls, os_, tn + noise


def _oracle_loss(raw, x, y):
    """-ExactMarginalLogLikelihood of the notebook model in fp64 (dense Cholesky)."""
    n, T = y.shape
    A = _khat(raw, x, n)[0]
    mean = torch.zeros(n, T, dtype=torch.float64)
    mean[:, 0] = raw["mean_module.constant"]
    r = (y - mean).reshape(-1, 1)
    L = torch.linalg.cholesky(A)
    a = torch.cholesky_solve(r, L)
    N = r.numel()
    return 0.5 * ((r * a).sum() + 2.0 * torch.log(torch.diagonal(L)).sum() + N * math.log(2 * math.pi)) / N


def test_notebook_2d_trains_like_the_fp64_oracle(cuda_dev):
    """The 2-d derivative notebook with a Matern-5/2 kernel: 10 x 10 Franke grid (300 rows, Cholesky branch), 50 Adam steps at lr 0.05."""
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    train_x, train_y = _franke_grid(10, 0.05, 0)
    m = _notebook_model(cuda_dev, train_x, train_y)
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
    """Posterior mean and variance on the notebook's 50 x 50 test grid (7 500 rows), exact and fast_pred_var."""
    from gpytorch_b200 import settings

    train_x, train_y = _franke_grid(10, 0.05, 1)
    m = _notebook_model(cuda_dev, train_x, train_y)
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
    x, y, xs = train_x.double(), train_y.double(), test_x.double()
    n, T = y.shape
    A, ls, os_, noise = _khat(raw, x, n)
    c = float(raw["mean_module.constant"])
    mean = torch.zeros(n, T, dtype=torch.float64)
    mean[:, 0] = c
    Ksx = mo.m52grad_dense(xs, x, ls, os_)
    mu_ref = (Ksx @ torch.linalg.solve(A, (y - mean).reshape(-1))).reshape(-1, T)
    mu_ref[:, 0] += c
    var_ref = (mo.m52grad_diag(xs.size(0), ls, 2, os_) - (Ksx * torch.linalg.solve(A, Ksx.t()).t()).sum(-1)).reshape(-1, T) + noise
    assert mu.shape == (2500, 3) and var.shape == (2500, 3)
    scale = train_y.abs().max(0).values.double()
    assert torch.all((mu - mu_ref).abs() <= 5e-3 * scale), ((mu - mu_ref).abs() / scale).max()
    assert torch.all((var - var_ref).abs() <= 5e-3 * var_ref.max(0).values), ((var - var_ref).abs() / var_ref.max(0).values).max()


def test_model_mll_and_gradients_on_the_cg_branch(cuda_dev):
    """N = 2 000 points, d = 5: 12 000 rows > max_cholesky_size; the CG terms and every parameter's gradient against fp64."""
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, d = 2000, 5
    g = torch.Generator().manual_seed(31)
    train_x = torch.rand(n, d, generator=g)
    w = torch.randn(d, generator=g)
    f = torch.sin(train_x @ w)
    df = torch.cos(train_x @ w)[:, None] * w[None, :]
    train_y = torch.cat([f[:, None], df], -1) + 0.05 * torch.randn(n, d + 1, generator=g)
    m = _notebook_model(cuda_dev, train_x, train_y)
    with torch.no_grad():
        m.base_kernel.lengthscale = torch.full((1, d), 0.8)
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
    A = mo.m52grad_dense(xg, xg, ls, sp(raw["covar_module.raw_outputscale"])) + \
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
    val.backward()
    assert all(torch.isfinite(v.grad).all() for v in m.parameters())


def test_reference_known_answer_through_the_public_api(cuda_dev):
    """test/kernels/test_matern52_kernel_grad.py::test_kernel: default lengthscale, norm of the difference < 1e-5."""
    import os

    import numpy as np

    from gpytorch_b200 import kernels

    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m52grad_golden.npz"))
    a = torch.tensor(gold["ka_a"], dtype=torch.float32, device=cuda_dev)
    b = torch.tensor(gold["ka_b"], dtype=torch.float32, device=cuda_dev)
    actual = torch.tensor(gold["ka_expected"], dtype=torch.float32, device=cuda_dev)
    kernel = kernels.Matern52KernelGrad().to(cuda_dev)
    res = kernel(a, b).to_dense()
    assert res.shape == (6, 6)
    assert float(torch.norm(res - actual)) < 1e-5
    diag = kernel(a, diag=True)
    assert torch.allclose(diag.cpu().double(), mo.m52grad_diag(2, math.log(2.0), 2), rtol=1e-6, atol=0)
