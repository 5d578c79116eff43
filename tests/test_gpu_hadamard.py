"""Hadamard multitask operator s K o B[t, t'] on the engine (gp_plan_set_tasks / gp_plan_set_task_covar / gp_task_covar_grad) against
the fp64 dense oracle of tests/hadamard_oracle.py: products entry by entry on the tensor-core and SIMT kernels (task boundaries
inside and on a 128-row tile, interleaved tasks, T = 1 and T = 32, cross plans with different task sets), bit-identity of T = 1,
B = [[1]] with the plain plan, rows and diagonal, the pivoted Cholesky of the non-constant diagonal, mBCG solves and the MLL with
per-task noise, the hyper-parameter and task-covariance gradients, CIQ sampling, determinism, NaN propagation and the refusals.

Product tolerance: 1e-5 of the row's absolute product sum (|s K o B| |V|)_i.  The 3xTF32 tensor-core kernel and the fp32 SIMT
kernel keep every entry to a few 1e-7 relative (ex2.approx: 2 ulp), and the sums to fp32 rounding over n terms.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import hadamard_oracle as ho  # noqa: E402
from oracle import kernels as ok  # noqa: E402

BACKENDS = ["tcgen05", "simt"]


def _plan(dev, x1, x2=None, backend="auto"):
    from gpytorch_b200.engine import Plan

    return Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)


def _random_B(T, g, rank=2):
    F = torch.randn(T, rank, generator=g, dtype=torch.float64)
    return ho.index_covar(F, 0.1 + torch.rand(T, generator=g, dtype=torch.float64))


def _tasks_case(case, g):
    """(n1, n2 or None, T, t1, t2 or None)"""
    if case == "boundary_in_tile":   # counts 100, 150, 50: row task boundaries inside 128-row tiles
        t = torch.cat([torch.full((100,), 0), torch.full((150,), 1), torch.full((50,), 2)])
        return 300, None, 3, t[torch.randperm(300, generator=g)], None
    if case == "boundary_on_tile":   # counts 128, 128, 64: boundaries exactly on tile edges
        t = torch.cat([torch.full((128,), 0), torch.full((128,), 1), torch.full((64,), 2)])
        return 320, None, 3, t, None
    if case == "interleaved":
        return 290, None, 4, torch.arange(290) % 4, None
    if case == "T1":
        return 333, None, 1, torch.zeros(333, dtype=torch.long), None
    if case == "T32":
        return 700, None, 32, torch.randint(0, 32, (700,), generator=g), None
    if case == "cross":              # rows of tasks {0, 1, 2}, columns of tasks {1, 2, 3}
        return 210, 333, 4, torch.randint(0, 3, (210,), generator=g), 1 + torch.randint(0, 3, (333,), generator=g)
    raise ValueError(case)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("case", ["boundary_in_tile", "boundary_on_tile", "interleaved", "T1", "T32", "cross"])
@pytest.mark.parametrize("kind", ["rbf", "matern32"])
def test_kmv_entrywise(cuda_dev, backend, case, kind):
    g = torch.Generator().manual_seed(100 * len(case) + len(kind))
    n1, n2, T, t1, t2 = _tasks_case(case, g)
    d = 5
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64)
    x2 = None if n2 is None else torch.rand(n2, d, generator=g, dtype=torch.float64)
    B = _random_B(T, g)
    ls, os_ = 0.4, 1.3
    p = _plan(cuda_dev, x1.float(), None if x2 is None else x2.float(), backend)
    p.set_hypers(kind, ls, os_, 0.0)
    p.set_tasks(t1.to(cuda_dev), None if t2 is None else t2.to(cuda_dev), T)
    p.set_task_covar(B.float())
    assert p.info()["backend"] == backend
    V = torch.randn(n2 or n1, 19, generator=g, dtype=torch.float64)
    out = p.kmv(V.float().to(cuda_dev)).double().cpu()
    xr = x1 if x2 is None else x2
    Kb = ho.hadamard_matrix(kind, x1.float().double(), xr.float().double(), t1, t1 if t2 is None else t2, ls, os_, B.float().double(),
                            x2 is None)
    ref = Kb @ V
    scale = Kb.abs() @ V.abs()
    err = (out - ref).abs()
    assert torch.all(err <= 1e-5 * scale + 1e-7), (err / scale).max().item()
    # repeated products are bit-identical
    out2 = p.kmv(V.float().to(cuda_dev)).double().cpu()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("backend", BACKENDS)
def test_single_task_identity_is_bit_identical(cuda_dev, backend):
    g = torch.Generator().manual_seed(5)
    n, d = 517, 6
    x = torch.rand(n, d, generator=g).to(cuda_dev)
    V = torch.randn(n, 16, generator=g).to(cuda_dev)
    plain = _plan(cuda_dev, x, backend=backend)
    plain.set_hypers("rbf", 0.5, 1.2, 0.1)
    mt = _plan(cuda_dev, x, backend=backend)
    mt.set_hypers("rbf", 0.5, 1.2, 0.1)
    mt.set_tasks(torch.zeros(n, dtype=torch.int32, device=cuda_dev), None, 1)
    mt.set_task_covar(torch.ones(1, 1))
    assert torch.equal(plain.kmv(V), mt.kmv(V))
    assert torch.equal(plain.kmv(V, add_noise=True), mt.kmv(V, add_noise=True))


@pytest.mark.parametrize("backend", BACKENDS)
def test_rows_and_diag(cuda_dev, backend):
    g = torch.Generator().manual_seed(7)
    n, d, T = 260, 4, 3
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    t = torch.randint(0, T, (n,), generator=g)
    B = _random_B(T, g)
    p = _plan(cuda_dev, x.float(), backend=backend)
    p.set_hypers("matern52", 0.6, 0.9, 0.0)
    p.set_tasks(t.to(cuda_dev), None, T)
    p.set_task_covar(B.float())
    Kb = ho.hadamard_matrix("matern52", x.float().double(), x.float().double(), t, t, 0.6, 0.9, B.float().double(), True)
    idx = torch.tensor([0, 5, n - 1, n, -1, 77])
    rows = p.rows(idx.to(cuda_dev)).double().cpu()
    for r, i in enumerate(idx.tolist()):
        if 0 <= i < n:
            assert torch.allclose(rows[r], Kb[i], rtol=1e-5, atol=1e-6)
        else:
            assert torch.isnan(rows[r]).all()
    dg = p.diag().double().cpu()
    assert torch.allclose(dg, torch.diagonal(Kb), rtol=1e-6, atol=0)
    assert dg.unique().numel() > 1   # s B[t_i, t_i] is not constant
    # cross plan diagonal: s k(x1_i, x2_i) B[t1_i, t2_i]
    x2 = torch.rand(n, d, generator=g, dtype=torch.float64)
    t2 = torch.randint(0, T, (n,), generator=g)
    pc = _plan(cuda_dev, x.float(), x2.float(), backend=backend)
    pc.set_hypers("rbf", 0.6, 0.9, 0.0)
    pc.set_tasks(t.to(cuda_dev), t2.to(cuda_dev), T)
    pc.set_task_covar(B.float())
    Kc = ho.hadamard_matrix("rbf", x.float().double(), x2.float().double(), t, t2, 0.6, 0.9, B.float().double(), False)
    assert torch.allclose(pc.diag().double().cpu(), torch.diagonal(Kc), rtol=1e-5, atol=1e-7)


def test_task_ids_out_of_range(cuda_dev):
    from gpytorch_b200.engine import Plan

    x = torch.rand(50, 3, device=cuda_dev)
    p = Plan(x)
    p.set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="shape"):
        p.set_tasks(torch.full((50,), 3, device=cuda_dev), None, 3)
    with pytest.raises(RuntimeError, match="shape"):
        p.set_tasks(torch.full((50,), -1, device=cuda_dev), None, 3)
    with pytest.raises(RuntimeError, match="shape"):
        p.set_tasks(torch.zeros(50, device=cuda_dev), None, 33)


@pytest.mark.parametrize("backend", BACKENDS)
def test_pivoted_cholesky_nonconstant_diagonal(cuda_dev, backend):
    from oracle import linalg as ol

    g = torch.Generator().manual_seed(11)
    n, d, T, rank = 400, 3, 4, 12
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    t = torch.randint(0, T, (n,), generator=g)
    B = torch.diag(torch.tensor([0.5, 2.0, 1.0, 1.5], dtype=torch.float64)) + 0.1
    p = _plan(cuda_dev, x.float(), backend=backend)
    p.set_hypers("rbf", 0.3, 1.1, 0.1)
    p.set_tasks(t.to(cuda_dev), None, T)
    p.set_task_covar(B.float())
    lt, piv, _ = p.pivoted_cholesky(rank, 1e-8)
    Kb = ho.hadamard_matrix("rbf", x.float().double(), x.float().double(), t, t, 0.3, 1.1, B.float().double(), True)
    _, piv_ref = ol.pivoted_cholesky(torch.diagonal(Kb).clone(), lambda i: Kb[i], rank, 1e-8)
    assert int(piv[0]) == int(piv_ref[0]) == int(torch.argmax(torch.diagonal(Kb)))   # first pivot: argmax of s B[t_i, t_i]
    R = lt.double().cpu()
    # the factor reproduces the pivot rows of K o B
    pr = piv.cpu()
    assert torch.allclose(R.t() @ R[:, pr], Kb[:, pr], atol=1e-4)


@pytest.mark.parametrize("backend", BACKENDS)
def test_mbcg_and_mll_with_task_noise(cuda_dev, backend):
    g = torch.Generator().manual_seed(13)
    n, d, T = 600, 3, 3
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    t = torch.randint(0, T, (n,), generator=g)
    B = _random_B(T, g)
    task_noise = torch.tensor([0.05, 0.2, 0.1], dtype=torch.float64)
    y = torch.randn(n, generator=g, dtype=torch.float64)
    ls, os_ = 0.35, 1.2
    p = _plan(cuda_dev, x.float(), backend=backend)
    p.set_hypers("rbf", ls, os_, 0.0)
    p.set_tasks(t.to(cuda_dev), None, T)
    p.set_task_covar(B.float())
    p.set_noise_diag(task_noise[t].float().to(cuda_dev))
    A = ho.khat("rbf", x.float().double(), t, ls, os_, B.float().double(), task_noise.float().double())
    rhs = torch.randn(n, 3, generator=g, dtype=torch.float64)
    sol, _, info = p.mbcg(rhs.float().to(cuda_dev), tolerance=1e-5, max_iter=2000)
    ref = torch.linalg.solve(A, rhs)
    assert torch.linalg.norm(sol.double().cpu() - ref) <= 1e-3 * torch.linalg.norm(ref), info
    # the MLL: exact inverse quadratic form; the stochastic log det within the estimator's error
    tp = 15
    gg = torch.Generator().manual_seed(3)
    rad = (torch.randint(0, 2, (n, tp), generator=gg).float() * 2 - 1).to(cuda_dev)
    res, _ = p.mll(y.float().to(cuda_dev), None, None, rad, num_probes=tp, precond_rank=0, cg_tol=1e-4, max_tridiag_iter=60,
                   max_cg_iter=2000)
    iq_ref = float(y @ torch.linalg.solve(A, y))
    ld_ref = float(torch.linalg.slogdet(A)[1])
    assert abs(res.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0
    # preconditioned MLL (pivoted Cholesky of K o B, per-task noise diagonal): the same inverse quadratic form
    eps1 = torch.randn(30, tp, generator=gg).to(cuda_dev)
    eps2 = torch.randn(n, tp, generator=gg).to(cuda_dev)
    res2, _ = p.mll(y.float().to(cuda_dev), eps1, eps2, rad, num_probes=tp, precond_rank=30, min_precond_size=100, cg_tol=1e-4,
                    max_tridiag_iter=60, max_cg_iter=2000)
    assert res2.precond_rank > 0
    assert abs(res2.inv_quad - iq_ref) <= 1e-3 * abs(iq_ref)
    assert abs(res2.logdet - ld_ref) <= 0.05 * abs(ld_ref) + 5.0


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("cross", [False, True])
def test_hyper_and_task_covar_gradients(cuda_dev, backend, ard, cross):
    g = torch.Generator().manual_seed(17 + 2 * ard + cross)
    n1, n2, d, T, s = 300, 241, 4, 3, 5
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64).float().double()
    x2 = torch.rand(n2, d, generator=g, dtype=torch.float64).float().double() if cross else x1
    t1 = torch.randint(0, T, (n1,), generator=g)
    t2 = torch.randint(0, T, (n2,), generator=g) if cross else t1
    B = _random_B(T, g).float().double()
    L = torch.randn(n1, s, generator=g, dtype=torch.float64).float().double()
    R = torch.randn(x2.size(0), s, generator=g, dtype=torch.float64).float().double()
    ls0 = [0.4, 0.5, 0.6, 0.7] if ard else [0.5]
    os0 = 1.3
    p = _plan(cuda_dev, x1.float(), x2.float() if cross else None, backend)
    p.set_hypers("matern52", ls0 if ard else ls0[0], os0, 0.0)
    p.set_tasks(t1.to(cuda_dev), t2.to(cuda_dev) if cross else None, T)
    p.set_task_covar(B.float())
    gl, go = p.bilinear_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    dB = p.task_covar_grad(L.float().to(cuda_dev), R.float().to(cuda_dev))
    ls = torch.tensor(ls0, dtype=torch.float64, requires_grad=True)
    os_ = torch.tensor(os0, dtype=torch.float64, requires_grad=True)
    Bv = B.clone().requires_grad_(True)
    K = ho.hadamard_matrix("matern52", x1, x2, t1, t2, ls if ard else ls[0], os_, Bv, not cross)
    F = (L * (K @ R)).sum()
    F.backward()
    scale = float((K.detach().abs() @ R.abs() * L.abs()).sum())
    # relative to each gradient, plus the fp32 rounding floor of the sums (a few 1e-7 of sum |L| |K o B| |R|)
    for a, b in zip(gl, ls.grad.tolist()):
        assert abs(a - b) <= 1e-3 * abs(b) + 2e-6 * scale / min(ls0), (gl, ls.grad)
    assert abs(go - float(os_.grad)) <= 1e-3 * abs(float(os_.grad)) + 2e-6 * scale / os0
    assert torch.all((dB - Bv.grad).abs() <= 1e-3 * Bv.grad.abs() + 2e-6 * scale / float(B.abs().min())), (dB, Bv.grad)
    # repeated calls: identical bits
    assert torch.equal(dB, p.task_covar_grad(L.float().to(cuda_dev), R.float().to(cuda_dev)))


def test_nan_propagation(cuda_dev):
    g = torch.Generator().manual_seed(19)
    n, d, T = 200, 3, 2
    x = torch.rand(n, d, generator=g)
    x[17, 1] = float("nan")
    t = torch.randint(0, T, (n,), generator=g)
    p = _plan(cuda_dev, x)
    p.set_hypers("rbf", 0.5, 1.0, 0.1)
    p.set_tasks(t.to(cuda_dev), None, T)
    p.set_task_covar(torch.eye(T))
    V = torch.randn(n, 2, generator=g).to(cuda_dev)
    assert torch.isnan(p.kmv(V)).all()
    assert torch.isnan(p.task_covar_grad(V, V)).all()
    gl, go = p.bilinear_grad(V, V)
    assert math.isnan(go) and all(math.isnan(v) for v in gl)


@pytest.mark.parametrize("backend", BACKENDS)
def test_ciq_and_lanczos_against_dense(cuda_dev, backend):
    """The multi-shift MINRES product and the Lanczos tridiagonal run on K o B + D: both against the dense fp64 operator."""
    g = torch.Generator().manual_seed(23)
    n, d, T = 400, 3, 3
    x = torch.rand(n, d, generator=g, dtype=torch.float64).float().double()
    t = torch.randint(0, T, (n,), generator=g)
    B = _random_B(T, g).float().double()
    task_noise = torch.tensor([0.1, 0.3, 0.2], dtype=torch.float64).float().double()
    p = _plan(cuda_dev, x.float(), backend=backend)
    p.set_hypers("rbf", 0.4, 1.0, 0.0)
    p.set_tasks(t.to(cuda_dev), None, T)
    p.set_task_covar(B.float())
    p.set_noise_diag(task_noise[t].float().to(cuda_dev))
    A = ho.khat("rbf", x, t, 0.4, 1.0, B, task_noise)
    b = torch.randn(n, 4, generator=g, dtype=torch.float64)
    tau = [0.05 * 3 ** q for q in range(6)]
    w = [0.2, 0.1, 0.3, 0.15, 0.05, 0.2]
    out, _ = p.ciq_sqrt_matmul(b.float().to(cuda_dev), tau, w, tol=1e-6, max_iter=2000, warn=False)
    ref = A @ sum(wq * torch.linalg.solve(A + tq * torch.eye(n, dtype=torch.float64), b) for tq, wq in zip(tau, w))
    assert torch.linalg.norm(out.double().cpu() - ref) <= 2e-3 * torch.linalg.norm(ref)
    q, tm = p.lanczos(torch.randn(n, generator=g).to(cuda_dev), 20)
    Q = q.double().cpu()
    assert torch.allclose(Q.t() @ A @ Q, tm.double().cpu(), atol=2e-3 * float(torch.linalg.matrix_norm(A, 2)))


def test_refusals(cuda_dev):
    from gpytorch_b200.engine import Plan

    n = 64
    x = torch.rand(n, 2, device=cuda_dev)
    t = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    ski = Plan(x)
    ski.set_ski([8, 8], [-0.5, -0.5], [0.3, 0.3])
    ski.set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="SKI"):
        ski.set_tasks(t, None, 1)
    terms = [Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)]
    sp = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    sp.set_sum(terms)
    with pytest.raises(RuntimeError, match="kernel-sum"):
        sp.set_tasks(t, None, 1)
    lr = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    lr.set_lowrank(torch.randn(n, 2, device=cuda_dev))
    with pytest.raises(RuntimeError, match="low-rank"):
        lr.set_tasks(t, None, 1)
    sh = Plan(x, row_begin=0, row_count=32).set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="row-sharded"):
        sh.set_tasks(t, None, 1)
    p = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    p.set_tasks(t, None, 1)
    with pytest.raises(RuntimeError, match="task covariance not set"):
        p.kmv(torch.ones(n, 1, device=cuda_dev))
    p.set_task_covar(torch.ones(1, 1))
    with pytest.raises(RuntimeError, match="task indices"):
        p.kmv_input_grad(torch.ones(n, 1, device=cuda_dev), torch.ones(n, 1, device=cuda_dev))
    with pytest.raises(RuntimeError, match="task indices"):
        p.set_lowrank(torch.randn(n, 2, device=cuda_dev))
    # clearing the tasks gives the plain operator back
    plain = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    v = torch.randn(n, 3, device=cuda_dev)
    p.set_tasks(None)
    assert torch.equal(p.kmv(v), plain.kmv(v))


# ---- the model layer: IndexKernel x RBF with HadamardGaussianLikelihood through ExactGP ------------------------------------------
def _model(dev, n, T, seed):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultivariateNormal

    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 2, generator=g)
    i = torch.randint(0, T, (n, 1), generator=g)
    y = torch.sin(6 * x[:, 0]) * (1 + i[:, 0].float()) + 0.1 * torch.randn(n, generator=g)

    class MultitaskGPModel(models.ExactGP):
        def __init__(self, train_x, train_i, train_y, likelihood):
            super().__init__((train_x, train_i), train_y, likelihood)
            self.mean_module = means.ConstantMean()
            self.covar_module = kernels.ScaleKernel(kernels.RBFKernel())
            self.task_covar_module = kernels.IndexKernel(num_tasks=T, rank=1)

        def forward(self, x, i):
            covar = self.covar_module(x).mul(self.task_covar_module(i))
            return MultivariateNormal(self.mean_module(x), covar)

    torch.manual_seed(seed)
    lik = likelihoods.HadamardGaussianLikelihood(num_tasks=T)
    m = MultitaskGPModel(x.to(dev), i.to(dev), y.to(dev), lik).to(dev)
    m.likelihood.noise = torch.linspace(0.05, 0.2, T, device=dev)
    m.covar_module.base_kernel.lengthscale = 0.3
    return m, x.double(), i.reshape(-1), y.double()


def _oracle_params(m):
    """fp64 leaf copies of the model's raw parameters and the oracle's constrained values built from them (same transforms)."""
    raw = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in m.named_parameters()}
    sp = torch.nn.functional.softplus
    ls = sp(raw["covar_module.base_kernel.raw_lengthscale"]).reshape(())
    os_ = sp(raw["covar_module.raw_outputscale"])
    B = ho.index_covar(raw["task_covar_module.covar_factor"], sp(raw["task_covar_module.raw_var"]))
    noise = 1e-4 + sp(raw["likelihood.noise_covar.raw_noise"])
    mean = raw["mean_module.raw_constant"]
    return raw, ls, os_, B, noise, mean


@pytest.mark.parametrize("branch", ["cholesky", "cg"])
def test_model_mll_and_gradients_against_fp64(cuda_dev, branch):
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, T = 300, 3
    m, x, i, y = _model(cuda_dev, n, T, 31)
    m.train()
    raw, ls, os_, B, noise, mean = _oracle_params(m)
    if branch == "cholesky":
        mll = ExactMarginalLogLikelihood(m.likelihood, m)
        out = m(*m.train_inputs)
        loss = mll(out, m.train_targets, m.train_inputs)
        ref = ho.mll("rbf", x, i, y, ls, os_, B, noise, mean)
        tol_v, tol_g = 1e-4, 2e-3
    else:
        # CG branch: the inverse quadratic form, whose gradient has no stochastic trace term
        with settings.max_cholesky_size(0), settings.cg_tolerance(1e-6):
            out = m(*m.train_inputs)
            khat = m.likelihood(out, m.train_inputs).lazy_covariance_matrix
            loss = khat.inv_quad((m.train_targets - out.mean).unsqueeze(-1))
        A = ho.khat("rbf", x, i, ls, os_, B, noise)
        r = y - mean
        ref = r @ torch.linalg.solve(A, r)
        tol_v, tol_g = 1e-3, 5e-3
    loss.backward()
    ref.backward()
    assert abs(float(loss) - float(ref)) <= tol_v * abs(float(ref)) + 1e-5
    for k, v in m.named_parameters():
        if raw[k].grad is None:
            continue
        got, want = v.grad.double().cpu(), raw[k].grad
        assert torch.linalg.norm(got - want) <= tol_g * torch.linalg.norm(want) + 1e-5, (k, got, want)
    # dB reached the IndexKernel parameters, and the per-task noise trains
    assert m.task_covar_module.covar_factor.grad.abs().sum() > 0 and m.likelihood.noise_covar.raw_noise.grad.abs().sum() > 0


@pytest.mark.parametrize("fast", [False, True])
def test_model_posterior_against_fp64(cuda_dev, fast):
    from gpytorch_b200 import settings

    n, T = 300, 3
    m, x, i, y = _model(cuda_dev, n, T, 37)
    _, ls, os_, B, noise, mean = _oracle_params(m)
    g = torch.Generator().manual_seed(41)
    xs = torch.rand(40, 2, generator=g)
    its = torch.randint(0, T, (40, 1), generator=g)
    m.eval()
    with torch.no_grad(), settings.fast_pred_var(fast), settings.max_root_decomposition_size(300):
        post = m(xs.to(cuda_dev), its.to(cuda_dev))
        mu, var = post.mean.double().cpu(), post.variance.double().cpu()
    with torch.no_grad():
        mu_ref, cov_ref = ho.posterior("rbf", x, i, y, xs.double(), its.reshape(-1), ls, os_, B, noise, mean)
    assert torch.allclose(mu, mu_ref, atol=2e-3 * float(y.abs().max()))
    assert torch.allclose(var, torch.diagonal(cov_ref), atol=2e-3 * float(B.diagonal().max() * os_))


def test_model_ciq_rsample(cuda_dev):
    from gpytorch_b200 import settings

    n, T = 3000, 4
    m, _, _, _ = _model(cuda_dev, n, T, 43)
    m.train()
    with torch.no_grad(), settings.ciq_samples(True):
        out = m.likelihood(m(*m.train_inputs), m.train_inputs)
        s = out.rsample(torch.Size([3]))
    assert s.shape == (3, n) and torch.isfinite(s).all()
