"""Missing observations on the engine: the masked Kronecker operator P_r ((s K) (x) B) P_c^T (gp_plan_set_kron_observed) against
tests/kron_mask_oracle.py within its derived bound on both data-plan backends, and settings.observation_nan_policy("mask")
through ExactMarginalLogLikelihood and ExactGP prediction on Kronecker, plain and Hadamard models.

Products: T in {1, 2, 5, 8, 32}, t in {1, 11, 33}, missing patterns none, one entry, 10 / 50 / 90 %, a whole point, a whole task
and observed rows straddling a 64-row tile, square and cross plans with N off the tile.  The largest error-to-bound ratio per
check is printed by test_zz_report (-s)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import hadamard_oracle as ho  # noqa: E402
import kmv_oracle as kmo  # noqa: E402
import kron_mask_oracle as km  # noqa: E402
import kron_oracle as ko  # noqa: E402
import multitask_oracle as mo  # noqa: E402

BACKENDS = ["tcgen05", "simt"]
PATH = {"tcgen05": "tc", "simt": "simt"}
LS, OS = 0.5, 1.3
RATIOS = {}


def _within(key, tag, got, ref, bnd):
    got, ref, bnd = (torch.as_tensor(v, dtype=torch.float64).cpu() for v in (got, ref, bnd))
    err = (got - ref).abs()
    frac = torch.where(bnd > 0, err / bnd, torch.where(err > 0, torch.inf, 0.0))
    assert bool(torch.isfinite(got).all()) and float(frac.max()) <= 1.0, (tag, key, float(frac.max()))
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(frac.max()))


def _kron(dev, kind, x1, x2, T, B, backend, rows=None, cols=None, noise=0.0, ls=LS):
    from gpytorch_b200.engine import KronPlan, Plan

    data = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend).set_hypers(kind, ls, OS, 0.0)
    n2 = (x1 if x2 is None else x2).size(0)
    geo = kmo.geometry(x1.size(0), n2, x1.size(1), backend, data.info()["n_sm"])
    p = KronPlan(data, T)
    p.set_noise(noise)
    p.set_task_covar(B)
    if rows is not None or cols is not None:
        p.set_observed(rows, cols)
    return p, geo


# (T, t, pattern, N1, N2 or None)
CASES = [(1, 11, "one", 333, None), (2, 1, "frac10", 333, None), (5, 11, "frac50", 333, None), (8, 33, "frac90", 333, None),
         (32, 1, "frac50", 150, None), (5, 11, "point", 333, None), (5, 11, "task", 333, None), (2, 11, "straddle", 333, None),
         (8, 33, "none", 333, None), (5, 11, "frac50", 210, 333), (2, 1, "straddle", 333, 130)]


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"T{c[0]}-t{c[1]}-{c[2]}-{c[3]}x{c[4]}")
def test_products_within_bound(cuda_dev, backend, case):
    T, t, pat, n1, n2 = case
    kind = ["rbf", "matern32", "matern52", "matern12"][CASES.index(case) % 4]
    x1 = kmo.points(n1, 4, 11)
    x2 = None if n2 is None else kmo.points(n2, 4, 12)
    B = mo.random_B(T, 13)
    rows = km.pattern(pat, n1, T, 14)
    cols = rows if n2 is None else km.pattern(pat, n2, T, 15)
    if pat == "none":
        rows = cols = None
        rows_arg = cols_arg = torch.arange(n1 * T)   # an explicit all-observed mask: the unmasked operator
    else:
        rows_arg, cols_arg = rows, cols
    noise = 0.1 if n2 is None else 0.0
    p, geo = _kron(cuda_dev, kind, x1, x2, T, B, backend, rows_arg, None if n2 is None else cols_arg, noise=noise)
    nc = cols.numel() if cols is not None else (n2 or n1) * T
    V = torch.randn(nc, t, generator=torch.Generator().manual_seed(16), dtype=torch.float64).float()
    xd1, xd2, Vd = x1.to(cuda_dev), None if x2 is None else x2.to(cuda_dev), V.to(cuda_dev)
    out = p.kmv(Vd, add_noise=bool(noise))
    ref = km.mask_exact(kind, xd1, xd2, B, LS, OS, Vd, T, t, rows, cols, noise=noise)
    _within(("kmv", PATH[backend]), f"{case}", out, ref, km.mask_bound(kind, xd1, xd2, B, LS, OS, Vd, T, t, rows, cols, geo,
                                                                        exact=ref, noise=noise))
    assert torch.equal(out, p.kmv(Vd, add_noise=bool(noise)))   # deterministic
    if pat == "none":   # an all-observed mask is the unmasked plan, bit for bit
        q, _ = _kron(cuda_dev, kind, x1, x2, T, B, backend, noise=noise)
        assert torch.equal(out, q.kmv(Vd, add_noise=bool(noise)))


@pytest.mark.parametrize("backend", BACKENDS)
def test_identity_mask_on_the_masked_path_is_bit_identical(cuda_dev, backend):
    """A cross plan observing every row but one column: the observed rows are bit-identical to the unmasked product of the
    zero-filled V (the masked mix adds exact zeros where the unmasked one multiplies them)."""
    T, t, n1, n2 = 3, 5, 333, 200
    x1, x2 = kmo.points(n1, 4, 21), kmo.points(n2, 4, 22)
    B = mo.random_B(T, 23)
    cols = torch.cat([torch.arange(0, 77), torch.arange(78, n2 * T)])
    p, _ = _kron(cuda_dev, "rbf", x1, x2, T, B, backend, None, cols)
    q, _ = _kron(cuda_dev, "rbf", x1, x2, T, B, backend)
    V = torch.randn(cols.numel(), t, generator=torch.Generator().manual_seed(24)).to(cuda_dev)
    Vf = torch.zeros(n2 * T, t, device=cuda_dev)
    Vf[cols.to(cuda_dev)] = V
    assert torch.equal(p.kmv(V), q.kmv(Vf))


@pytest.mark.parametrize("backend", BACKENDS)
def test_agrees_with_hadamard_over_the_observed_rows(cuda_dev, backend):
    from gpytorch_b200.engine import Plan

    T, t, n = 5, 7, 400
    x = kmo.points(n, 3, 31)
    B = mo.random_B(T, 32)
    rows = km.pattern("frac50", n, T, 33)
    p, _ = _kron(cuda_dev, "matern52", x, None, T, B, backend, rows, None, noise=0.05)
    xr = x[rows // T]
    h = Plan(xr.to(cuda_dev), backend=backend).set_hypers("matern52", LS, OS, 0.05)
    h.set_tasks((rows % T).to(cuda_dev), None, T)
    h.set_task_covar(B)
    V = torch.randn(rows.numel(), t, generator=torch.Generator().manual_seed(34)).to(cuda_dev)
    A = km.mask_matrix("matern52", x, None, LS, OS, B, rows, rows)
    scale = A.abs() @ V.double().abs().cpu() + 0.05 * V.double().abs().cpu()
    a, b = p.kmv(V, add_noise=True).double().cpu(), h.kmv(V, add_noise=True).double().cpu()
    assert torch.all((a - b).abs() <= 1e-5 * scale + 1e-7)


@pytest.mark.parametrize("backend", BACKENDS)
def test_rows_diagonal_and_pivots(cuda_dev, backend):
    T, n = 4, 300
    x = kmo.points(n, 3, 41)
    B = mo.random_B(T, 42)
    rows = km.pattern("frac50", n, T, 43)
    p, _ = _kron(cuda_dev, "rbf", x, None, T, B, backend, rows, None)
    A = km.mask_matrix("rbf", x, None, LS, OS, B, rows, rows)
    idx = torch.tensor([0, 1, rows.numel() // 2, rows.numel() - 1])
    got = p.rows(idx.to(cuda_dev)).double().cpu()
    assert got.shape == (4, rows.numel())
    assert torch.allclose(got, A[idx], rtol=1e-5, atol=1e-6)
    bad = p.rows(torch.tensor([rows.numel()], device=cuda_dev))   # outside the observed rows: a NaN row, as unmasked
    assert torch.isnan(bad).all()
    dg = p.diag().double().cpu()
    assert torch.allclose(dg, torch.diagonal(A), rtol=1e-6, atol=1e-7)
    lt, piv, _ = p.pivoted_cholesky(10, 0.0)
    ref_lt, ref_piv = ko.pivoted_cholesky(A, 10)
    assert int(piv[0]) == int(torch.argmax(torch.diagonal(A).float()))   # the diagonal s B[a, a] is not constant
    assert int(piv[0]) == int(ref_piv[0])
    assert torch.allclose(lt[0].double().cpu(), ref_lt[0].double(), atol=1e-5)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("cross", [False, True])
def test_dB_and_gradients_within_bound(cuda_dev, backend, cross):
    T, t, d = 3, 6, 3
    n1, n2 = (2049, 1000) if cross else (1450, None)
    x1 = kmo.points(n1, d, 51)
    x2 = kmo.points(n2, d, 52) if cross else None
    B = mo.random_B(T, 53)
    rows = km.pattern("frac10", n1, T, 54)
    cols = km.pattern("frac50", n2, T, 55) if cross else rows
    g = torch.Generator().manual_seed(56)
    L, R = torch.randn(rows.numel(), t, generator=g), torch.randn(cols.numel(), t, generator=g)
    p, geo = _kron(cuda_dev, "matern32", x1, x2, T, B, backend, rows, cols if cross else None)
    x1d, x2d, Ld, Rd = x1.to(cuda_dev), None if x2 is None else x2.to(cuda_dev), L.to(cuda_dev), R.to(cuda_dev)
    dB = p.task_covar_grad(Ld, Rd)
    _within(("dB", PATH[backend]), f"cross={cross}", dB, km.mask_dB("matern32", x1d, x2d, LS, OS, Ld, Rd, T, t, rows, cols),
            km.mask_dB_bound("matern32", x1d, x2d, LS, OS, Ld, Rd, T, t, rows, cols, geo))
    assert torch.equal(dB, p.task_covar_grad(Ld, Rd))
    gl, gs = p.bilinear_grad(Ld, Rd)
    path = PATH[backend]
    rl, rs = km.mask_grad("matern32", x1d, x2d, B, LS, OS, Ld, Rd, T, t, rows, cols)
    bl, bs = km.mask_grad_bound("matern32", x1d, x2d, B, LS, OS, Ld, Rd, T, t, rows, cols, path, p.data.info()["n_sm"])
    _within(("grad", path), f"cross={cross}", torch.tensor(list(gl) + [gs]), torch.cat([rl.cpu(), torch.tensor([float(rs)])]),
            torch.cat([bl.cpu(), torch.tensor([float(bs)])]))


def test_nan_and_refusals(cuda_dev):
    T, n = 3, 200
    x = kmo.points(n, 3, 61)
    B = mo.random_B(T, 62)
    rows = km.pattern("frac50", n, T, 63)
    p, _ = _kron(cuda_dev, "rbf", x, None, T, B, "auto", rows, None)
    V = torch.randn(rows.numel(), 4, device=cuda_dev)
    Bn = B.clone()
    Bn[1, 2] = float("nan")
    p.set_task_covar(Bn)
    assert torch.isnan(p.kmv(V)).all()              # a non-finite B: NaN on every observed row
    p.set_task_covar(B)
    assert torch.isfinite(p.kmv(V)).all()
    with pytest.raises(RuntimeError):
        p.set_observed(rows, rows[1:])              # a square plan takes equal masks
    with pytest.raises(RuntimeError):
        p.set_observed(rows.flip(0), None)          # not increasing
    with pytest.raises(RuntimeError):
        p.set_observed(torch.tensor([0, n * T]), None)   # out of range
    p.set_observed(None, None)                      # unmasked again
    assert p.kmv(torch.randn(n * T, 2, device=cuda_dev)).shape == (n * T, 2)


# ---- models -------------------------------------------------------------------------------------------------------------------
def _mt_model(dev, n, T, seed, frac):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultitaskMultivariateNormal

    g = torch.Generator().manual_seed(seed)
    x = torch.linspace(0, 1, n).unsqueeze(-1)
    y = torch.stack([torch.sin(x[:, 0] * 2 * math.pi), torch.cos(x[:, 0] * 2 * math.pi)][:T], -1) + 0.1 * torch.randn(n, T, generator=g)
    y[torch.rand(n, T, generator=g) < frac] = float("nan")

    class MultitaskGPModel(models.ExactGP):
        def __init__(self, train_x, train_y, likelihood):
            super().__init__(train_x, train_y, likelihood)
            self.mean_module = means.MultitaskMean(means.ConstantMean(), num_tasks=T)
            self.covar_module = kernels.MultitaskKernel(kernels.RBFKernel(), num_tasks=T, rank=1)

        def forward(self, x):
            return MultitaskMultivariateNormal(self.mean_module(x), self.covar_module(x))

    torch.manual_seed(seed)
    lik = likelihoods.MultitaskGaussianLikelihood(num_tasks=T)
    return MultitaskGPModel(x.to(dev), y.to(dev), lik).to(dev), x.double(), y.double()


def _params(m, T):
    sp = torch.nn.functional.softplus
    raw = {k: v.detach().double().cpu() for k, v in m.named_parameters()}
    ls = sp(raw["covar_module.data_covar_module.raw_lengthscale"]).reshape(())
    B = ko.index_covar(raw["covar_module.task_covar_module.covar_factor"], sp(raw["covar_module.task_covar_module.raw_var"]))
    tn = 1e-4 + sp(raw["likelihood.raw_task_noises"])
    noise = 1e-4 + sp(raw["likelihood.raw_noise"])
    mean = torch.stack([raw[f"mean_module.base_means.{a}.raw_constant"] for a in range(T)]).reshape(-1)
    return ls, B, tn, noise, mean


def _dense_masked(x, y, xs, ls, B, tn, noise, mean):
    """fp64 masked MLL (divided by the full n T) and the posterior of f at xs conditioned on the observed rows."""
    n, T = y.shape
    obs = ~torch.isnan(y.reshape(-1))
    A = ko.khat("rbf", x, ls, 1.0, B, tn, noise)[obs][:, obs]
    r = (y - mean).reshape(-1)[obs]
    L = torch.linalg.cholesky(A)
    a = torch.cholesky_solve(r.unsqueeze(-1), L).squeeze(-1)
    mll = -0.5 * ((r * a).sum() + 2 * torch.log(torch.diagonal(L)).sum() + obs.sum() * math.log(2 * math.pi)) / (n * T)
    Ksx = ko.kron_matrix("rbf", xs, x, ls, 1.0, B, False)[:, obs]
    Kss = ko.kron_matrix("rbf", xs, xs, ls, 1.0, B, True)
    mu = (Ksx @ a).reshape(-1, T) + mean
    cov = Kss - Ksx @ torch.cholesky_solve(Ksx.t(), L)
    return mll, mu, cov


@pytest.mark.parametrize("precond", [False, True])
def test_kron_model_mll_and_posterior_against_dense(cuda_dev, precond):
    """The masked MLL (CG branch, with and without the pivoted-Cholesky preconditioner), the posterior mean and the exact and
    fast_pred_var covariances against the fp64 conditional on the observed rows."""
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, T = 500, 2
    m, x, y = _mt_model(cuda_dev, n, T, 71, 0.3)
    with torch.no_grad():
        m.covar_module.data_covar_module.lengthscale = 0.2
    xs = torch.linspace(0, 1, 37).unsqueeze(-1).double()
    ref_mll, ref_mu, ref_cov = _dense_masked(x, y, xs, *_params(m, T))
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    m.train()
    with settings.observation_nan_policy("mask"), settings.max_cholesky_size(0), settings.cg_tolerance(1e-6), settings.eval_cg_tolerance(1e-6), \
            settings.max_cg_iterations(3000), settings.num_trace_samples(15), settings.probe_seed(5), \
            settings.min_preconditioning_size(0 if precond else 10**9):
        val = mll(m(m.train_inputs[0]), m.train_targets)
        val.backward()
        assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
        m.eval()
        with torch.no_grad():
            post = m(xs.float().to(cuda_dev))
            mu, cov = post.mean.double().cpu(), post.covariance_matrix.double().cpu()
            with settings.fast_pred_var(), settings.max_root_decomposition_size(300):
                m._clear_caches()
                cov_love = m(xs.float().to(cuda_dev)).covariance_matrix.double().cpu()
    assert abs(float(val) - float(ref_mll)) < 2e-2 * abs(float(ref_mll)) + 2e-2
    assert torch.allclose(mu, ref_mu, atol=2e-3), (mu - ref_mu).abs().max()
    assert torch.allclose(cov, ref_cov, atol=2e-3), (cov - ref_cov).abs().max()
    assert torch.allclose(cov_love.diagonal(), ref_cov.diagonal(), atol=5e-3), (cov_love.diagonal() - ref_cov.diagonal()).abs().max()


def test_reference_notebook_with_missing_targets_trains(cuda_dev):
    """The reference's Kronecker notebook with about 30 % of train_y NaN: 50 Adam steps under observation_nan_policy("mask"), the
    fp64 dense masked MLL at the trained parameters close to the engine's, and the posterior mean close to the truth."""
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    n, T = 100, 2
    m, x, y = _mt_model(cuda_dev, n, T, 0, 0.3)
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.1)
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    with settings.observation_nan_policy("mask"):
        for _ in range(50):
            opt.zero_grad()
            loss = -mll(m(m.train_inputs[0]), m.train_targets)
            loss.backward()
            opt.step()
        assert math.isfinite(float(loss))
        xs = torch.linspace(0, 1, 51).unsqueeze(-1)
        ref_mll, ref_mu, _ = _dense_masked(x, y, xs.double(), *_params(m, T))
        m.eval()
        with torch.no_grad():
            mu = m.likelihood(m(xs.to(cuda_dev))).mean.double().cpu()
    assert abs(-float(loss) - float(ref_mll)) < 0.05 * abs(float(ref_mll)) + 0.05
    assert torch.allclose(mu, ref_mu, atol=5e-3), (mu - ref_mu).abs().max()
    truth = torch.stack([torch.sin(xs[:, 0] * 2 * math.pi), torch.cos(xs[:, 0] * 2 * math.pi)], -1).double()
    assert torch.all((mu - truth).abs().mean(0) < 0.08), (mu - truth).abs().mean(0)


def test_no_missing_entries_is_bit_identical_to_ignore(cuda_dev):
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    m, _, _ = _mt_model(cuda_dev, 300, 2, 81, 0.0)
    mll = ExactMarginalLogLikelihood(m.likelihood, m)
    xs = torch.linspace(0, 1, 11).unsqueeze(-1).to(cuda_dev)
    res = []
    for pol in ("ignore", "mask"):
        m.train()
        with settings.observation_nan_policy(pol), settings.probe_seed(3), torch.no_grad():
            v = mll(m(m.train_inputs[0]), m.train_targets)
            m.eval()
            res.append((v, m(xs).mean, m(xs).covariance_matrix))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def _plain_model(dev, x, y, hadamard=False, T=3):
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.distributions import MultivariateNormal

    class Plain(models.ExactGP):
        def __init__(self, tx, ty, lik):
            super().__init__(tx, ty, lik)
            self.mean_module = means.ConstantMean()
            self.covar_module = kernels.ScaleKernel(kernels.RBFKernel())
            if hadamard:
                self.task_covar_module = kernels.IndexKernel(num_tasks=T, rank=1)

        def forward(self, x, i=None):
            c = self.covar_module(x)
            if hadamard:
                c = c.mul(self.task_covar_module(i))
            return MultivariateNormal(self.mean_module(x), c)

    torch.manual_seed(0)
    lik = likelihoods.GaussianLikelihood()
    return Plain(x, y, lik).to(dev)


@pytest.mark.parametrize("hadamard", [False, True])
def test_plain_and_hadamard_models_equal_their_observed_subset(cuda_dev, hadamard):
    """NaN targets under "mask" against the same model built on the observed subset: posterior means bit for bit, the MLL equal
    to the subset model's MLL times n_obs / N (the MLL divides by the full N, as the reference does)."""
    from gpytorch_b200 import settings
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    g = torch.Generator().manual_seed(91)
    n, T = 1200, 3
    x = torch.rand(n, 2, generator=g).to(cuda_dev)
    ti = (torch.arange(n) % T).unsqueeze(-1).to(cuda_dev)
    y = torch.sin(4 * x[:, 0]) + 0.1 * torch.randn(n, generator=g).to(cuda_dev)
    y[torch.rand(n, generator=g).to(cuda_dev) < 0.25] = float("nan")
    obs = ~torch.isnan(y)
    ins = (x, ti) if hadamard else (x,)
    sub_ins = (x[obs], ti[obs]) if hadamard else (x[obs],)
    full = _plain_model(cuda_dev, ins, y, hadamard, T)
    sub = _plain_model(cuda_dev, sub_ins, y[obs], hadamard, T)
    sub.load_state_dict(full.state_dict())
    xs = torch.rand(50, 2, generator=g).to(cuda_dev)
    ts = (torch.arange(50) % T).unsqueeze(-1).to(cuda_dev)
    test_ins = (xs, ts) if hadamard else (xs,)
    vals, means_ = [], []
    with settings.observation_nan_policy("mask"), settings.probe_seed(4), settings.max_cholesky_size(0):
        for mdl, ins_ in ((full, ins), (sub, sub_ins)):
            mdl.train()
            vals.append(float(ExactMarginalLogLikelihood(mdl.likelihood, mdl)(mdl(*ins_), mdl.train_targets)))
            mdl.eval()
            with torch.no_grad():
                means_.append(mdl(*test_ins).mean)
    n_obs = int(obs.sum())
    assert torch.equal(means_[0], means_[1])
    assert abs(vals[0] - vals[1] * n_obs / n) <= 1e-5 * abs(vals[0])


def test_masked_operator_plans_are_square(cuda_dev):
    from gpytorch_b200.operators import KernelLinearOperator, MaskedLinearOperator

    x = torch.rand(300, 2, device=cuda_dev)
    op = KernelLinearOperator(x, None, "rbf", torch.tensor(0.5, device=cuda_dev))
    mask = torch.rand(300, device=cuda_dev) < 0.7
    mo_ = MaskedLinearOperator(op, mask, mask)
    assert mo_.same and mo_.plan().same and mo_.shape == (int(mask.sum()), int(mask.sum()))


def test_zz_report(cuda_dev):
    """Largest |engine - fp64| / bound per check (printed with -s)."""
    import subprocess
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"\n[kron mask] {smi.stdout.strip()}")
    for k, v in sorted(RATIOS.items()):
        print(f"[kron mask] {k}: max error / bound = {v:.3g}")
