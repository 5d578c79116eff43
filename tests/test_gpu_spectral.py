"""Spectral mixture kernels on the device (run with -m gpu): ONE engine operator (gp_plan_set_spectral, csrc/spectral.cu).  Every
comparison is against the fp64 oracle of tests/spectral_oracle.py: K.V entry by entry within its derived bound (also at time
stamps up to 1e5, where the reference's fp32 phase is off by far more), rows, diagonals, pivots, the MLL, the parameter
gradients, determinism, NaN inputs, refusals, and the public API (the reference's tutorial model, a long series, a batch)."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

import spectral_oracle as so  # noqa: E402
from oracle import linalg as ol, mll as om  # noqa: E402
import pivchol_oracle as po  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _params(Q, d, seed):
    """fp32-representable weights [Q], means and scales [Q, d] (the engine's own precision)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.rand(Q, generator=g) * 1.2 + 0.2)
    mu = (torch.rand(Q, d, generator=g) * 0.6 + 0.02)
    v = (torch.rand(Q, d, generator=g) * 0.4 + 0.05)
    return w, mu, v


def _points(n, d, seed, scale=6.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g) * scale - scale / 2


def _plan(dev, X1, X2, w, mu, v, S=1.0, noise=0.0):
    from gpytorch_b200.engine import Plan

    p = Plan(X1.to(dev), None if X2 is None else X2.to(dev)).set_hypers("rbf", 1.0, S, noise)
    return p.set_spectral(w, mu, v)


CASES = [  # Q, d, n1, n2 (None: square), t, S
    (1, 1, 63, None, 1, 1.0),
    (4, 1, 1000, 777, 16, 0.7),
    (16, 1, 129, None, 11, 1.3),
    (4, 2, 4099, None, 16, 1.0),
    (8, 4, 129, 63, 5, 2.0),
    (4, 8, 777, None, 16, 0.5),
    (3, 3, 1, 129, 3, 1.0),
    (10, 3, 200, None, 16, 1.0),
]


@pytest.mark.parametrize("case", CASES)
def test_kmv_within_bound(cuda_dev, case):
    Q, d, n1, n2, t, S = case
    w, mu, v = _params(Q, d, 100 + Q + d)
    x1 = _points(n1, d, 1)
    x2 = None if n2 is None else _points(n2, d, 2)
    xr = x1 if x2 is None else x2
    V = torch.randn(xr.size(0), t, generator=torch.Generator().manual_seed(3))
    p = _plan(cuda_dev, x1, x2, w, mu, v, S)
    out = p.kmv(V.to(cuda_dev)).double().cpu()
    ref = so.covariance(x1, xr, w, mu, v, S) @ V.double()
    bound = so.kmv_bound(x1, xr, w, mu, v, V, S)
    err = (out - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    p.close()


def test_phase_at_large_time_stamps(cuda_dev):
    """x = 0 .. 99 999 with one mean at 0.49: the engine stays within the |x|-independent bound, the reference-style fp32 formula
    2 pi (mu x - mu x') does not."""
    n, t = 100_000, 4
    x = torch.arange(n, dtype=torch.float32).reshape(-1, 1)
    w, mu, v = torch.tensor([0.8, 0.5]), torch.tensor([[0.49], [0.0625]]), torch.tensor([[2e-4], [1e-3]])
    V = torch.randn(n, t, generator=torch.Generator().manual_seed(5))
    p = _plan(cuda_dev, x, None, w, mu, v)
    out = p.kmv(V.to(cuda_dev)).double().cpu()
    rows = torch.cat([torch.arange(0, 8), torch.arange(n - 8, n), torch.tensor([50_000, 77_777])])
    xd, Vd = x.to(cuda_dev).double(), V.to(cuda_dev).double()
    ref = torch.cat([so.covariance(xd[r:r + 1], xd, w, mu, v) @ Vd for r in rows.tolist()]).cpu()
    bound = torch.cat([so.kmv_bound(xd[r:r + 1], xd, w, mu, v, Vd) for r in rows.tolist()]).cpu()
    err = (out[rows] - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # entry by entry: the engine's rows within the entry bound, the reference's fp32 formula 2 pi (mu x - mu x') far outside it
    K = so.covariance(xd[rows.to(cuda_dev)], xd, w, mu, v)
    eb = so.entry_bound(xd[rows.to(cuda_dev)], xd, w, mu, v)
    assert bool(((p.rows(rows.to(cuda_dev)).double() - K).abs() <= eb).all())
    xf, muf, vf = x.to(cuda_dev), mu.to(cuda_dev), v.to(cuda_dev)
    xr = xf[rows.to(cuda_dev)]
    naive = torch.zeros(rows.numel(), n, device=cuda_dev)
    for q in range(w.numel()):
        e = torch.exp((xr * vf[q] - (xf * vf[q]).reshape(1, -1)).pow(2) * (-2 * math.pi ** 2))
        c = torch.cos((xr * muf[q] - (xf * muf[q]).reshape(1, -1)) * (2 * math.pi))
        naive += float(w[q]) * e * c
    ratio = ((naive.double() - K).abs() / eb).max().item()
    assert ratio > 100, ratio
    p.close()


def test_q1_small_mean_matches_rbf_plan(cuda_dev):
    """Q = 1, mu -> 0: w exp(-2 pi^2 v^2 tau^2) is an RBF kernel of lengthscale 1 / (2 pi v) and outputscale w."""
    from gpytorch_b200.engine import Plan

    n, t = 3000, 16
    x = _points(n, 1, 8)
    w, mu, v = torch.tensor([1.3]), torch.tensor([[1e-7]]), torch.tensor([[0.35]])
    V = torch.randn(n, t, generator=torch.Generator().manual_seed(9)).to(cuda_dev)
    p = _plan(cuda_dev, x, None, w, mu, v)
    q = Plan(x.to(cuda_dev)).set_hypers("rbf", [1.0 / (2 * math.pi * 0.35)], 1.3, 0.0)
    assert rel(p.kmv(V), q.kmv(V)) < 1e-5
    p.close(), q.close()


def test_rows_diag_and_pivots(cuda_dev):
    n, Q, d = 700, 3, 2
    x = _points(n, d, 11)
    w, mu, v = _params(Q, d, 12)
    S = 0.8
    K = so.covariance(x, x, w, mu, v, S)
    p = _plan(cuda_dev, x, None, w, mu, v, S, noise=0.1)
    idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
    rows = p.rows(idx).double().cpu()
    assert bool(((rows - K[idx]).abs() <= so.entry_bound(x[idx], x, w, mu, v, S)).all())
    kd = S * float(w.double().sum()) ** d
    assert torch.allclose(p.diag().double().cpu(), torch.full((n,), kd, dtype=torch.float64), rtol=1e-6)
    bad = p.rows(torch.tensor([n, -1]))
    assert bool(bad.isnan().all())
    # pivots (PC_KIND_SPECTRAL): step 0 ties on the constant diagonal (lowest index on both sides); at every later step the two
    # best candidates of the fp64 greedy pivoting lie more than 2 rank times the entry bound apart (asserted, not assumed)
    g = torch.Generator().manual_seed(33)
    xp = torch.rand(48, d, generator=g) * 3 - 1.5
    wp, mup, vp = torch.rand(Q, generator=g) * 1.2 + 0.2, torch.rand(Q, d, generator=g) * 0.6 + 0.02, torch.rand(Q, d, generator=g) * 0.15 + 0.05
    Kp = so.covariance(xp, xp, wp, mup, vp, S)
    kdp = S * float(wp.double().sum()) ** d
    diag32 = torch.full((48,), float(torch.tensor(kdp, dtype=torch.float32)), dtype=torch.float64)
    rank = 10
    L, piv_o = ol.pivoted_cholesky(diag32, lambda i: Kp[i], rank)
    gaps = po.pivot_gaps(diag32, L, piv_o)
    assert gaps[0] == 0.0 and min(gaps[1:]) > 2 * rank * so.entry_bound(xp, xp, wp, mup, vp, S).max().item()
    pp = _plan(cuda_dev, xp, None, wp, mup, vp, S, noise=0.1)
    lt, piv, st = pp.pivoted_cholesky(rank, 1e-3)
    assert st == 0 and lt.size(0) == rank
    assert torch.equal(piv.cpu(), piv_o)
    pp.close()
    # cross plan: rows and the diagonal of K(x1, x2) with equal sizes
    x2 = _points(n, d, 13)
    pc = _plan(cuda_dev, x, x2, w, mu, v, S)
    Kc = so.covariance(x, x2, w, mu, v, S)
    assert bool(((pc.rows(idx).double().cpu() - Kc[idx]).abs() <= so.entry_bound(x[idx], x2, w, mu, v, S)).all())
    dc = pc.diag().double().cpu()
    assert bool(((dc - Kc.diagonal()).abs() <= so.entry_bound(x, x2, w, mu, v, S, diag=True)).all())
    p.close(), pc.close()


def test_mll_on_the_cg_path_matches_oracle(cuda_dev):
    n, Q, d, rank = 2500, 4, 1, 30
    x, y = om.synthetic_problem(n, d, 4, torch.float32)
    # a span of 10 gives the spectrum enough detail for the rank-30 preconditioner to fill (1e-3 tolerance); with noise 1 the fp32
    # oracle itself lands within 7e-6 of the fp64 one (at noise 0.1 the fp32 SLQ log-determinant alone moves the MLL by 2e-4)
    x = x * 10
    w, mu, v = _params(Q, d, 15)
    S, noise = 1.0, 1.0
    K = so.covariance(x, x, w, mu, v, S)
    p = _plan(cuda_dev, x, None, w, mu, v, S, noise=noise)
    pn = om.make_probe_noise(n, rank, 10, 7)
    kd = S * float(w.double().sum()) ** d
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, kd, noise, tuple(a.double() for a in pn), precond_size=rank, K=K)
    res, _ = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000)
    assert res.precond_rank == rank == o64.precond.L.size(1)
    assert abs(res.mll - o64.mll) <= 1e-4 * max(1.0, abs(o64.mll)), (res.mll, o64.mll)
    p.close()


@pytest.mark.parametrize("Q,d,S", [(1, 1, 1.0), (4, 1, 0.6), (16, 1, 1.0), (3, 2, 1.4), (8, 4, 1.0), (4, 8, 0.9)])
def test_bilinear_grad_matches_fp64_autograd_and_repeats_bit_for_bit(cuda_dev, Q, d, S):
    n, m, s = 500, 430, 13
    x1, x2 = _points(n, d, 21), _points(m, d, 22)
    w, mu, v = _params(Q, d, 23)
    g = torch.Generator().manual_seed(24)
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, x1, x2, w, mu, v, S)
    gl, gs = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    assert p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev)) == (gl, gs)
    wt, mt, vt, st = (t.double().clone().requires_grad_(True) for t in (w, mu, v, torch.tensor(S)))
    F = (L.double() * (so.covariance_torch(x1, x2, wt, mt, vt, st) @ R.double())).sum()
    F.backward()
    ref = torch.cat([wt.grad, mt.grad.reshape(-1), vt.grad.reshape(-1)])
    got = torch.tensor(gl, dtype=torch.float64)
    assert got.shape == ref.shape
    assert torch.allclose(got, ref, rtol=2e-4, atol=2e-4 * ref.abs().max().item())
    assert abs(gs - st.grad.item()) <= 2e-4 * max(abs(st.grad.item()), 1e-3 * ref.abs().max().item())
    # repeated products are bit-identical too
    V = torch.randn(m, 7, generator=g).to(cuda_dev)
    assert torch.equal(p.kmv(V), p.kmv(V))
    p.close()


def test_nan_inputs_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    n, d = 300, 2
    w, mu, v = _params(3, d, 31)
    x = _points(n, d, 31)
    x[5, 1] = float("nan")
    p = _plan(cuda_dev, x, None, w, mu, v)
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(p.kmv(V).isnan().all())
    assert bool(p.rows(torch.tensor([0, 1])).isnan().all()) and bool(p.diag().isnan().all())
    gl, gs = p.bilinear_grad(V, V)
    assert all(math.isnan(t) for t in gl + [gs])
    q = _plan(cuda_dev, _points(n, d, 32), None, w, mu, v)
    lib = q.lib
    other = Plan(_points(n, d, 33).to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    tasks = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    for call, fn in [("gp_plan_set_backend", lambda: _lib.check(lib.gp_plan_set_backend(q._h, 2))),
                     ("gp_plan_set_tasks", lambda: q.set_tasks(tasks, None, 2)),
                     ("gp_plan_set_sum", lambda: q.set_sum([other])),
                     ("gp_plan_set_product", lambda: q.set_product([other, other])),
                     ("gp_plan_set_ski", lambda: q.set_ski([16] * d, [-4.0] * d, [0.5] * d)),
                     ("gp_plan_set_additive", lambda: q.set_additive(1, [1.0] * d)),
                     ("gp_plan_set_kron", lambda: _lib.check(lib.gp_plan_set_kron(q._h, other._h, 2))),
                     ("gp_plan_set_deriv", lambda: _lib.check(lib.gp_plan_set_deriv(q._h, other._h)))]:
        with pytest.raises(RuntimeError, match=f"{call} is not available on a spectral mixture plan"):
            fn()
    with pytest.raises(RuntimeError, match="gp_kmv_input_grad is not available on a spectral mixture plan"):
        q.kmv_input_grad(V, V)
    with pytest.raises(RuntimeError, match="gp_kdense_input_grad is not available on a spectral mixture plan"):
        q.dense_input_grad(torch.zeros(n, n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="a spectral mixture plan as a term is not available"):
        other.set_sum([q])
    with pytest.raises(RuntimeError, match="a spectral mixture plan as a factor is not available"):
        other.set_product([q, q])
    with pytest.raises(RuntimeError, match=r"gp_plan_set_kron \(as the data plan\) is not available on a spectral mixture plan"):
        _lib.check(lib.gp_plan_set_kron(other._h, q._h, 2))
    with pytest.raises(RuntimeError, match=r"\(as the data plan\) is not available on a spectral mixture plan"):
        _lib.check(lib.gp_plan_set_deriv(other._h, q._h))
    with pytest.raises(RuntimeError, match="Q d <= 32"):
        _plan(cuda_dev, _points(n, 4, 34), None, *_params(9, 4, 35))
    q.set_spectral(None)   # back to a plain RBF plan
    assert torch.isfinite(q.kmv(V)).all()
    for r in (p, q, other):
        r.close()


def _sm_model(train_x, train_y, Q, scaled=False, batch=None):
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, likelihoods, means, models

    d = 1 if train_x.dim() == 1 else train_x.size(-1)

    class SpectralMixtureGP(models.ExactGP):
        def __init__(self):
            bs = torch.Size([batch]) if batch else torch.Size()
            super().__init__(train_x, train_y, likelihoods.GaussianLikelihood(batch_shape=bs))
            self.mean_module = means.ConstantMean(batch_shape=bs)
            k = kernels.SpectralMixtureKernel(num_mixtures=Q, ard_num_dims=d, batch_shape=bs if batch else None)
            k.initialize_from_data(train_x.cpu(), train_y.cpu())   # the reference's draws, from torch's CPU generator
            self.covar_module = kernels.ScaleKernel(k) if scaled else k

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    return SpectralMixtureGP().to(train_x.device)


@pytest.mark.parametrize("cholesky_size", [800, 0])
def test_reference_tutorial_model(cuda_dev, cholesky_size):
    """The reference's test_spectral_mixture_gp_regression model: 15 points of sin(2 pi x) on [0, 1], Q = 4, seed 4,
    initialize_from_data, 300 Adam steps at lr 0.01; the mean extrapolated to [0, 1.5] within 0.02 on average.  N = 15 runs the
    dense branch (gp_krows and gp_bilinear_grad with n columns), and again the CG path with max_cholesky_size(0)."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    torch.manual_seed(4)
    train_x = torch.linspace(0, 1, 15)
    train_y = torch.sin(train_x * (2 * math.pi))
    test_x = torch.linspace(0, 1.5, 51)
    test_y = torch.sin(test_x * (2 * math.pi))
    train_x, train_y, test_x = train_x.to(cuda_dev), train_y.to(cuda_dev), test_x.to(cuda_dev)
    model = _sm_model(train_x, train_y, 4)
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    # on the CG path a 15-point problem is solved to 1e-4 with 16 trace probes, so that the stochastic MLL gradient stays close to
    # the dense one over the 300 steps (the training defaults, tolerance 1 and 10 probes, end at a mean error of 0.021)
    with settings.max_cholesky_size(cholesky_size), settings.cg_tolerance(1e-4), settings.num_trace_samples(16):
        for i in range(300):
            opt.zero_grad()
            loss = -mll(model(train_x), train_y)
            loss.backward()
            if i == 0:
                for name, prm in model.named_parameters():
                    assert prm.grad is not None, name
            opt.step()
        model.eval()
        with torch.no_grad():
            pred = model.likelihood(model(test_x)).mean
    mae = (test_y - pred.cpu()).abs().mean().item()
    assert mae < 0.02, mae


def test_long_series_trains_predicts_and_samples(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    torch.manual_seed(0)
    n = 20_000
    train_x = torch.arange(n, dtype=torch.float32) * 0.05
    train_y = (torch.sin(2 * math.pi * 0.13 * train_x) + 0.5 * torch.sin(2 * math.pi * 0.031 * train_x)
               + 0.1 * torch.randn(n))
    train_x, train_y = train_x.to(cuda_dev), train_y.to(cuda_dev)
    model = _sm_model(train_x, train_y, 4, scaled=True)
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=0.05)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = -mll(model(train_x), train_y)
        loss.backward()
        losses.append(loss.item())
        opt.step()
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    assert model.covar_module.base_kernel.raw_mixture_means.grad is not None
    model.eval()
    test_x = (n + torch.arange(200, dtype=torch.float32)).to(cuda_dev) * 0.05
    with torch.no_grad():
        f = model(test_x)
        assert f.mean.shape == (200,) and bool(torch.isfinite(f.mean).all()) and bool((f.variance > 0).all())
        with settings.fast_pred_var():
            f2 = model(test_x)
            assert rel(f2.mean, f.mean) < 1e-2 and bool(torch.isfinite(f2.variance).all())
        # CIQ samples of the lazy posterior covariance (LOVE: K** - U U^T on the test points' spectral plan)
        with settings.fast_pred_var(), settings.fast_pred_samples(), settings.ciq_samples(True):
            s = model(test_x).rsample(torch.Size([3]))
            assert s.shape == (3, 200) and bool(torch.isfinite(s).all())


def test_predictions_after_lazy_love_samples_are_unchanged(cuda_dev):
    """fast_pred_samples builds the lazy LOVE covariance K** - U U^T on the test points' spectral plan.  That plan must stay apart
    from the ordinary spectral operators over the same test points: exact and fast_pred_var predictions made after the samples
    equal the ones made before."""
    from gpytorch_b200 import settings

    torch.manual_seed(2)
    n, m = 2000, 150
    train_x = (torch.arange(n, dtype=torch.float32) * 0.05).to(cuda_dev)
    train_y = (torch.sin(2 * math.pi * 0.13 * train_x) + 0.1 * torch.randn(n, device=cuda_dev)).contiguous()
    model = _sm_model(train_x, train_y, 3, scaled=True)
    model.eval()
    test_x = ((n + torch.arange(m, dtype=torch.float32)) * 0.05).to(cuda_dev)
    with torch.no_grad():
        f0 = model(test_x)
        mean0, var0 = f0.mean.clone(), f0.variance.clone()
        with settings.fast_pred_var():
            fvar0 = model(test_x).variance.clone()
        for _ in range(3):
            with settings.fast_pred_var(), settings.fast_pred_samples(), settings.ciq_samples(True):
                s = model(test_x).rsample(torch.Size([2]))
                assert s.shape == (2, m) and bool(torch.isfinite(s).all())
            f1 = model(test_x)
            assert torch.allclose(f1.mean, mean0, rtol=1e-5, atol=1e-6)
            assert torch.allclose(f1.variance, var0, rtol=1e-5, atol=1e-6 * float(var0.abs().max()))
            with settings.fast_pred_var():
                fvar1 = model(test_x).variance
            assert torch.allclose(fvar1, fvar0, rtol=1e-5, atol=1e-6 * float(fvar0.abs().max()))


def test_batch_shape_model_trains(cuda_dev):
    import gpytorch_b200 as gp

    torch.manual_seed(1)
    n = 200
    x = torch.linspace(0, 4, n)
    train_x = torch.stack([x, x]).unsqueeze(-1)
    train_y = torch.stack([torch.sin(2 * math.pi * 0.7 * x), torch.cos(2 * math.pi * 1.3 * x)]) + 0.05 * torch.randn(2, n)
    train_x, train_y = train_x.to(cuda_dev), train_y.to(cuda_dev)
    model = _sm_model(train_x, train_y, 3, scaled=True, batch=2)
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=0.05)
    losses = []
    for _ in range(15):
        opt.zero_grad()
        loss = -mll(model(train_x), train_y).sum()
        loss.backward()
        losses.append(loss.item())
        opt.step()
    assert losses[-1] < losses[0]
    g = model.covar_module.base_kernel.raw_mixture_weights.grad
    assert g is not None and g.shape == (2, 3) and bool((g != 0).all())
