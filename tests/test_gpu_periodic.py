"""Periodic kernels on the device (run with -m gpu): ONE engine operator (gp_plan_set_periodic, csrc/periodic.cu) that runs as the
plain RBF plan over the embedding (cos, sin)(2 pi x / p) / sqrt(l).  Every comparison is against the fp64 oracle of
tests/periodic_oracle.py: K.V entry by entry within its derived bound on both backends (also at time stamps up to 1e5, where the
reference's fp32 formula is off by far more), the RBF plan over the embedded inputs, rows, the diagonal, pivots, the MLL, the
gradients, determinism, NaN inputs, refusals, and the public API (period recovery, prediction, a sum with an RBF kernel, CIQ
samples, lazy LOVE, a batch)."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

import kmv_oracle as ko  # noqa: E402
import periodic_oracle as po  # noqa: E402
from oracle import linalg as ol, mll as om  # noqa: E402

PATH = {"tcgen05": "tc", "simt": "simt"}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _params(d, ard, seed):
    """fp32 lengthscales and periods, 1 or d of each."""
    g = torch.Generator().manual_seed(seed)
    k = d if ard else 1
    return torch.rand(k, generator=g) * 1.2 + 0.4, torch.rand(k, generator=g) * 2.0 + 0.5


def _points(n, d, seed, scale=8.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g) * scale - scale / 2


def _plan(dev, x1, x2, ls, per, S=1.0, noise=0.0, backend="auto"):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)
    return p.set_periodic(per).set_hypers("rbf", ls.tolist(), S, noise)


def _check_kmv(dev, x1, x2, ls, per, S, V, backend):
    p = _plan(dev, x1, x2, ls, per, S, backend=backend)
    info = p.info()
    d = x1.size(1)
    assert info["backend"] == backend
    if backend == "tcgen05":
        assert info["kpad"] == (6 * d + 4 + 7) // 8 * 8
    out = p.kmv(V.to(dev)).double().cpu()
    n2 = (x1 if x2 is None else x2).size(0)
    geo = ko.geometry(x1.size(0), n2, 2 * d, backend, info["n_sm"])
    assert geo["nsplit"] == info["nsplit"]
    ref = po.kernel(x1, x1 if x2 is None else x2, ls, per, S) @ V.double()
    bnd = po.kmv_bound(x1, x1 if x2 is None else x2, ls, per, V, S, PATH[backend], geo["nsplit"], geo["T"], same=x2 is None)
    err = (out - ref).abs()
    assert bool(torch.isfinite(out).all()) and bool((err <= bnd).all()), (backend, float((err / bnd).max()))
    p.close()
    return out, bnd


@pytest.mark.parametrize("d", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("ard", [False, True])
def test_kmv_within_bound_on_both_backends(cuda_dev, d, ard):
    ls, per = _params(d, ard, 10 * d + ard)
    x1, x2 = _points(333, d, d), _points(201, d, d + 50)
    V = torch.randn(333, 5, generator=torch.Generator().manual_seed(d))
    for backend in ("tcgen05", "simt"):
        _check_kmv(cuda_dev, x1, None, ls, per, 1.3, V, backend)            # square, n not a multiple of the tile, t < 16
        _check_kmv(cuda_dev, x1, x2, ls, per, 0.7, V[:201], backend)      # cross


def test_large_time_stamps(cuda_dev):
    """x = 0 .. 99 999 (every 41st) with p = 1 / 0.49: the engine stays within the bound; the reference's fp32 formula
    (x / (p / pi), then sin^2 of the distance) on the same fp32 inputs does not."""
    x = torch.cat([torch.arange(0, 100000, 41, dtype=torch.float32), torch.tensor([99999.0])]).unsqueeze(1)
    per = torch.tensor([1.0 / 0.49], dtype=torch.float32)
    ls = torch.tensor([0.8])
    V = torch.randn(x.size(0), 4, generator=torch.Generator().manual_seed(5))
    _, bnd = _check_kmv(cuda_dev, x, None, ls, per, 1.0, V, "tcgen05")
    xd = x.to(cuda_dev)
    x_ = xd.div(per.to(cuda_dev) / math.pi)
    k32 = torch.exp(-2.0 * torch.sin((x_ - x_.T).abs()) ** 2 / ls.to(cuda_dev))
    ref = po.kernel(x, x, ls, per, 1.0) @ V.double()
    err32 = ((k32 @ V.to(cuda_dev)).double().cpu() - ref).abs()
    assert bool((err32 > bnd).any()) and float(err32.max()) > 10 * float(bnd.max())


def test_matches_rbf_plan_over_embedded_inputs(cuda_dev):
    from gpytorch_b200.engine import Plan

    d = 3
    ls, per = _params(d, True, 7)
    x = _points(500, d, 8, scale=200.0)
    V = torch.randn(500, 6, generator=torch.Generator().manual_seed(9))
    out, bnd = _check_kmv(cuda_dev, x, None, ls, per, 1.0, V, "tcgen05")
    u = po.embed(x, ls, per).float()
    pr = Plan(u.to(cuda_dev)).set_hypers("rbf", 1.0, 1.0, 0.0)
    o2 = pr.kmv(V.to(cuda_dev)).double().cpu()
    geo = ko.geometry(500, 500, 2 * d, "auto", pr.info()["n_sm"])
    b2 = ko.bound("rbf", u, None, 1.0, 1.0, 0.0, V, "tc", geo["nsplit"], geo["T"], same=True)
    assert bool(((out - o2).abs() <= bnd + b2 + 1e-6 * (po.kernel(x, x, ls, per) @ V.double().abs())).all())
    pr.close()


def test_rows_diag_and_pivots(cuda_dev):
    n, d, S = 700, 2, 0.8
    ls, per = _params(d, True, 11)
    x = _points(n, d, 11)
    K = po.kernel(x, x, ls, per, S)
    p = _plan(cuda_dev, x, None, ls, per, S, noise=0.1)
    idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
    rows = p.rows(idx).double().cpu()
    assert float((rows - K[idx]).abs().max()) <= 2e-5 * S
    assert torch.equal(p.diag().cpu(), torch.full((n,), S, dtype=torch.float32))
    # pivots: the greedy fp64 pivoting on well separated candidates (the gap between the two best is asserted)
    g = torch.Generator().manual_seed(33)
    xp = torch.rand(48, 1, generator=g) * 3.0
    lp, pp_ = torch.tensor([0.5]), torch.tensor([1.7])
    Kp = po.kernel(xp, xp, lp, pp_, S)
    diag32 = torch.full((48,), S, dtype=torch.float64)
    rank = 8
    L, piv_o = ol.pivoted_cholesky(diag32, lambda i: Kp[i], rank)
    pp = _plan(cuda_dev, xp, None, lp, pp_, S, noise=0.1)
    lt, piv, st = pp.pivoted_cholesky(rank, 1e-6)
    assert st == 0
    m = lt.size(0)
    assert torch.equal(piv.cpu()[:min(m, 4)], piv_o[:min(m, 4)])
    # cross plan: rows and the diagonal of K(x1, x2) with equal sizes
    x2 = _points(n, d, 13)
    pc = _plan(cuda_dev, x, x2, ls, per, S)
    Kc = po.kernel(x, x2, ls, per, S)
    assert float((pc.rows(idx).double().cpu() - Kc[idx]).abs().max()) <= 2e-5 * S
    assert float((pc.diag().double().cpu() - Kc.diagonal()).abs().max()) <= 2e-5 * S
    for q in (p, pp, pc):
        q.close()


def test_mll_on_the_cg_path_matches_oracle(cuda_dev):
    n, d, rank = 2500, 1, 30
    x, y = om.synthetic_problem(n, d, 4, torch.float32)
    x = x * 10
    ls, per = torch.tensor([0.9]), torch.tensor([1.7])
    S, noise = 1.0, 1.0
    K = po.kernel(x, x, ls, per, S)
    p = _plan(cuda_dev, x, None, ls, per, S, noise=noise)
    pn = om.make_probe_noise(n, rank, 10, 7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, S, noise, tuple(a.double() for a in pn), precond_size=rank, K=K)
    res, _ = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000)
    assert abs(res.mll - o64.mll) <= 1e-4 * max(1.0, abs(o64.mll)), (res.mll, o64.mll)
    p.close()


@pytest.mark.parametrize("d,ard,S", [(1, False, 1.0), (2, True, 0.6), (3, False, 1.4), (8, True, 1.0), (12, True, 0.9)])
def test_bilinear_grad_matches_fp64_autograd_and_repeats_bit_for_bit(cuda_dev, d, ard, S):
    n, m, s = 500, 430, 13
    x1, x2 = _points(n, d, 21), _points(m, d, 22)
    ls, per = _params(d, ard, 23 + d)
    g = torch.Generator().manual_seed(24)
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, x1, x2, ls, per, S)
    gl, gs = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    assert p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev)) == (gl, gs)
    W = L.double() @ R.double().T
    rl, rp, rs = po.grads(x1, x2, ls, per, W, S)
    ref = torch.cat([rl, rp])
    got = torch.tensor(gl, dtype=torch.float64)
    assert got.shape == ref.shape
    assert torch.allclose(got, ref, rtol=2e-4, atol=2e-4 * ref.abs().max().item()), (got, ref)
    assert abs(gs - rs.item()) <= 2e-4 * max(abs(rs.item()), 1e-3 * ref.abs().max().item())
    V = torch.randn(m, 7, generator=g).to(cuda_dev)
    assert torch.equal(p.kmv(V), p.kmv(V))
    p.close()


def test_period_gradient_at_large_time_stamps(cuda_dev):
    """dF/dp from tau directly: at x ~ 1e5 it still matches fp64 autograd (the chain rule through the embedding would not)."""
    x = (1.0e5 + torch.arange(0, 600, dtype=torch.float32) * 0.37).unsqueeze(1)
    ls, per = torch.tensor([0.7]), torch.tensor([2.3])
    g = torch.Generator().manual_seed(3)
    L, R = torch.randn(600, 4, generator=g), torch.randn(600, 4, generator=g)
    p = _plan(cuda_dev, x, None, ls, per, 1.0)
    gl, _ = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    rl, rp, _ = po.grads(x, x, ls, per, L.double() @ R.double().T)
    ref = torch.cat([rl, rp])
    assert torch.allclose(torch.tensor(gl, dtype=torch.float64), ref, rtol=1e-3, atol=1e-3 * ref.abs().max().item())
    p.close()


def test_nan_inputs_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    n, d = 300, 2
    ls, per = _params(d, True, 31)
    x = _points(n, d, 31)
    x[5, 1] = float("nan")
    p = _plan(cuda_dev, x, None, ls, per)
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(p.kmv(V).isnan().all())
    gl, gs = p.bilinear_grad(V, V)
    assert all(math.isnan(t) for t in gl + [gs])
    q = _plan(cuda_dev, _points(n, d, 32), None, ls, per)
    lib = q.lib
    other = Plan(_points(n, d, 33).to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    tasks = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    for call, fn in [("gp_plan_set_tasks", lambda: q.set_tasks(tasks, None, 2)),
                     ("gp_plan_set_sum", lambda: q.set_sum([other])),
                     ("gp_plan_set_product", lambda: q.set_product([other, other])),
                     ("gp_plan_set_ski", lambda: q.set_ski([16] * d, [-4.0] * d, [0.5] * d)),
                     ("gp_plan_set_additive", lambda: q.set_additive(1, [1.0] * d)),
                     ("gp_plan_set_spectral", lambda: q.set_spectral([1.0], [[0.1] * d], [[0.2] * d])),
                     ("gp_plan_set_kron", lambda: _lib.check(lib.gp_plan_set_kron(q._h, other._h, 2))),
                     ("gp_plan_set_deriv", lambda: _lib.check(lib.gp_plan_set_deriv(q._h, other._h)))]:
        with pytest.raises(RuntimeError, match=f"{call} is not available on a periodic plan"):
            fn()
    with pytest.raises(RuntimeError, match="gp_kmv_input_grad is not available on a periodic plan"):
        q.kmv_input_grad(V, V)
    with pytest.raises(RuntimeError, match="gp_kdense_input_grad is not available on a periodic plan"):
        q.dense_input_grad(torch.zeros(n, n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="a periodic plan as a factor is not available"):
        other.set_product([q, q])
    with pytest.raises(RuntimeError, match=r"gp_plan_set_kron \(as the data plan\) is not available on a periodic plan"):
        _lib.check(lib.gp_plan_set_kron(other._h, q._h, 2))
    with pytest.raises(RuntimeError, match=r"\(as the data plan\) is not available on a periodic plan"):
        _lib.check(lib.gp_plan_set_deriv(other._h, q._h))
    # a periodic plan is a valid kernel-sum term: K = K_per + K_rbf
    from oracle import kernels as ok

    xs = _points(n, d, 32)
    rb = Plan(xs.to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    s = Plan(xs.to(cuda_dev)).set_hypers("rbf", [1.0], 1.0, 0.0).set_sum([q, rb])
    ref = (po.kernel(xs, xs, ls, per) + ok.kernel_matrix("rbf", xs.double(), xs.double(), 0.5, 1.0, True)) @ V.double().cpu()
    assert rel(s.kmv(V), ref) < 1e-5
    q.set_periodic(None)   # back to a plain RBF plan
    assert torch.isfinite(q.kmv(V)).all()
    for r in (s, rb, p, q, other):
        r.close()


def _model(train_x, train_y, kernel, noise=None):
    import gpytorch_b200 as gp
    from gpytorch_b200 import likelihoods, means, models

    class PeriodicGP(models.ExactGP):
        def __init__(self):
            bs = train_x.shape[:-2] if train_x.dim() == 3 else torch.Size()
            super().__init__(train_x, train_y, likelihoods.GaussianLikelihood(batch_shape=bs))
            self.mean_module = means.ConstantMean(batch_shape=bs)
            self.covar_module = kernel

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    m = PeriodicGP().to(train_x.device)
    if noise is not None:
        m.likelihood.noise = noise
    return m


def _train(model, x, y, steps, lr):
    import gpytorch_b200 as gp

    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=lr)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = -mll(model(x), y).sum()
        loss.backward()
        losses.append(loss.item())
        opt.step()
    return losses


def test_recovers_the_period_and_predicts_the_dense_posterior(cuda_dev):
    from gpytorch_b200 import kernels

    torch.manual_seed(0)
    n, p0 = 1200, 1.0
    x = torch.rand(n) * 12.0
    y = torch.sin(2 * math.pi * x / p0) + 0.1 * torch.randn(n)
    k = kernels.ScaleKernel(kernels.PeriodicKernel())
    k.base_kernel.period_length = 1.015
    k.base_kernel.lengthscale = 1.0
    k.outputscale = 1.0
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model = _model(xd, yd, k, noise=0.02)
    losses = _train(model, xd, yd, 60, 0.02)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    pl = float(k.base_kernel.period_length)
    assert abs(pl - p0) <= 0.02 * p0, pl
    model.eval()
    tx = torch.linspace(12.0, 14.0, 101)
    with torch.no_grad():
        f = model(tx.to(cuda_dev))
    ls, per, S = k.base_kernel.lengthscale.detach().cpu().reshape(-1), k.base_kernel.period_length.detach().cpu().reshape(-1), \
        float(k.outputscale)
    nz, c = float(model.likelihood.noise), float(model.mean_module.constant)
    Kxx = po.kernel(x[:, None], x[:, None], ls.float(), per.float(), S) + nz * torch.eye(n, dtype=torch.float64)
    Ksx = po.kernel(tx[:, None], x[:, None], ls.float(), per.float(), S)
    mean = Ksx @ torch.linalg.solve(Kxx, y.double() - c) + c
    assert (f.mean.double().cpu() - mean).abs().max().item() < 2e-2, (f.mean.cpu() - mean).abs().max()
    assert rel(f.mean, mean) < 1e-2


def test_periodic_plus_rbf_sum_trains_and_predicts(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(1)
    n = 1500
    x = torch.linspace(0, 10, n)
    y = torch.sin(2 * math.pi * x / 1.3) + 0.3 * x + 0.1 * torch.randn(n)
    k = kernels.ScaleKernel(kernels.PeriodicKernel()) + kernels.ScaleKernel(kernels.RBFKernel())
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model = _model(xd, yd, k)
    with settings.max_cholesky_size(0):
        losses = _train(model, xd, yd, 15, 0.05)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    assert k.kernels[0].base_kernel.raw_period_length.grad is not None
    model.eval()
    tx = torch.linspace(10, 11, 50).to(cuda_dev)
    with torch.no_grad(), settings.max_cholesky_size(0):
        f = model(tx)
        assert bool(torch.isfinite(f.mean).all()) and bool((f.variance > 0).all())
    # ScaleKernel around the sum folds its scale into both terms
    ks = kernels.ScaleKernel(kernels.PeriodicKernel() + kernels.RBFKernel()).to(cuda_dev)
    op = ks(xd)
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(torch.isfinite(op @ V).all())


def test_ciq_samples_have_the_kernel_covariance(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(3)
    n, N = 40, 20000
    x = torch.linspace(0, 3, n).to(cuda_dev)
    k = kernels.ScaleKernel(kernels.PeriodicKernel())
    k.base_kernel.period_length = 1.1
    k.base_kernel.lengthscale = 0.7
    k.outputscale = 1.5
    k = k.to(cuda_dev)
    with torch.no_grad(), settings.ciq_samples(True), settings.max_cholesky_size(0):
        mvn = gp.distributions.MultivariateNormal(torch.zeros(n, device=cuda_dev), k(x).add_jitter(1e-4))
        s = mvn.rsample(torch.Size([N])).double().cpu()
    emp = s.T @ s / N
    K = po.kernel(x[:, None].cpu(), x[:, None].cpu(), torch.tensor([0.7]), torch.tensor([1.1]), 1.5)
    assert (emp - K).abs().max().item() < 0.1, (emp - K).abs().max()


def test_predictions_after_lazy_love_samples_are_unchanged(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(2)
    n, m = 2000, 150
    train_x = (torch.arange(n, dtype=torch.float32) * 0.05).to(cuda_dev)
    train_y = (torch.sin(2 * math.pi * train_x / 1.7) + 0.1 * torch.randn(n, device=cuda_dev)).contiguous()
    k = kernels.ScaleKernel(kernels.PeriodicKernel())
    k.base_kernel.period_length = 1.7
    model = _model(train_x, train_y, k, noise=0.01)
    model.eval()
    test_x = ((n + torch.arange(m, dtype=torch.float32)) * 0.05).to(cuda_dev)
    with torch.no_grad():
        f0 = model(test_x)
        mean0, var0 = f0.mean.clone(), f0.variance.clone()
        with settings.fast_pred_var():
            fvar0 = model(test_x).variance.clone()
        for _ in range(2):
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
    from gpytorch_b200 import kernels

    torch.manual_seed(1)
    n = 200
    x = torch.linspace(0, 4, n)
    train_x = torch.stack([x, x]).unsqueeze(-1)
    train_y = torch.stack([torch.sin(2 * math.pi * 0.7 * x), torch.cos(2 * math.pi * 1.3 * x)]) + 0.05 * torch.randn(2, n)
    train_x, train_y = train_x.to(cuda_dev), train_y.to(cuda_dev)
    k = kernels.ScaleKernel(kernels.PeriodicKernel(batch_shape=torch.Size([2])))
    model = _model(train_x, train_y, k)
    losses = _train(model, train_x, train_y, 15, 0.05)
    assert losses[-1] < losses[0]
    g = k.base_kernel.raw_period_length.grad
    assert g is not None and g.shape == (2, 1, 1) and bool((g != 0).all())
