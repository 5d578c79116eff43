"""Rational quadratic kernels on the device (run with -m gpu): plans of kind GP_RQ (gp_plan_set_hypers_rq) on the tensor-core and
CUDA-core K.V.  Every comparison is against the fp64 oracle of tests/rq_oracle.py: K.V entry by entry within its derived bound on
both backends over an alpha sweep up to 1e4 and at the ring edges, rows, the diagonal, pivots, the MLL, the gradients (with
determinism), input gradients, NaN inputs, refusals, and the public API (prediction against the dense posterior, sums with RBF and
periodic terms, CIQ samples, lazy LOVE, a batch)."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

import kmv_oracle as ko  # noqa: E402
import periodic_oracle as po  # noqa: E402
import rq_oracle as ro  # noqa: E402
from oracle import kernels as ok, linalg as ol, mll as om  # noqa: E402

PATH = {"tcgen05": "tc", "simt": "simt"}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _ls(d, ard, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(d if ard else 1, generator=g) * 1.2 + 0.4


def _points(n, d, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g) * scale - scale / 2


def _plan(dev, x1, x2, ls, alpha, S=1.0, noise=0.0, backend="auto"):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)
    return p.set_hypers_rq(ls.tolist(), alpha, S, noise)


def _check_kmv(dev, x1, x2, ls, alpha, S, V, backend):
    p = _plan(dev, x1, x2, ls, alpha, S, backend=backend)
    info = p.info()
    assert info["backend"] == backend
    out = p.kmv(V.to(dev)).double().cpu()
    xc = x1 if x2 is None else x2
    geo = ko.geometry(x1.size(0), xc.size(0), x1.size(1), backend, info["n_sm"])
    assert geo["nsplit"] == info["nsplit"]
    a32 = float(torch.tensor(alpha, dtype=torch.float32))
    ref = ro.kernel(x1, xc, ls, a32, S) @ V.double()
    bnd = ro.kmv_bound(x1, xc, ls, a32, V, S, PATH[backend], geo["nsplit"], geo["T"], same=x2 is None)
    err = (out - ref).abs()
    assert bool(torch.isfinite(out).all()) and bool((err <= bnd).all()), (backend, alpha, float((err / bnd).max()))
    p.close()


@pytest.mark.parametrize("d,ard", [(1, False), (2, True), (3, False), (8, True), (16, False)])
def test_kmv_within_bound_on_both_backends(cuda_dev, d, ard):
    ls = _ls(d, ard, d)
    g = torch.Generator().manual_seed(100 + d)
    for alpha in (0.05, 0.5, 2.0, 50.0, 1e4):
        x1, x2 = _points(700, d, d + 1), _points(530, d, d + 2)
        V = torch.randn(530, 5, generator=g)
        for backend in ("tcgen05", "simt"):
            _check_kmv(cuda_dev, x1, x2, ls, alpha, 0.8, V, backend)
        _check_kmv(cuda_dev, x1, None, ls, alpha, 1.2, torch.randn(700, 3, generator=g), "tcgen05")


def test_kmv_at_the_ring_split_and_diagonal_tile_edges(cuda_dev):
    g = torch.Generator().manual_seed(7)
    for d, T, n1, n2 in ko.ring_cases()[:4]:
        ls = _ls(d, True, d)
        x1, x2 = _points(n1, d, 3), _points(n2, d, 4)
        _check_kmv(cuda_dev, x1, x2, ls, 3.0, 1.0, torch.randn(n2, 4, generator=g), "tcgen05")
    for n in (63, 64, 65, 129, 257):
        x = _points(n, 2, n)
        _check_kmv(cuda_dev, x, None, _ls(2, False, 1), 1e4, 1.0, torch.randn(n, 2, generator=g), "tcgen05")


def test_rows_diag_and_pivots(cuda_dev):
    n, d, S, alpha = 700, 2, 0.8, 1.7
    ls = _ls(d, True, 11)
    x = _points(n, d, 11)
    K = ro.kernel(x, x, ls, alpha, S)
    p = _plan(cuda_dev, x, None, ls, alpha, S, noise=0.1)
    idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
    assert float((p.rows(idx).double().cpu() - K[idx]).abs().max()) <= 2e-5 * S
    assert torch.equal(p.diag().cpu(), torch.full((n,), S, dtype=torch.float32))
    g = torch.Generator().manual_seed(33)
    xp = torch.rand(48, 1, generator=g) * 3.0
    lp = torch.tensor([0.5])
    Kp = ro.kernel(xp, xp, lp, alpha, S)
    L, piv_o = ol.pivoted_cholesky(torch.full((48,), S, dtype=torch.float64), lambda i: Kp[i], 8)
    pp = _plan(cuda_dev, xp, None, lp, alpha, S, noise=0.1)
    lt, piv, st = pp.pivoted_cholesky(8, 1e-6)
    assert st == 0
    m = lt.size(0)
    assert torch.equal(piv.cpu()[:min(m, 4)], piv_o[:min(m, 4)])
    x2 = _points(n, d, 13)
    pc = _plan(cuda_dev, x, x2, ls, alpha, S)
    Kc = ro.kernel(x, x2, ls, alpha, S)
    assert float((pc.rows(idx).double().cpu() - Kc[idx]).abs().max()) <= 2e-5 * S
    assert float((pc.diag().double().cpu() - Kc.diagonal()).abs().max()) <= 2e-5 * S
    for q in (p, pp, pc):
        q.close()


def test_mll_on_the_cg_path_matches_oracle(cuda_dev):
    n, d, rank = 2500, 2, 30
    x, y = om.synthetic_problem(n, d, 4, torch.float32)
    ls, alpha, S, noise = torch.tensor([0.9]), 2.0, 1.0, 0.5
    K = ro.kernel(x, x, ls, alpha, S)
    p = _plan(cuda_dev, x, None, ls, alpha, S, noise=noise)
    pn = om.make_probe_noise(n, rank, 10, 7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, S, noise, tuple(a.double() for a in pn), precond_size=rank, K=K)
    res, _ = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000)
    assert abs(res.mll - o64.mll) <= 1e-4 * max(1.0, abs(o64.mll)), (res.mll, o64.mll)
    p.close()


@pytest.mark.parametrize("d,ard,S,alpha,backend", [(1, False, 1.0, 0.5, "tcgen05"), (3, False, 1.4, 20.0, "tcgen05"),
                                                   (2, True, 0.6, 2.0, "auto"), (8, True, 1.0, 0.3, "auto"),
                                                   (2, False, 0.9, 3.0, "simt")])
def test_bilinear_grad_matches_fp64_autograd_and_repeats_bit_for_bit(cuda_dev, d, ard, S, alpha, backend):
    n, m, s = 500, 430, 13
    x1, x2 = _points(n, d, 21), _points(m, d, 22)
    ls = _ls(d, ard, 23 + d)
    g = torch.Generator().manual_seed(24)
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, x1, x2, ls, alpha, S, backend=backend)
    gl, gs = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    assert len(gl) == ls.numel() + 1
    assert p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev)) == (gl, gs)
    W = L.double() @ R.double().T
    a32 = float(torch.tensor(alpha, dtype=torch.float32))
    rl, ra, rs = ro.grads(x1, x2, ls, a32, W, S)
    ref = torch.cat([rl.reshape(-1), ra.reshape(1)])
    got = torch.tensor(gl, dtype=torch.float64)
    assert torch.allclose(got, ref, rtol=2e-4, atol=2e-4 * ref.abs().max().item()), (got, ref)
    assert abs(gs - rs.item()) <= 2e-4 * max(abs(rs.item()), 1e-3 * ref.abs().max().item())
    p.close()


def test_alpha_gradient_dominated_by_small_t(cuda_dev):
    """Close points at alpha = 1e3: every t is below 1e-4, where phi is the series (a plain difference would cancel)."""
    n, d, s, alpha = 600, 2, 4, 1e3
    x1 = _points(n, d, 41, scale=0.05)
    ls = torch.tensor([0.8])
    g = torch.Generator().manual_seed(42)
    L, R = torch.rand(n, s, generator=g), torch.rand(n, s, generator=g)   # positive weights: the total does not cancel
    for backend in ("tcgen05", "simt"):
        p = _plan(cuda_dev, x1, x1.clone(), ls, alpha, 1.0, backend=backend)
        gl, _ = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
        _, ra, _ = ro.grads(x1, x1.clone(), ls, alpha, L.double() @ R.double().T)
        assert abs(gl[1] - ra.item()) <= 2e-4 * abs(ra.item()), (backend, gl[1], ra.item())
        p.close()


def test_input_gradients_match_fp64_autograd(cuda_dev):
    n, m, d, s, alpha, S = 400, 300, 3, 5, 1.5, 1.3
    x1, x2 = _points(n, d, 51), _points(m, d, 52)
    ls = _ls(d, True, 53)
    g = torch.Generator().manual_seed(54)
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, x1, x2, ls, alpha, S)
    d1, d2 = p.kmv_input_grad(L.to(cuda_dev), R.to(cuda_dev), True, True)
    a = x1.double().requires_grad_(True)
    b = x2.double().requires_grad_(True)
    F = (L.double() * (ro.kernel(a, b, ls.double(), alpha, S) @ R.double())).sum()
    ga, gb = torch.autograd.grad(F, (a, b))
    assert rel(d1, ga) < 1e-4 and rel(d2, gb) < 1e-4
    p.close()


def test_dkl_and_posterior_input_gradients(cuda_dev):
    """An MLL backward through learned features and the posterior mean / variance gradients at test points, against dense fp64."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels

    torch.manual_seed(5)
    n, d = 300, 2
    x = torch.rand(n, d) * 2 - 1
    y = torch.sin(3 * x[:, 0]) + 0.5 * x[:, 1] + 0.05 * torch.randn(n)
    k = kernels.ScaleKernel(kernels.RQKernel())
    k.base_kernel.alpha = 1.5
    k.base_kernel.lengthscale = 0.6
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    W = torch.randn(d, d).to(cuda_dev).requires_grad_(True)
    feats = xd @ W
    model = _model(feats.detach(), yd, k, noise=0.05)
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    loss = -mll(model(feats), yd)   # n <= max_cholesky_size: the dense branch, exact (no probe noise in the log-det gradient)
    loss.backward()
    assert W.grad is not None and bool(torch.isfinite(W.grad).all())
    # dense fp64 check of dLoss/dW
    Wd = W.detach().double().cpu().requires_grad_(True)
    f = x.double() @ Wd
    ls, al, S = 0.6, float(k.base_kernel.alpha), float(k.outputscale)
    nz, c = float(model.likelihood.noise), float(model.mean_module.constant)
    K = S * torch.pow(1 + ((f[:, None] - f[None]) ** 2).sum(-1) / (2 * al * ls * ls), -al) + nz * torch.eye(n, dtype=torch.float64)
    r = y.double() - c
    nll = 0.5 * (r @ torch.linalg.solve(K, r) + torch.logdet(K) + n * math.log(2 * math.pi)) / n
    (gW,) = torch.autograd.grad(nll, Wd)
    assert rel(W.grad, gW) < 2e-2, (W.grad.cpu(), gW)
    # posterior mean / variance gradients with respect to the test inputs
    model.set_train_data(feats.detach(), yd, strict=False)
    model.eval()
    tx = (torch.rand(20, d) * 2 - 1).to(cuda_dev).requires_grad_(True)
    out = model(tx)
    (out.mean.sum() + out.variance.sum()).backward()
    ftr = feats.detach().double().cpu()
    txd = tx.detach().double().cpu().requires_grad_(True)
    kern = lambda a, b: S * torch.pow(1 + ((a[:, None] - b[None]) ** 2).sum(-1) / (2 * al * ls * ls), -al)  # noqa: E731
    Kxx = kern(ftr, ftr) + nz * torch.eye(n, dtype=torch.float64)
    Ksx = kern(txd, ftr)
    mean = Ksx @ torch.linalg.solve(Kxx, r) + c
    var = S - (Ksx * torch.linalg.solve(Kxx, Ksx.T).T).sum(-1)
    (gt,) = torch.autograd.grad(mean.sum() + var.sum(), txd)
    assert rel(tx.grad, gt) < 2e-2, (tx.grad.cpu(), gt)


def test_nan_inputs_alpha_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    n, d = 300, 2
    ls = _ls(d, True, 31)
    x = _points(n, d, 31)
    x[5, 1] = float("nan")
    p = _plan(cuda_dev, x, None, ls, 2.0)
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(p.kmv(V).isnan().all())
    gl, gs = p.bilinear_grad(V, V)
    assert len(gl) == 3 and all(math.isnan(t) for t in gl + [gs])
    q = _plan(cuda_dev, _points(n, d, 32), None, ls, 2.0)
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(RuntimeError, match="alpha"):
            q.set_hypers_rq(ls.tolist(), bad, 1.0, 0.0)
    assert q.alpha == 2.0   # all or nothing: the plan kept its alpha
    with pytest.raises(RuntimeError, match="gp_plan_set_hypers_rq"):
        q.set_hypers("rq", ls.tolist(), 1.0, 0.0)
    lib = q.lib
    other = Plan(_points(n, d, 33).to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    tasks = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    for call, fn in [("gp_plan_set_tasks", lambda: q.set_tasks(tasks, None, 2)),
                     ("gp_plan_set_product", lambda: q.set_product([other, other])),
                     ("gp_plan_set_ski", lambda: q.set_ski([16] * d, [-4.0] * d, [0.5] * d)),
                     ("gp_plan_set_additive", lambda: q.set_additive(1, [1.0] * d)),
                     ("gp_plan_set_spectral", lambda: q.set_spectral([1.0], [[0.1] * d], [[0.2] * d])),
                     ("gp_plan_set_periodic", lambda: q.set_periodic([1.0])),
                     ("gp_plan_set_kron", lambda: _lib.check(lib.gp_plan_set_kron(q._h, other._h, 2))),
                     ("gp_plan_set_deriv", lambda: _lib.check(lib.gp_plan_set_deriv(q._h, other._h)))]:
        with pytest.raises(RuntimeError, match=f"{call} is not available on a rational quadratic plan"):
            fn()
    with pytest.raises(RuntimeError, match="a rational quadratic plan as a factor is not available"):
        other.set_product([q, q])
    with pytest.raises(RuntimeError, match=r"gp_plan_set_kron \(as the data plan\) is not available on a rational quadratic plan"):
        _lib.check(lib.gp_plan_set_kron(other._h, q._h, 2))
    with pytest.raises(RuntimeError, match=r"\(as the data plan\) is not available on a rational quadratic plan"):
        _lib.check(lib.gp_plan_set_deriv(other._h, q._h))
    # an RQ plan is a kernel-sum term: K = K_rq + K_rbf, on the tensor-core path of the sum
    xs = _points(n, d, 32)
    rb = Plan(xs.to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    s = Plan(xs.to(cuda_dev)).set_hypers("rbf", [1.0], 1.0, 0.0).set_sum([q, rb])
    ref = (ro.kernel(xs, xs, ls, 2.0) + ok.kernel_matrix("rbf", xs.double(), xs.double(), 0.5, 1.0, True)) @ V.double().cpu()
    assert rel(s.kmv(V), ref) < 1e-5
    q.set_hypers("rbf", ls.tolist(), 1.0, 0.0)   # back to a plain RBF plan
    assert q.bilinear_grad(V, V)[0].__len__() == d
    for r in (s, rb, p, q, other):
        r.close()


def _model(train_x, train_y, kernel, noise=None):
    import gpytorch_b200 as gp
    from gpytorch_b200 import likelihoods, means, models

    class RQGP(models.ExactGP):
        def __init__(self):
            bs = train_x.shape[:-2] if train_x.dim() == 3 else torch.Size()
            super().__init__(train_x, train_y, likelihoods.GaussianLikelihood(batch_shape=bs))
            self.mean_module = means.ConstantMean(batch_shape=bs)
            self.covar_module = kernel

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    m = RQGP().to(train_x.device)
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


def test_fitted_model_predicts_the_dense_posterior(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(0)
    n, alpha0 = 1500, 0.8
    x = torch.rand(n) * 10.0
    K0 = ro.kernel(x[:, None], x[:, None], torch.tensor([0.7]), alpha0) + 1e-6 * torch.eye(n, dtype=torch.float64)
    y = (torch.linalg.cholesky(K0) @ torch.randn(n, dtype=torch.float64)).float() + 0.1 * torch.randn(n)
    k = kernels.ScaleKernel(kernels.RQKernel())
    k.base_kernel.alpha, k.base_kernel.lengthscale, k.outputscale = 1.0, 0.6, 1.0
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model = _model(xd, yd, k, noise=0.02)
    with settings.max_cholesky_size(0):
        losses = _train(model, xd, yd, 30, 0.05)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    assert k.base_kernel.raw_alpha.grad is not None
    model.eval()
    tx = torch.linspace(0.0, 10.0, 101)
    with torch.no_grad(), settings.max_cholesky_size(0):
        f = model(tx.to(cuda_dev))
    ls, al, S = float(k.base_kernel.lengthscale), float(k.base_kernel.alpha), float(k.outputscale)
    nz, c = float(model.likelihood.noise), float(model.mean_module.constant)
    Kxx = ro.kernel(x[:, None], x[:, None], ls, al, S) + nz * torch.eye(n, dtype=torch.float64)
    Ksx = ro.kernel(tx[:, None], x[:, None], ls, al, S)
    mean = Ksx @ torch.linalg.solve(Kxx, y.double() - c) + c
    assert rel(f.mean, mean) < 1e-2, rel(f.mean, mean)
    with torch.no_grad():   # the dense branch (N <= max_cholesky_size) runs through gp_krows
        fd = model(tx.to(cuda_dev))
    assert rel(fd.mean, mean) < 1e-2, rel(fd.mean, mean)


def test_composite_sums_train_and_predict(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(1)
    n = 1500
    x = torch.linspace(0, 10, n)
    y = torch.sin(2 * math.pi * x / 1.3) + 0.3 * x + 0.2 * torch.sin(7 * x) + 0.1 * torch.randn(n)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    for k in (kernels.ScaleKernel(kernels.RBFKernel()) + kernels.ScaleKernel(kernels.RQKernel()),
              kernels.ScaleKernel(kernels.RBFKernel()) + kernels.ScaleKernel(kernels.PeriodicKernel())
              + kernels.ScaleKernel(kernels.RQKernel())):
        model = _model(xd, yd, k)
        with settings.max_cholesky_size(0):
            losses = _train(model, xd, yd, 12, 0.05)
        assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
        assert k.kernels[-1].base_kernel.raw_alpha.grad is not None
        model.eval()
        tx = torch.linspace(10, 11, 50).to(cuda_dev)
        with torch.no_grad(), settings.max_cholesky_size(0):
            f = model(tx)
            assert bool(torch.isfinite(f.mean).all()) and bool((f.variance > 0).all())


def test_ciq_samples_have_the_kernel_covariance(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(3)
    n, N = 40, 20000
    x = torch.linspace(0, 3, n).to(cuda_dev)
    k = kernels.ScaleKernel(kernels.RQKernel())
    k.base_kernel.alpha, k.base_kernel.lengthscale, k.outputscale = 0.7, 0.5, 1.5
    k = k.to(cuda_dev)
    with torch.no_grad(), settings.ciq_samples(True), settings.max_cholesky_size(0):
        mvn = gp.distributions.MultivariateNormal(torch.zeros(n, device=cuda_dev), k(x).add_jitter(1e-4))
        s = mvn.rsample(torch.Size([N])).double().cpu()
    emp = s.T @ s / N
    K = ro.kernel(x[:, None].cpu(), x[:, None].cpu(), 0.5, float(k.base_kernel.alpha), 1.5)
    assert (emp - K).abs().max().item() < 0.1, (emp - K).abs().max()


def test_predictions_after_lazy_love_samples_are_unchanged(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(2)
    n, m = 2000, 150
    train_x = (torch.arange(n, dtype=torch.float32) * 0.005).to(cuda_dev)
    train_y = (torch.sin(3 * train_x) + 0.1 * torch.randn(n, device=cuda_dev)).contiguous()
    k = kernels.ScaleKernel(kernels.RQKernel())
    model = _model(train_x, train_y, k, noise=0.01)
    model.eval()
    test_x = ((n + torch.arange(m, dtype=torch.float32)) * 0.005).to(cuda_dev)
    with torch.no_grad():
        f0 = model(test_x)
        mean0, var0 = f0.mean.clone(), f0.variance.clone()
        for _ in range(2):
            with settings.fast_pred_var(), settings.fast_pred_samples(), settings.ciq_samples(True):
                s = model(test_x).rsample(torch.Size([2]))
                assert s.shape == (2, m) and bool(torch.isfinite(s).all())
            f1 = model(test_x)
            assert torch.allclose(f1.mean, mean0, rtol=1e-5, atol=1e-6)
            assert torch.allclose(f1.variance, var0, rtol=1e-5, atol=1e-6 * float(var0.abs().max()))


def test_batch_shape_model_trains(cuda_dev):
    from gpytorch_b200 import kernels

    torch.manual_seed(1)
    n = 200
    x = torch.linspace(0, 4, n)
    train_x = torch.stack([x, x]).unsqueeze(-1)
    train_y = torch.stack([torch.sin(2 * x), torch.cos(5 * x)]) + 0.05 * torch.randn(2, n)
    train_x, train_y = train_x.to(cuda_dev), train_y.to(cuda_dev)
    k = kernels.ScaleKernel(kernels.RQKernel(batch_shape=torch.Size([2])))
    model = _model(train_x, train_y, k)
    losses = _train(model, train_x, train_y, 15, 0.05)
    assert losses[-1] < losses[0]
    g = k.base_kernel.raw_alpha.grad
    assert g is not None and g.shape == (2, 1) and bool((g != 0).all())
