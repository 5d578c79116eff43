"""Piecewise polynomial kernels on the device (run with -m gpu): plans on the compact-support backend (gp_plan_set_hypers_pp).
Every comparison is against tests/ppoly_oracle.py: K.V entry by entry within its derived bound (square and cross, ragged tiles,
q = 0..3, d in {1, 2, 3, 5, 8}, ARD, sparse and dense schedules, a chain of pairs just inside r = 1 across tile boundaries, duplicate
points), the evaluated tile pairs against the host restatement, bit-identical repeats, rows, the diagonal and pivots, the MLL and
the lengthscale / outputscale gradients against fp64, NaN inputs, the C refusals, and the public API (training, the dense
posterior, fast_pred_var, CIQ samples, fixed noise, a batch), and one MLL evaluation with gradients at N = 10^6."""
import math
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import ppoly_oracle as po  # noqa: E402
from oracle import linalg as ol, mll as om  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _plan(dev, x1, x2, q, ls, S=1.0, noise=0.0):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev))
    return p.set_hypers_pp(q, [float(v) for v in torch.as_tensor(ls).reshape(-1)], S, noise)


def _check_kmv(dev, x1, x2, q, ls, S, V):
    p = _plan(dev, x1, x2, q, ls, S)
    info = p.info()
    assert info["backend"] == "compact"
    out = p.kmv(V.to(dev)).double().cpu()
    xc = x1 if x2 is None else x2
    ref = po.kernel(x1, xc, ls, q, S) @ V.double()
    bnd = po.kmv_bound(x1, xc, ls, q, S, V)
    err = (out - ref).abs()
    assert bool(torch.isfinite(out).all()) and bool((err <= bnd).all()), (q, float((err / bnd).max()))
    _, _, R = po.schedule(x1.numpy(), None if x2 is None else x2.numpy(), ls)
    assert info["tile_pairs"] == int(R.sum()) and info["tile_pairs_total"] == R.size
    again = p.kmv(V.to(dev)).double().cpu()
    assert torch.equal(out, again)   # no atomics: repeated calls are bit-identical
    p.close()
    return float((err / bnd).max()), int(R.sum()), R.size


@pytest.mark.parametrize("q", [0, 1, 2, 3])
@pytest.mark.parametrize("d,ard", [(1, False), (2, True), (3, False), (5, True), (8, True)])
def test_kmv_within_bound_square_and_cross(cuda_dev, q, d, ard):
    g = torch.Generator().manual_seed(100 * q + d)
    n1, n2 = 1000 + 37, 700 + 5   # neither a multiple of 128 nor of 64
    x1 = torch.rand(n1, d, generator=g)
    x2 = torch.rand(n2, d, generator=g)
    ls = (0.15 + 0.1 * torch.rand(d if ard else 1, generator=g)) * (d ** 0.5)
    V = torch.randn(n2, 5, generator=g)
    _check_kmv(cuda_dev, x1, x2, q, ls, 1.3, V)
    _, pairs, total = _check_kmv(cuda_dev, x1, None, q, ls, 0.7, torch.randn(n1, 16, generator=g))
    if d <= 2:
        assert pairs < total   # the schedule prunes


def test_dense_schedule_duplicates_and_clusters(cuda_dev):
    g = torch.Generator().manual_seed(7)
    x = torch.rand(900, 3, generator=g)
    _, pairs, total = _check_kmv(cuda_dev, x, None, 2, torch.tensor([50.0]), 1.0, torch.randn(900, 4, generator=g))
    assert pairs == total
    dup = x[torch.randint(0, 40, (900,), generator=g)]   # many exact duplicates: r = 0 off the diagonal
    _check_kmv(cuda_dev, dup, None, 1, torch.tensor([0.3, 0.2, 0.4]), 1.0, torch.randn(900, 4, generator=g))
    c = torch.rand(6, 2, generator=g)
    cl = c[torch.randint(0, 6, (1500,), generator=g)] + 0.02 * torch.randn(1500, 2, generator=g)
    _check_kmv(cuda_dev, cl, None, 3, torch.tensor([0.05]), 1.0, torch.randn(1500, 3, generator=g))


def test_pairs_just_inside_the_support_across_tile_boundaries(cuda_dev):
    """q = 0, d = 1: k = (1 - r)_+ with j = 1.  Points on a line at spacing 1/70 of the lengthscale: every point reaches about 70
    neighbours on each side, across every 64- and 128-point tile boundary, and a pair at r just below 1 contributes 1 - r, far above
    the bound, so a dropped tile pair would show."""
    n = 2000
    x = (torch.arange(n, dtype=torch.float64) * (1.0 / 70.0 + 1e-7)).float()[:, None]
    x = x[torch.randperm(n, generator=torch.Generator().manual_seed(1))]   # the caller's order is not the spatial one
    V = torch.ones(n, 1)
    _check_kmv(cuda_dev, x, None, 0, torch.tensor([1.0]), 1.0, V)
    ref = po.kernel(x, x, [1.0], 0) @ V.double()
    bnd = po.kmv_bound(x, x, [1.0], 0, 1.0, V)
    far = ref.clone()
    K = po.kernel(x, x, [1.0], 0)
    perm = po.morton_perm(x.numpy())
    K[np.ix_(perm[128:256], perm[256 + 64:256 + 128])] = 0.0   # one boundary tile pair dropped
    assert bool(((K @ V.double() - far).abs() > bnd).any())


def test_rows_diag_and_pivots(cuda_dev):
    g = torch.Generator().manual_seed(11)
    n, d, S = 700, 2, 0.8
    x = torch.rand(n, d, generator=g)
    ls = torch.tensor([0.2, 0.3])
    K = po.kernel(x, x, ls, 2, S)
    p = _plan(cuda_dev, x, None, 2, ls, S, noise=0.1)
    idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
    assert float((p.rows(idx).double().cpu() - K[idx]).abs().max()) <= 2e-6 * S
    assert torch.equal(p.diag().cpu(), torch.full((n,), S, dtype=torch.float32))
    x2 = torch.rand(n, d, generator=g)
    pc = _plan(cuda_dev, x, x2, 2, ls, S)
    Kc = po.kernel(x, x2, ls, 2, S)
    assert float((pc.rows(idx).double().cpu() - Kc[idx]).abs().max()) <= 2e-6 * S
    assert float((pc.diag().double().cpu() - Kc.diagonal()).abs().max()) <= 2e-6 * S
    xp = torch.rand(64, 1, generator=g) * 3.0
    Kp = po.kernel(xp, xp, [0.5], 1, S)
    L, piv_o = ol.pivoted_cholesky(torch.full((64,), S, dtype=torch.float64), lambda i: Kp[i], 8)
    pp = _plan(cuda_dev, xp, None, 1, [0.5], S, noise=0.1)
    lt, piv, st = pp.pivoted_cholesky(8, 1e-6)
    assert st == 0
    m = lt.size(0)
    assert torch.equal(piv.cpu()[:min(m, 4)], piv_o[:min(m, 4)])
    for r in (p, pc, pp):
        r.close()


@pytest.mark.parametrize("q,d,ard,S", [(0, 1, False, 1.0), (1, 2, True, 1.4), (2, 2, False, 0.6), (3, 3, True, 1.0),
                                       (2, 5, True, 0.9)])
def test_bilinear_grad_matches_fp64_autograd_and_repeats(cuda_dev, q, d, ard, S):
    g = torch.Generator().manual_seed(40 + q + d)
    n, m, s = 600, 430, 13
    x1, x2 = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    ls = (0.3 + 0.2 * torch.rand(d if ard else 1, generator=g)) * d ** 0.5
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, x1, x2, q, ls, S)
    gl, gs = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    rl, rs = po.grads(x1, x2, ls.numpy(), q, S, L, R)
    # fp32 terms summed in fp32 within a tile and in fp64 across: the errors scale with the sums of the terms' magnitudes
    W = L.double().abs() @ R.double().abs().T
    near = (po.dist(x1, x2, ls) < 1.0).double()
    sc_s = float((W * po.kernel(x1, x2, ls, q)).sum())
    sc_l = S * po.max_slope(q, d) * float((W * near).sum()) / float(ls.min())
    assert abs(gs - rs) <= 1e-5 * sc_s, (gs, rs)
    assert np.abs(np.array(gl) - rl).max() <= 1e-5 * sc_l, (gl, rl)
    assert p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev)) == (gl, gs)
    p.close()


def test_mll_matches_the_oracle(cuda_dev):
    n, d, rank = 2500, 2, 30
    x, y = om.synthetic_problem(n, d, 4, torch.float32)
    ls, S, noise, q = [0.9, 1.2], 1.0, 0.3, 2
    K = po.kernel(x, x, ls, q, S)
    p = _plan(cuda_dev, x, None, q, ls, S, noise=noise)
    pn = om.make_probe_noise(n, rank, 10, 7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, S, noise, tuple(a.double() for a in pn), precond_size=rank, K=K)
    res, _ = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000)
    assert abs(res.mll - o64.mll) <= 1e-4 * max(1.0, abs(o64.mll)), (res.mll, o64.mll)
    p.close()


def test_nan_inputs_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(31)
    n, d = 300, 2
    x = torch.rand(n, d, generator=g)
    x[5, 1] = float("nan")
    p = _plan(cuda_dev, x, None, 2, [0.3, 0.3])
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(p.kmv(V).isnan().all())
    assert bool(p.rows(torch.tensor([0, 5])).isnan().all())
    gl, gs = p.bilinear_grad(V, V)
    assert len(gl) == 2 and all(math.isnan(t) for t in gl + [gs])
    q = _plan(cuda_dev, torch.rand(n, d, generator=g), None, 2, [0.3])
    for bad in (4, -1):
        with pytest.raises(RuntimeError, match="q expected to be 0, 1, 2 or 3"):
            q.set_hypers_pp(bad, [0.3], 1.0, 0.0)
    assert q.info()["backend"] == "compact"   # all or nothing
    with pytest.raises(RuntimeError, match="gp_plan_set_hypers_pp"):
        q.set_hypers("ppoly", [0.3], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="1 <= d <= 16"):
        _plan(cuda_dev, torch.rand(50, 17, generator=g), None, 2, [1.0])
    lib = q.lib
    other = Plan(torch.rand(n, d, generator=g).to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    tasks = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    for call, fn in [("gp_plan_set_tasks", lambda: q.set_tasks(tasks, None, 2)),
                     ("gp_plan_set_product", lambda: q.set_product([other, other])),
                     ("gp_plan_set_sum", lambda: q.set_sum([other, other])),
                     ("gp_plan_set_ski", lambda: q.set_ski([16] * d, [-4.0] * d, [0.5] * d)),
                     ("gp_plan_set_additive", lambda: q.set_additive(1, [1.0] * d)),
                     ("gp_plan_set_spectral", lambda: q.set_spectral([1.0], [[0.1] * d], [[0.2] * d])),
                     ("gp_plan_set_periodic", lambda: q.set_periodic([1.0])),
                     ("gp_plan_set_hypers_rq", lambda: q.set_hypers_rq([0.3], 1.0, 1.0, 0.0)),
                     ("gp_plan_set_hypers_poly", lambda: q.set_hypers_poly(2, 1.0, 1.0, 0.0)),
                     ("gp_plan_set_backend", lambda: _lib.check(lib.gp_plan_set_backend(q._h, _lib.GP_BACKEND_SIMT))),
                     ("gp_kmv_input_grad", lambda: q.kmv_input_grad(V[:, :1], V[:, :1], True, False)),
                     ("gp_plan_set_kron", lambda: _lib.check(lib.gp_plan_set_kron(q._h, other._h, 2))),
                     ("gp_plan_set_deriv", lambda: _lib.check(lib.gp_plan_set_deriv(q._h, other._h))),
                     (r"gp_plan_set_product \(a factor\)", lambda: other.set_product([q, q])),
                     (r"gp_plan_set_sum \(a term\)", lambda: other.set_sum([q, q])),
                     (r"gp_plan_set_kron \(the data plan\)", lambda: _lib.check(lib.gp_plan_set_kron(other._h, q._h, 2)))]:
        with pytest.raises(RuntimeError, match=f"{call}: the plan runs the compact-support backend"):
            fn()
    with pytest.raises(RuntimeError, match="gp_plan_set_hypers_pp takes a plain plan"):
        other.set_periodic([1.0])
        other.set_hypers_pp(2, [0.3], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="gp_plan_tile_pairs"):
        _lib.check(lib.gp_plan_tile_pairs(other._h, None, None))
    q.set_hypers("rbf", [0.3], 1.0, 0.0)   # back to a plain plan
    assert q.info()["backend"] in ("tcgen05", "simt") and bool(torch.isfinite(q.kmv(V)).all())
    for r in (p, q, other):
        r.close()


def _model(train_x, train_y, kernel, noise=None, fixed=None):
    import gpytorch_b200 as gp
    from gpytorch_b200 import likelihoods, means, models

    class PPGP(models.ExactGP):
        def __init__(self):
            bs = train_x.shape[:-2] if train_x.dim() == 3 else torch.Size()
            lik = likelihoods.FixedNoiseGaussianLikelihood(fixed) if fixed is not None else likelihoods.GaussianLikelihood(batch_shape=bs)
            super().__init__(train_x, train_y, lik)
            self.mean_module = means.ConstantMean(batch_shape=bs)
            self.covar_module = kernel

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    m = PPGP().to(train_x.device)
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
    n = 2000
    x = torch.rand(n, 2)
    y = torch.sin(6 * x[:, 0]) * torch.cos(4 * x[:, 1]) + 0.1 * torch.randn(n)
    k = kernels.ScaleKernel(kernels.PiecewisePolynomialKernel(q=2, ard_num_dims=2))
    k.base_kernel.lengthscale, k.outputscale = 0.4, 1.0
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model = _model(xd, yd, k, noise=0.05)
    with settings.max_cholesky_size(0):
        losses = _train(model, xd, yd, 25, 0.05)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    assert k.base_kernel.raw_lengthscale.grad is not None and k.raw_outputscale.grad is not None
    model.eval()
    tx = torch.rand(150, 2)
    ls = k.base_kernel.lengthscale.detach().cpu().reshape(-1)
    S, nz, c = float(k.outputscale.detach()), float(model.likelihood.noise.detach()), float(model.mean_module.constant.detach())
    Kxx = po.kernel(x, x, ls, 2, S) + nz * torch.eye(n, dtype=torch.float64)
    Ksx = po.kernel(tx, x, ls, 2, S)
    mean = Ksx @ torch.linalg.solve(Kxx, y.double() - c) + c
    var = S - (Ksx * torch.linalg.solve(Kxx, Ksx.T).T).sum(-1)
    with torch.no_grad(), settings.max_cholesky_size(0):
        f = model(tx.to(cuda_dev))
        assert rel(f.mean, mean) < 1e-2, rel(f.mean, mean)   # CG at the prediction tolerance
        # the posterior variance S - k^T K^-1 k is a small difference of O(S) terms: compared in units of S
        assert float((f.variance.double().cpu() - var).abs().max()) < 2e-2 * S
        with settings.fast_pred_var():
            fl = model(tx.to(cuda_dev))
            assert rel(fl.mean, mean) < 1e-2 and float((fl.variance.double().cpu() - var).abs().max()) < 2e-2 * S
    with torch.no_grad():   # the dense branch (N <= max_cholesky_size) runs through gp_krows
        fd = model(tx.to(cuda_dev))
    assert rel(fd.mean, mean) < 1e-2, rel(fd.mean, mean)


def test_fixed_noise_and_batch_models_train(cuda_dev):
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(1)
    n = 600
    x = torch.rand(n, 2)
    y = torch.sin(5 * x.sum(-1)) + 0.05 * torch.randn(n)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    k = kernels.ScaleKernel(kernels.PiecewisePolynomialKernel(q=1))
    k.base_kernel.lengthscale = 0.5
    model = _model(xd, yd, k, fixed=torch.full((n,), 0.01, device=cuda_dev))
    with settings.max_cholesky_size(0):
        losses = _train(model, xd, yd, 10, 0.05)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    bx = torch.stack([x, x + 0.5]).to(cuda_dev)
    by = torch.stack([y, torch.cos(3 * x[:, 0])]).to(cuda_dev)
    kb = kernels.ScaleKernel(kernels.PiecewisePolynomialKernel(q=3, batch_shape=torch.Size([2])), batch_shape=torch.Size([2]))
    kb.base_kernel.lengthscale = 0.5
    mb = _model(bx, by, kb)
    with settings.max_cholesky_size(0):
        losses = _train(mb, bx, by, 8, 0.05)
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]


def test_ciq_samples_have_the_kernel_covariance(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, settings

    torch.manual_seed(3)
    n, N = 40, 20000
    x = torch.linspace(0, 3, n).to(cuda_dev)
    k = kernels.ScaleKernel(kernels.PiecewisePolynomialKernel(q=2))
    k.base_kernel.lengthscale, k.outputscale = 0.8, 1.5
    k = k.to(cuda_dev)
    with torch.no_grad(), settings.ciq_samples(True), settings.max_cholesky_size(0):
        mvn = gp.distributions.MultivariateNormal(torch.zeros(n, device=cuda_dev), k(x).add_jitter(1e-4))
        s = mvn.rsample(torch.Size([N])).double().cpu()
    emp = s.T @ s / N
    K = po.kernel(x[:, None].cpu(), x[:, None].cpu(), [0.8], 2, 1.5)
    assert (emp - K).abs().max().item() < 0.1, (emp - K).abs().max()


def test_one_mll_with_gradients_at_a_million_points(cuda_dev):
    """N = 10^6 uniform points on the unit square, l = 0.02 (about 1.3 10^3 neighbours per point), q = 2: the MLL and its
    gradients complete, the plan evaluates the tile pairs the host restatement lists, and no N x N buffer is ever allocated."""
    n, ls, q = 1_000_000, 0.02, 2
    g = torch.Generator().manual_seed(5)
    x = torch.rand(n, 2, generator=g)
    y = torch.sin(8 * x[:, 0]) + torch.cos(6 * x[:, 1]) + 0.1 * torch.randn(n, generator=g)
    free0 = torch.cuda.mem_get_info(cuda_dev)[0]
    p = _plan(cuda_dev, x, None, q, [ls], 1.0, noise=0.2)
    info = p.info()
    assert info["tile_pairs"] == po.count_pairs(x.numpy(), None, [ls])
    assert info["tile_pairs"] < info["tile_pairs_total"] / 50
    pn = om.make_probe_noise(n, 15, 10, 3)
    res, solve = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, 15, 2000, want_solve=True)
    assert math.isfinite(res.mll) and res.cg_iters > 0
    gl, gs = p.bilinear_grad(solve[:, None], solve[:, None])
    assert math.isfinite(gl[0]) and math.isfinite(gs)
    used = free0 - torch.cuda.mem_get_info(cuda_dev)[0]
    assert used < 8 * 2 ** 30, used   # an N x N fp32 matrix would take 4 TB
    p.close()
