"""Input gradients of kernel products and dense kernel blocks (gp_kmv_input_grad / gp_kdense_input_grad, csrc/xgrad.cu) and the
test-input gradients of exact-GP posteriors through the public API.

Bounds, derived, not tuned (u = 2^-24; the full derivation is tests/xgrad_oracle.py:input_grad_bound):
  * primitives.  Entry-wise |engine - fp64 closed form| <= s sqrt(C)/l_c sum_j Wabs_ij q_ij (|z_ic - z_jc| eps_ij + E_ijc), where
    Wabs_ij = sum_c |G_ic| |V_jc| (product form; the t-term fp32 dot for w_ij costs t u of it) or |W_ij| (dense form), q the
    covariance's dk/da in the packed units, and eps_ij collects: the fp32 packing of z (two roundings, E = 2 u (|z_i| + |z_j|)
    absolute on the direction and (DP + 3) u |a| + E |z_i - z_j| on the argument a, amplified by |d ln q / da|), ex2.approx and
    sqrt.approx (2^-22 each), and the fp32 sums (<= n terms per split, then the per-split partials summed in a fixed order:
    2 n u) with the final scaling (3 u).  Every rounding is taken at its extreme with the same sign: a worst-case bound.
  * API.  The fp64 references rebuild mean and variance from the engine's own caches (_mean_cache alpha, _covar_cache R), so CG
    and Lanczos error do not enter.  The engine's gradient then differs by the primitive's error above, <= (n + t + 40) u of the
    sum of magnitudes (about 1e-4 of it at n = 4099), and that sum exceeds |gradient| by the cancellation of the kernel
    derivative's odd direction, at most 10x for the smooth models used: rtol 2e-3 of max|gradient|.  The exact covariance
    additionally goes through the fp32 Cholesky of K_hat (n <= max_cholesky_size), off by kappa(K_hat) u (Higham, Thm 10.3):
    kappa <= 1 + n s / sigma^2 = 1 + 400 * 1.5 / 0.1 ~ 6e3 gives 4e-4; rtol 5e-3.  The qUCB loss adds the fp32 Cholesky of the
    m x m predictive covariance (+ sigma^2 I; kappa <= 1 + m s / sigma^2 = 106) and the same bound.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok  # noqa: E402
from xgrad_oracle import input_grad, input_grad_bound  # noqa: E402

KINDS = ["rbf", "matern12", "matern32", "matern52"]
GP_E_SHAPE, GP_E_STATE = 1, 7

# (backend, n1 or "sq", n2, t, d)
CONFIGS = [("tcgen05", 1, 4097, 1, 6), ("simt", 7, 63, 3, 6), ("tcgen05", 129, 64, 16, 10), ("simt", 129, 65, 17, 3),
           ("tcgen05", 7, 4097, 100, 6), ("tcgen05", "sq", 65, 3, 6), ("simt", "sq", 129, 17, 10)]


def _plan(dev, x1, x2, backend, kind, ls, s):
    from gpytorch_b200.engine import Plan

    return Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend).set_hypers(kind, ls, s, 0.0)


def _check(got, ref, bound, what):
    err = (got.double().cpu() - ref).abs()
    assert torch.isfinite(got).all(), what
    assert (err <= bound).all(), (what, float((err - bound).max()), float(err.max()), float(bound.max()))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("cfg", CONFIGS, ids=[f"{c[0]}-{c[1]}x{c[2]}-t{c[3]}-d{c[4]}" for c in CONFIGS])
def test_primitives_match_fp64(cuda_dev, kind, ard, cfg):
    backend, n1, n2, t, d = cfg
    sq = n1 == "sq"
    g = torch.Generator().manual_seed(hash((kind, ard, str(cfg))) % 2**31)
    x2 = torch.rand(n2, d, generator=g)
    x1 = x2 if sq else torch.rand(n1, d, generator=g)
    n1 = x1.size(0)
    ls = [0.3 + 0.5 * c / d for c in range(d)] if ard else 0.45
    s = 1.3
    p = _plan(cuda_dev, x1, None if sq else x2, backend, kind, ls, s)
    lsv = torch.tensor(ls, dtype=torch.float64)
    G, V = torch.randn(n1, t, generator=g), torch.randn(n2, t, generator=g)
    d1, d2 = p.kmv_input_grad(G.to(cuda_dev), V.to(cuda_dev))
    Wp = G.double() @ V.double().T
    Wabs = G.double().abs() @ V.double().abs().T
    if sq:
        assert d2 is None
        _check(d1, input_grad(kind, x1, x1, lsv, s, Wp, same=True),
               input_grad_bound(kind, x1, x1, lsv, s, Wabs, 2 * t, same=True), "product, square")
    else:
        r1, r2 = input_grad(kind, x1, x2, lsv, s, Wp)
        b1, b2 = input_grad_bound(kind, x1, x2, lsv, s, Wabs, t)
        _check(d1, r1, b1, "product DX1")
        _check(d2, r2, b2, "product DX2")
    # dense form on the same plan
    W = torch.randn(n1, n2, generator=g)
    e1, e2 = p.dense_input_grad(W.to(cuda_dev))
    if sq:
        _check(e1, input_grad(kind, x1, x1, lsv, s, W.double(), same=True),
               input_grad_bound(kind, x1, x1, lsv, s, W.double().abs(), 0, same=True), "dense, square")
    else:
        r1, r2 = input_grad(kind, x1, x2, lsv, s, W.double())
        b1, b2 = input_grad_bound(kind, x1, x2, lsv, s, W.double().abs(), 0)
        _check(e1, r1, b1, "dense DX1")
        _check(e2, r2, b2, "dense DX2")


@pytest.mark.parametrize("kind", KINDS)
def test_coinciding_points_contribute_zero(cuda_dev, kind):
    g = torch.Generator().manual_seed(11 + KINDS.index(kind))
    x2 = torch.rand(200, 4, generator=g)
    x1 = torch.rand(5, 4, generator=g)
    x1[2] = x2[17]                                                       # a test point equal to a training point
    G, V = torch.randn(5, 2, generator=g), torch.randn(200, 2, generator=g)
    p = _plan(cuda_dev, x1, x2, "simt", kind, 0.4, 1.0)
    d1, d2 = p.kmv_input_grad(G.to(cuda_dev), V.to(cuda_dev))
    lsv = torch.tensor(0.4, dtype=torch.float64)
    r1, r2 = input_grad(kind, x1, x2, lsv, 1.0, G.double() @ V.double().T)
    b1, b2 = input_grad_bound(kind, x1, x2, lsv, 1.0, G.double().abs() @ V.double().abs().T, 2)
    _check(d1, r1, b1, "DX1 with a coinciding pair")
    _check(d2, r2, b2, "DX2 with a coinciding pair")
    # duplicated points on a square plan
    xs = torch.rand(150, 4, generator=g)
    xs[40] = xs[3]
    xs[41] = xs[3]
    Gs, Vs = torch.randn(150, 3, generator=g), torch.randn(150, 3, generator=g)
    ps = _plan(cuda_dev, xs, None, "tcgen05", kind, 0.4, 1.0)
    ds, _ = ps.kmv_input_grad(Gs.to(cuda_dev), Vs.to(cuda_dev))
    _check(ds, input_grad(kind, xs, xs, lsv, 1.0, Gs.double() @ Vs.double().T, same=True),
           input_grad_bound(kind, xs, xs, lsv, 1.0, Gs.double().abs() @ Vs.double().abs().T, 6, same=True), "square, duplicates")


def test_nan_input_propagates(cuda_dev):
    g = torch.Generator().manual_seed(5)
    x1, x2 = torch.rand(9, 3, generator=g), torch.rand(70, 3, generator=g)
    x2[13, 1] = float("nan")
    p = _plan(cuda_dev, x1, x2, "simt", "matern12", 0.5, 1.0)
    d1, d2 = p.kmv_input_grad(torch.randn(9, 2, device=cuda_dev), torch.randn(70, 2, device=cuda_dev))
    assert torch.isnan(d1).all() and torch.isnan(d2).all()
    e1, e2 = p.dense_input_grad(torch.randn(9, 70, device=cuda_dev))
    assert torch.isnan(e1).all() and torch.isnan(e2).all()


def test_repeated_and_strided_calls_are_bit_identical(cuda_dev):
    g = torch.Generator().manual_seed(21)
    x1, x2 = torch.rand(33, 5, generator=g), torch.rand(3000, 5, generator=g)
    p = _plan(cuda_dev, x1, x2, "tcgen05", "matern52", [0.3, 0.4, 0.5, 0.6, 0.7], 1.1)
    Gw, Vw = torch.randn(33, 60, generator=g).to(cuda_dev), torch.randn(3000, 60, generator=g).to(cuda_dev)
    G, V = Gw[:, 5:45], Vw[:, 7:47]                                      # ldg > t
    a1, a2 = p.kmv_input_grad(G, V)
    b1, b2 = p.kmv_input_grad(G.contiguous(), V.contiguous())
    c1, c2 = p.kmv_input_grad(G, V)
    assert torch.equal(a1, b1) and torch.equal(a2, b2) and torch.equal(a1, c1) and torch.equal(a2, c2)
    # strided outputs through the C ABI (ld1 > d)
    o1 = torch.full((33, 9), 7.0, device=cuda_dev)
    st = p.lib.gp_kmv_input_grad(p._h, C.c_void_p(G.data_ptr()), G.stride(0), C.c_void_p(V.data_ptr()), V.stride(0), 40,
                                 C.c_void_p(o1.data_ptr()), 9, C.c_void_p(0), 0)
    torch.cuda.synchronize()
    assert st == 0 and torch.equal(o1[:, :5], a1) and (o1[:, 5:] == 7.0).all()
    Ww = torch.randn(33, 3100, generator=g).to(cuda_dev)
    W = Ww[:, 50:3050]
    e1, e2 = p.dense_input_grad(W)
    f1, f2 = p.dense_input_grad(W.contiguous())
    assert torch.equal(e1, f1) and torch.equal(e2, f2)


def test_refusals(cuda_dev):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(3)
    x = torch.rand(300, 2, generator=g).to(cuda_dev)
    G = torch.randn(300, 2, device=cuda_dev)
    o = torch.empty(300, 70, device=cuda_dev)

    def call(p, t=2, dx2=None, rows=300):
        return p.lib.gp_kmv_input_grad(p._h, C.c_void_p(G.data_ptr()), 2, C.c_void_p(G.data_ptr()), 2, t,
                                       C.c_void_p(o.data_ptr()), 70, C.c_void_p(0 if dx2 is None else dx2.data_ptr()), 70)

    def dense(p):
        W = torch.zeros(300, 300, device=cuda_dev)
        return p.lib.gp_kdense_input_grad(p._h, C.c_void_p(W.data_ptr()), 300, C.c_void_p(o.data_ptr()), 70, C.c_void_p(0), 0)

    ski = Plan(x).set_ski([16, 16], [-0.2, -0.2], [0.1, 0.1]).set_hypers("rbf", 0.5, 1.0, 0.1)
    assert call(ski) == GP_E_SHAPE and dense(ski) == GP_E_SHAPE
    t1 = Plan(x, backend="simt").set_hypers("rbf", 0.5, 1.0, 0.0)
    t2 = Plan(x, backend="tcgen05").set_hypers("matern32", 0.5, 1.0, 0.0)
    s = Plan(x).set_hypers("rbf", [1.0], 1.0, 0.1).set_sum([t1, t2])
    assert call(s) == GP_E_SHAPE and dense(s) == GP_E_SHAPE
    assert call(t1) == 0 and call(t2) == 0                              # every term answers on its own
    lr = Plan(x, backend="tcgen05").set_hypers("rbf", 0.5, 1.0, 0.0)
    lr.set_lowrank(torch.randn(300, 4, device=cuda_dev) * 0.01)
    assert call(lr) == GP_E_STATE and dense(lr) == GP_E_STATE
    sq = Plan(x, backend="tcgen05").set_hypers("rbf", 0.5, 1.0, 0.0)
    assert call(sq, t=0) == GP_E_SHAPE                                 # t < 1
    assert call(sq, dx2=o) == GP_E_SHAPE                               # square: DX2 must be NULL
    shard = Plan(x, backend="simt", row_begin=0, row_count=150).set_hypers("rbf", 0.5, 1.0, 0.0)
    assert call(shard) == GP_E_SHAPE
    wide = Plan(torch.rand(300, 65, device=cuda_dev), backend="simt").set_hypers("rbf", 3.0, 1.0, 0.0)
    assert call(wide) == GP_E_SHAPE                                    # d > 64, the limit of gp_bilinear_grad
    with pytest.raises(RuntimeError, match="row-sharded"):
        shard.kmv_input_grad(G[:150], G)


# ---- API ---------------------------------------------------------------------------------------------------------------------
def _model(dev, x, y, kernel, lik_kind):
    import gpytorch_b200 as gp

    n = x.size(0)
    if lik_kind == "fixed":
        lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=(0.05 + 0.1 * torch.rand(n, generator=torch.Generator().manual_seed(1))).to(dev))
    else:
        lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            if kernel == "ard":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel(ard_num_dims=2, active_dims=[0, 2]))
            else:
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel()) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    lik = lik.to(dev)
    if kernel == "ard":
        model.covar_module.base_kernel.lengthscale = torch.tensor([[0.4, 0.7]])
        model.covar_module.outputscale = 1.5
        terms = [("rbf", [0, 2], torch.tensor([0.4, 0.7], dtype=torch.float64), 1.5)]
    else:
        a, b = model.covar_module.kernels
        a.base_kernel.lengthscale = 0.5; a.outputscale = 1.2
        b.base_kernel.lengthscale = 0.8; b.outputscale = 0.3
        terms = [("rbf", [0, 1, 2], 0.5, 1.2), ("matern52", [0, 1, 2], 0.8, 0.3)]
    model.mean_module.constant = 0.3
    if lik_kind == "gauss":
        lik.noise = 0.1
    model.eval(); lik.eval()
    return model, lik, terms


def _kfun(terms, a, b):
    return sum(ok.kernel_matrix(kind, a[:, dims], b[:, dims], ls, s, x1_eq_x2=False) for kind, dims, ls, s in terms)


def _data(n, m, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g)
    y = torch.sin(5 * x[:, 0]) + torch.cos(3 * x[:, 2]) + 0.1 * torch.randn(n, generator=g)
    return x, y, torch.rand(m, 3, generator=g)


def _close(got, ref, rtol, what):
    got = got.double().cpu()
    scale = float(ref.abs().max())
    assert float((got - ref).abs().max()) <= rtol * scale, (what, float((got - ref).abs().max()), scale)


@pytest.mark.parametrize("kernel", ["ard", "additive"])
@pytest.mark.parametrize("lik_kind", ["gauss", "fixed"])
@pytest.mark.parametrize("mode", ["exact", "love"])
def test_api_posterior_input_gradients(cuda_dev, kernel, lik_kind, mode):
    from gpytorch_b200 import settings

    n, m = 400, 7
    x, y, xs = _data(n, m, seed=31 + (kernel == "ard") + 2 * (lik_kind == "fixed"))
    model, lik, terms = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), kernel, lik_kind)
    xs_d = xs.to(cuda_dev)
    with torch.no_grad(), settings.fast_pred_var(mode == "love"):
        post0 = model(xs_d)
        mean0, var0 = post0.mean.clone(), post0.variance.clone()
    xg = xs_d.clone().requires_grad_(True)
    with settings.fast_pred_var(mode == "love"):
        post = model(xg)
        mean, var = post.mean, post.variance
        assert torch.equal(mean.detach(), mean0) and torch.equal(var.detach(), var0)   # forward values do not change
        gm, = torch.autograd.grad(mean.sum(), xg, retain_graph=True)
        gv, = torch.autograd.grad(var.sum(), xg)
    X = x.double()
    alpha = model._mean_cache.double().cpu()
    s_tot = sum(t[3] for t in terms)
    a = xs.double().clone().requires_grad_(True)
    ks = _kfun(terms, a, X)
    rm, = torch.autograd.grad((0.3 + ks @ alpha).sum(), a, retain_graph=True)
    if mode == "love":
        R = model._covar_cache.double().cpu()
        rv, = torch.autograd.grad((s_tot - ((ks @ R) ** 2).sum(-1)).sum(), a)
        rtol_v = 2e-3
    else:
        D = lik.noise_covar.noise.double().cpu() if lik_kind == "fixed" else torch.full((n,), 0.1, dtype=torch.float64)
        D = D.float().double()                                              # the fp32 noise the engine holds
        Khat = _kfun(terms, X, X) + torch.diag(D)
        rv, = torch.autograd.grad((s_tot - (ks * torch.linalg.solve(Khat, ks.T).T).sum(-1)).sum(), a)
        rtol_v = 5e-3
    _close(gm, rm, 2e-3, "d mean / dx*")
    _close(gv, rv, rtol_v, "d variance / dx*")


def test_api_large_n_mean_and_love_gradients(cuda_dev):
    """N = 4099 > max_cholesky_size: the mean cache comes from CG at a tight eval_cg_tolerance, the LOVE root from Lanczos; the
    references take both caches from the engine, so only the primitive's error is compared."""
    from gpytorch_b200 import settings

    n, m = 4099, 33
    x, y, xs = _data(n, m, seed=41)
    model, lik, terms = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), "ard", "gauss")
    xg = xs.to(cuda_dev).requires_grad_(True)
    with settings.eval_cg_tolerance(1e-4), settings.fast_pred_var():
        post = model(xg)
        gm, = torch.autograd.grad(post.mean.sum(), xg, retain_graph=True)
        gv, = torch.autograd.grad(post.variance.sum(), xg)
    a = xs.double().clone().requires_grad_(True)
    ks = _kfun(terms, a, x.double())
    rm, = torch.autograd.grad((ks @ model._mean_cache.double().cpu()).sum(), a, retain_graph=True)
    R = model._covar_cache.double().cpu()
    rv, = torch.autograd.grad((1.5 - ((ks @ R) ** 2).sum(-1)).sum(), a)
    _close(gm, rm, 2e-3, "d mean / dx*, N = 4099")
    _close(gv, rv, 2e-3, "d LOVE variance / dx*, N = 4099")
    # one test point (the gradient arrives as an expanded [1, t] block); rows of the posterior are independent
    x1 = xs[:1].to(cuda_dev).requires_grad_(True)
    with settings.eval_cg_tolerance(1e-4), settings.fast_pred_var():
        post = model(x1)
        g1, = torch.autograd.grad(post.mean.sum() + post.variance.sum(), x1)
    _close(g1, rm[:1] + rv[:1], 2e-3, "one test point")


def test_api_qucb_through_rsample(cuda_dev):
    """qUCB-style loss mean_s max_i (mu_i + beta |L eps_s|_i) of likelihood(post).rsample(base_samples=eps), backpropagated to x*,
    against the same loss in fp64 (exact covariance, dense Cholesky of K** - K*x K_hat^-1 Kx* + sigma^2 I)."""
    n, m, S, beta = 400, 6, 64, 2.0
    x, y, xs = _data(n, m, seed=51)
    model, lik, terms = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), "additive", "gauss")
    eps = torch.randn(S, m, generator=torch.Generator().manual_seed(52))
    xg = xs.to(cuda_dev).requires_grad_(True)
    post = lik(model(xg))
    smp = post.rsample(base_samples=eps.to(cuda_dev))
    mu = post.mean
    loss = (mu + beta * (smp - mu).abs()).max(-1).values.mean()
    g, = torch.autograd.grad(loss, xg)
    X = x.double()
    alpha = model._mean_cache.double().cpu()
    a = xs.double().clone().requires_grad_(True)
    ks = _kfun(terms, a, X)
    Khat = _kfun(terms, X, X) + 0.1 * torch.eye(n, dtype=torch.float64)
    mu_r = 0.3 + ks @ alpha
    cov = _kfun(terms, a, a) - ks @ torch.linalg.solve(Khat, ks.T) + 0.1 * torch.eye(m, dtype=torch.float64)
    L = torch.linalg.cholesky(cov)
    smp_r = mu_r + eps.double() @ L.T
    loss_r = (mu_r + beta * (smp_r - mu_r).abs()).max(-1).values.mean()
    gr, = torch.autograd.grad(loss_r, a)
    _close(g, gr, 5e-3, "qUCB loss")


def test_api_lazy_love_and_ski_stay_detached(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n, m = 400, 9
    x, y, xs = _data(n, m, seed=61)
    model, lik, _ = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), "additive", "gauss")
    xg = xs.to(cuda_dev).requires_grad_(True)
    with settings.fast_pred_samples():
        post = model(xg)
        gm, = torch.autograd.grad(post.mean.sum(), xg, retain_graph=True)      # the mean is differentiable
        assert torch.isfinite(gm).all() and gm.abs().max() > 0
        assert post.lazy_covariance_matrix.to_dense().grad_fn is None           # the lazy LOVE covariance is not
        assert post.variance.grad_fn is None
        assert post.rsample(torch.Size([2])).shape == (2, m)
    # KISS-GP: the joint SKI path is detached w.r.t. x*
    x2 = x[:, :2].contiguous()
    lik2 = gp.likelihoods.GaussianLikelihood()

    class S(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x2.to(cuda_dev), y.to(cuda_dev), lik2)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), 24, num_dims=2))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    ms = S().to(cuda_dev)
    lik2.to(cuda_dev)
    lik2.noise = 0.1
    ms(x2.to(cuda_dev))                                                 # sizes the grid from the training inputs
    ms.eval(); lik2.eval()
    xs2 = (0.1 + 0.8 * xs[:, :2]).to(cuda_dev).requires_grad_(True)
    for flag in (False, True):
        with settings.ski_grid_prediction(flag), settings.fast_pred_var():
            p2 = ms(xs2)
            assert torch.isfinite(p2.mean).all() and torch.isfinite(p2.variance).all()
            gx = torch.autograd.grad(p2.mean.sum(), xs2, allow_unused=True)[0] if p2.mean.requires_grad else None
            assert gx is None or float(gx.abs().max()) == 0.0
