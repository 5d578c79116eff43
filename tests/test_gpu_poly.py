"""Polynomial kernels on the device (run with -m gpu): plans of kind GP_POLY (gp_plan_set_hypers_poly) on the tensor-core and
CUDA-core K.V.  Every comparison is against the fp64 oracle of tests/poly_oracle.py: K.V entry by entry within its derived bound
on both backends over a power / offset / width sweep and at the ring and split edges, rows, the square and cross diagonal, the
first pivot, the rank-deficient pivoted Cholesky, the MLL, the gradients (with determinism), input gradients with the diagonal
term, NaN inputs, and the public API (a fitted polynomial + RBF model against the dense posterior, CIQ samples, lazy LOVE, a
batch of two)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import kmv_oracle as ko  # noqa: E402
import poly_oracle as po  # noqa: E402
from oracle import linalg as ol  # noqa: E402

PATH = {"tcgen05": "tc", "simt": "simt"}


def _points(n, d, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, d, generator=g) * 2 - 1) * scale / math.sqrt(d)


def _plan(dev, x1, x2, p, c, S=1.0, noise=0.0, backend="auto"):
    from gpytorch_b200.engine import Plan

    pl = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend)
    return pl.set_hypers_poly(p, c, S, noise)


def _check_kmv(dev, x1, x2, p, c, S, V, backend):
    pl = _plan(dev, x1, x2, p, c, S, backend=backend)
    info = pl.info()
    assert info["backend"] == backend
    out = pl.kmv(V.to(dev)).double().cpu()
    xc = x1 if x2 is None else x2
    geo = ko.geometry(x1.size(0), xc.size(0), x1.size(1), backend, info["n_sm"])
    assert geo["nsplit"] == info["nsplit"]
    c32 = float(torch.tensor(c, dtype=torch.float32))
    ref = po.kernel(x1, xc, p, c32, float(torch.tensor(S, dtype=torch.float32))) @ V.double()
    bnd = po.kmv_bound(x1, xc, p, c32, V, S, PATH[backend], geo["nsplit"], geo["T"])
    err = (out - ref).abs()
    assert bool(torch.isfinite(out).all()) and bool((err <= bnd).all()), (backend, p, c, float((err / bnd).max()))
    pl.close()


@pytest.mark.parametrize("d", [1, 3, 8, 20, 41, 64])
def test_kmv_within_bound_on_both_backends(cuda_dev, d):
    n1, n2 = 700, 450
    for p, c, scale in [(1, 0.0, 1.0), (2, 0.1, 1.0), (3, 10.0, 0.5), (5, 0.1, 3.0), (8, 1.0, 0.3)]:
        x1, x2 = _points(n1, d, 11 + p, scale), _points(n2, d, 17 + p, scale)
        V = torch.randn(n1, 5, generator=torch.Generator().manual_seed(p))
        backends = ["simt"] + (["tcgen05"] if 3 * d + 4 <= 128 else [])
        for b in backends:
            _check_kmv(cuda_dev, x1, None, p, c, 1.3, V, b)                     # square
            _check_kmv(cuda_dev, x1, x2, p, c, 0.7, V[:n2], b)                  # cross


def test_kmv_at_ring_split_edges_and_wide_norms(cuda_dev):
    # column counts at tile and split edges, and inputs whose norms span four decades (entries grow as |x|^2p)
    for n2 in (63, 64, 65, 8 * 64 + 1):
        x1, x2 = _points(300, 4, 1), _points(n2, 4, 2)
        V = torch.randn(n2, 16, generator=torch.Generator().manual_seed(n2))
        _check_kmv(cuda_dev, x1, x2, 3, 0.1, 1.0, V, "tcgen05")
        _check_kmv(cuda_dev, x1, x2, 3, 0.1, 1.0, V, "simt")
    x = _points(513, 5, 3) * torch.logspace(-2, 2, 513).unsqueeze(1)
    V = torch.randn(513, 3, generator=torch.Generator().manual_seed(4))
    for p in (1, 2, 4):
        _check_kmv(cuda_dev, x, None, p, 0.5, 1.0, V, "tcgen05")
        _check_kmv(cuda_dev, x, None, p, 0.5, 1.0, V, "simt")


def test_rows_and_diagonals(cuda_dev):
    x1, x2 = _points(300, 3, 5, 2.0), _points(260, 3, 6, 2.0)
    for b in ("tcgen05", "simt"):
        pl = _plan(cuda_dev, x1, None, 3, 0.2, 1.5, backend=b)
        idx = torch.tensor([0, 7, 299], device=cuda_dev)
        rows = pl.rows(idx).double().cpu()
        K = po.kernel(x1, x1, 3, 0.2, 1.5)
        assert torch.allclose(rows, K[[0, 7, 299]], rtol=1e-5, atol=1e-5 * K.abs().max().item())
        dg = pl.diag().double().cpu()
        assert torch.allclose(dg, po.diag(x1, 3, 0.2, 1.5), rtol=1e-5)   # S (|x|^2 + c)^p, not the constant S
        pc = _plan(cuda_dev, x1[:260], x2, 3, 0.2, 1.5, backend=b)
        assert torch.allclose(pc.diag().double().cpu(), 1.5 * ((x1[:260].double() * x2.double()).sum(1) + 0.2) ** 3, rtol=1e-5,
                              atol=1e-6)


def test_first_pivot_is_the_argmax_diagonal_and_rank_deficient_factor_is_valid(cuda_dev):
    x = _points(800, 3, 7, 2.0)
    pl = _plan(cuda_dev, x, None, 2, 0.5, 1.0, noise=0.1)
    lt, piv, st = pl.pivoted_cholesky(15, 1e-3)
    dg = po.diag(x, 2, 0.5)
    assert int(piv[0]) == int(torch.argmax(dg))
    # d = 1, p = 2: K has rank 3, the rank-15 factor runs past it without NaN or a NaN warning
    x1 = _points(600, 1, 8, 2.0)
    pl1 = _plan(cuda_dev, x1, None, 2, 0.5, 1.0, noise=0.1)
    lt, piv, st = pl1.pivoted_cholesky(15, 1e-3)
    assert st == 0, st   # not GP_W_PIVCHOL_NAN
    L = lt.double().cpu()   # [m, n]
    assert L.size(0) >= 3 and bool(torch.isfinite(L).all())
    K = po.kernel(x1, x1, 2, 0.5)
    assert (L.T @ L - K).abs().max() <= 1e-3 * K.abs().max()


def test_mll_matches_the_dense_oracle(cuda_dev):
    from oracle import mll as om

    n, d = 1200, 3
    x = _points(n, d, 9)
    y = torch.sin(3 * x.sum(1)) + 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(1))
    for p in (1, 2, 3):
        pl = _plan(cuda_dev, x, None, p, 0.5, 1.0, noise=0.05)
        pn = om.make_probe_noise(n, 30, 10, 1)
        res, _ = pl.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, 30, 2000)
        K = po.kernel(x, x, p, 0.5) + 0.05 * torch.eye(n, dtype=torch.float64)
        Lc = torch.linalg.cholesky(K)
        yd = y.double()
        inv_quad = float(yd @ torch.cholesky_solve(yd[:, None], Lc)[:, 0])
        logdet = float(2 * torch.log(torch.diagonal(Lc)).sum())
        assert abs(res.inv_quad - inv_quad) <= 1e-3 * abs(inv_quad), (p, res.inv_quad, inv_quad)
        assert abs(res.logdet - logdet) <= 0.05 * abs(logdet) + 5.0, (p, res.logdet, logdet)


def test_gradients_against_fp64_autograd_and_repeatable(cuda_dev):
    x1, x2 = _points(500, 4, 12), _points(300, 4, 13)
    L, R = torch.randn(500, 3, generator=torch.Generator().manual_seed(1)), torch.randn(300, 3, generator=torch.Generator().manual_seed(2))
    W = L.double() @ R.double().T
    for b in ("tcgen05", "simt"):
        for p, c in [(1, 0.3), (2, 0.0), (3, 2.0)]:
            pl = _plan(cuda_dev, x1, x2, p, c, 1.2, backend=b)
            gl, go = pl.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
            gl2, go2 = pl.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
            assert gl == gl2 and go == go2
            gc, gs = po.grads(x1, x2, p, float(torch.tensor(c, dtype=torch.float32)), W, float(torch.tensor(1.2)))
            scale = (W.abs() * po.entry_bound(x1, x2, max(p - 1, 1), c, "simt")[1]).sum().item() * p * 1.2
            assert abs(gl[0] - float(gc)) <= 1e-4 * scale + 1e-6, (b, p, gl[0], float(gc))
            assert abs(go - float(gs)) <= 1e-4 * (W.abs() * po.entry_bound(x1, x2, p, c, "simt")[1]).sum().item(), (b, p)


def test_input_gradients_include_the_diagonal_term(cuda_dev):
    x, x2 = _points(200, 3, 14), _points(150, 3, 15)
    G, V = torch.randn(200, 2, generator=torch.Generator().manual_seed(3)), torch.randn(200, 2, generator=torch.Generator().manual_seed(4))
    pl = _plan(cuda_dev, x, None, 3, 0.4, 1.1)
    d1, _ = pl.kmv_input_grad(G.to(cuda_dev), V.to(cuda_dev))
    ref, _ = po.input_grads(x, None, 3, 0.4, G.double() @ V.double().T, 1.1)
    assert torch.allclose(d1.double().cpu(), ref, rtol=1e-4, atol=1e-4 * ref.abs().max().item())
    pc = _plan(cuda_dev, x, x2, 2, 0.4, 1.1)
    W = torch.randn(200, 150, generator=torch.Generator().manual_seed(5))
    a, b = pc.dense_input_grad(W.to(cuda_dev))
    ra, rb = po.input_grads(x, x2, 2, 0.4, W, 1.1)
    assert torch.allclose(a.double().cpu(), ra, rtol=1e-4, atol=1e-4 * ra.abs().max().item())
    assert torch.allclose(b.double().cpu(), rb, rtol=1e-4, atol=1e-4 * rb.abs().max().item())


def test_nan_inputs_give_nan(cuda_dev):
    x = _points(100, 2, 16)
    x[5, 1] = float("nan")
    pl = _plan(cuda_dev, x, None, 2, 0.1, 1.0)
    out = pl.kmv(torch.ones(100, 1, device=cuda_dev))
    assert bool(torch.isnan(out).all())


def _fit_data(n=300, d=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g) * 2 - 1
    y = 0.8 * x[:, 0] ** 2 - 0.5 * x[:, 1] + 0.2 * torch.sin(6 * x[:, 0]) + 0.05 * torch.randn(n, generator=g)
    return x, y


def test_fitted_poly_plus_rbf_model_matches_the_dense_posterior(cuda_dev):
    import gpytorch_b200 as gp

    x, y = _fit_data()
    xt = torch.rand(40, 2, generator=torch.Generator().manual_seed(9)) * 2 - 1
    x, y, xt = x.to(cuda_dev), y.to(cuda_dev), xt.to(cuda_dev)

    class M(gp.models.ExactGP):
        def __init__(self, x, y, lik):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.PolynomialKernel(2)) + gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    m = M(x, y, lik).to(cuda_dev)
    m.train(); lik.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.05)
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, m)
    for _ in range(15):
        opt.zero_grad()
        loss = -mll(m(x), y)
        loss.backward()
        opt.step()
    poly = m.covar_module.kernels[0]
    assert poly.base_kernel.raw_offset.grad is not None and torch.isfinite(poly.base_kernel.raw_offset.grad).all()
    m.eval(); lik.eval()
    with torch.no_grad(), gp.settings.fast_pred_var(False):
        pred = lik(m(xt))
        mean, var = pred.mean.double().cpu(), pred.variance.double().cpu()
    # dense posterior in fp64 from the fitted hyper-parameters
    rb = m.covar_module.kernels[1]
    s1, c, s2 = float(poly.outputscale), float(poly.base_kernel.offset), float(rb.outputscale)
    ls, nz, mu = float(rb.base_kernel.lengthscale), float(lik.noise), float(m.mean_module.constant)
    X, Xt = x.double().cpu(), xt.double().cpu()

    def k(a, b):
        return s1 * po.kernel(a, b, 2, c) + s2 * torch.exp(-0.5 * torch.cdist(a, b) ** 2 / ls ** 2)

    Kxx = k(X, X) + nz * torch.eye(X.size(0), dtype=torch.float64)
    Ks = k(Xt, X)
    sol = torch.linalg.solve(Kxx, y.double().cpu() - mu)
    ref_mean = mu + Ks @ sol
    ref_var = torch.diagonal(k(Xt, Xt)) - (Ks * torch.linalg.solve(Kxx, Ks.T).T).sum(1) + nz
    assert (mean - ref_mean).abs().max() <= 1e-2 * ref_mean.abs().max() + 1e-3
    assert (var - ref_var).abs().max() <= 2e-2 * ref_var.abs().max() + 1e-3
    # lazy LOVE and CIQ samples through the same model
    with torch.no_grad(), gp.settings.fast_pred_var(True):
        pv = lik(m(xt)).variance.double().cpu()
    assert (pv - ref_var).abs().max() <= 5e-2 * ref_var.abs().max() + 1e-2
    with torch.no_grad(), gp.settings.ciq_samples(True):
        s = m(xt).rsample(torch.Size([64]))
    assert s.shape[-1] == 40 and bool(torch.isfinite(s).all())


def test_batch_of_two(cuda_dev):
    import gpytorch_b200 as gp

    k = gp.kernels.ScaleKernel(gp.kernels.PolynomialKernel(3, batch_shape=torch.Size([2])), batch_shape=torch.Size([2])).to(cuda_dev)
    with torch.no_grad():
        k.base_kernel.offset = torch.tensor([[0.5], [2.0]], device=cuda_dev)
        k.outputscale = torch.tensor([1.0, 0.3], device=cuda_dev)
    x = torch.stack([_points(150, 2, 20), _points(150, 2, 21)]).to(cuda_dev)
    V = torch.randn(2, 150, 2, generator=torch.Generator().manual_seed(1)).to(cuda_dev)
    op = k(x)
    out = op.matmul(V).double().cpu()
    for b, (c, s) in enumerate([(0.5, 1.0), (2.0, 0.3)]):
        ref = po.kernel(x[b].cpu(), x[b].cpu(), 3, c, s) @ V[b].double().cpu()
        assert (out[b] - ref).abs().max() <= 1e-4 * ref.abs().max()
