"""GPU parity at the REAL configurations (run with -m gpu on an H100).

* C2 at full size (N = 50 000, d = 10, RBF, rank-100 preconditioner): the whole MLL evaluation against the oracle run in
  the reference's default dtype (fp32) on identical inputs and probe base samples -- size-dependent paths (nsplit = 3, 391
  row tiles / 782 column tiles, ring wrap-around) are only exercised here.
* C3-shaped (Matern-5/2, d = 20 => KP = 64, three shared-memory stages in the tensor-core kernel), multi-tile, ragged N: K.V and the
  MLL against the fp64 oracle, both backends.
* third-party anchors that are NOT this repository's restatement: scikit-learn's GaussianProcessRegressor log marginal
  likelihood (dense Cholesky) and scipy.sparse.linalg.cg.
* the stale-plan hazard: inputs updated in place must be re-packed.

Tolerance rule for Krylov quantities (DESIGN.md section 2): |gpu - o64| <= max(1e-4 |o64|, 3 |o32 - o64|), i.e. the engine may
be no further from the fp64 oracle than three times what the reference's own fp32 run is.  At N = 50 000 an fp64 oracle run
is not affordable, so the fp32-vs-fp64 gap is measured at N = 12 000 (same data distribution, same hyper-parameters) and the
full-size run is compared with the fp32 oracle: |gpu - o32| <= max(1e-4, 3 gap) |o32|.
"""
import math
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok, linalg as ol, mll as om  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def relf(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.fixture(scope="module")
def Plan(cuda_dev):
    from gpytorch_b200.engine import Plan as P

    return P


def _host_gb():
    try:
        import psutil

        return psutil.virtual_memory().available / 1e9
    except Exception:
        return 0.0


def _gpu_mll(Plan, dev, x, y, pn, kind, ls, rank, backend="auto", want_solve=True):
    p = Plan(x.to(dev), backend=backend).set_hypers(kind, ls, 1.0, 0.1)
    res, sol = p.mll(y.to(dev), pn[0].to(dev), pn[1].to(dev), pn[2].to(dev), 10, rank, 2000, want_solve=want_solve)
    info = p.info()
    p.close()
    return res, sol, info


@pytest.mark.timeout(1500)
def test_c2_full_size_mll_matches_fp32_oracle(Plan, cuda_dev):
    if _host_gb() < 36:
        pytest.skip("the N=50000 oracle needs ~25 GB of host memory for the dense K")
    kind, ls, rank, d = "rbf", 1.0, 100, 10
    # (1) how far is the reference's own fp32 run from fp64?  measured at N = 12000
    n0 = 12000
    x0, y0 = om.synthetic_problem(n0, d, 0, torch.float32)
    pn0 = om.make_probe_noise(n0, rank, 10, 1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm(kind, x0.double(), y0.double(), 0.0, ls, 1.0, 0.1, tuple(a.double() for a in pn0), precond_size=rank)
        o32 = om.mll_bbmm(kind, x0, y0, 0.0, ls, 1.0, 0.1, pn0, precond_size=rank)
    gap_iq, gap_ld = relf(o32.inv_quad, o64.inv_quad), relf(o32.logdet, o64.logdet)
    g0, _, _ = _gpu_mll(Plan, cuda_dev, x0, y0, pn0, kind, ls, rank, "tcgen05")
    assert g0.cg_iters == o64.iters == o32.iters
    assert relf(g0.inv_quad, o64.inv_quad) <= max(1e-4, 3 * gap_iq), (g0.inv_quad, o64.inv_quad, o32.inv_quad)
    assert relf(g0.logdet, o64.logdet) <= max(1e-4, 3 * gap_ld), (g0.logdet, o64.logdet, o32.logdet)
    del o64
    # (2) the full configuration against the fp32 oracle
    n = 50000
    x, y = om.synthetic_problem(n, d, 0, torch.float32)
    pn = om.make_probe_noise(n, rank, 10, 1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o = om.mll_bbmm(kind, x, y, 0.0, ls, 1.0, 0.1, pn, precond_size=rank)
    piv_o = o.precond.pivots.clone()
    sol_o = o.solves[:, -1].clone() if o.solves is not None else None
    tm_o = o.t_mat.clone()
    iq_o, ld_o, it_o, mll_o = o.inv_quad, o.logdet, o.iters, o.mll
    del o
    for backend in ("tcgen05", "simt"):
        p = Plan(x.to(cuda_dev), backend=backend).set_hypers(kind, ls, 1.0, 0.1)
        info = p.info()
        assert info["backend"] == backend
        if backend == "tcgen05":
            assert info["nsplit"] >= 2   # the size-dependent split path is what this test is for
        # pivots are integer work: bit-exact even at full size
        lt, piv, st = p.pivoted_cholesky(rank, 1e-3)
        assert st == 0 and torch.equal(piv.cpu(), piv_o)
        res, sol = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000, want_solve=True)
        assert res.cg_iters == it_o == 21 and res.tridiag_size == 20 and res.precond_rank == 100
        tol_iq, tol_ld = max(1e-4, 3 * gap_iq), max(1e-4, 3 * gap_ld)
        assert relf(res.inv_quad, iq_o) <= tol_iq, (backend, res.inv_quad, iq_o, tol_iq)
        assert relf(res.logdet, ld_o) <= tol_ld, (backend, res.logdet, ld_o, tol_ld)
        assert abs(res.mll - mll_o) <= (tol_iq * abs(iq_o) + tol_ld * abs(ld_o)) / (2 * n)
        if sol_o is not None:
            assert rel(sol, sol_o) <= 5e-3, (backend, rel(sol, sol_o))   # cg_tolerance = 1: 21 fp32 iterations on each side
        p.close()


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_c3_shape_matern52_d20_multitile(Plan, cuda_dev, backend):
    """Matern-5/2, d = 20 (KP = 64): many row / column tiles, ragged N, two column splits."""
    n, d, kind, ls, rank = 9037, 20, "matern52", 2.0, 100
    x, y = om.synthetic_problem(n, d, 0, torch.float32)
    g = torch.Generator().manual_seed(7)
    v = torch.randn(n, 11, generator=g, dtype=torch.float64)
    K = ok.kernel_matrix(kind, x.double(), x.double(), ls, 1.0, True)
    p = Plan(x.to(cuda_dev), backend=backend).set_hypers(kind, ls, 1.0, 0.1)
    info = p.info()
    assert info["backend"] == backend
    if backend == "tcgen05":
        assert info["kpad"] == 64
    assert rel(p.kmv(v.float().to(cuda_dev)), K @ v) < (5e-6 if backend == "tcgen05" else 2e-6)
    assert rel(p.kmv(v.float().to(cuda_dev), add_noise=True), K @ v + 0.1 * v) < (5e-6 if backend == "tcgen05" else 2e-6)
    # a few exact rows
    idx = torch.tensor([0, 127, 128, 4500, n - 1])
    assert (p.rows(idx).double().cpu() - K[idx]).abs().max() < 2e-6
    # the MLL with the rank-100 preconditioner
    pn = om.make_probe_noise(n, rank, 10, 1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm(kind, x.double(), y.double(), 0.0, ls, 1.0, 0.1, tuple(a.double() for a in pn), precond_size=rank, K=K)
        o32 = om.mll_bbmm(kind, x, y, 0.0, ls, 1.0, 0.1, pn, precond_size=rank)
    res, sol = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000, want_solve=True)
    assert res.cg_iters == o64.iters and res.precond_rank == o64.precond.L.size(1)
    lt, piv, st = p.pivoted_cholesky(rank, 1e-3)
    assert torch.equal(piv.cpu(), o64.precond.pivots)
    assert abs(res.inv_quad - o64.inv_quad) <= max(1e-4 * abs(o64.inv_quad), 3 * abs(o32.inv_quad - o64.inv_quad))
    assert abs(res.logdet - o64.logdet) <= max(1e-4 * abs(o64.logdet), 3 * abs(o32.logdet - o64.logdet))
    assert rel(sol, o64.solves[:, -1]) <= max(5e-4, 3 * rel(o32.solves[:, -1], o64.solves[:, -1]))
    p.close()


def test_sklearn_and_scipy_third_party_anchor(Plan, cuda_dev):
    """Ground truth that is not this repository's own restatement: scikit-learn's exact log marginal likelihood (dense
    Cholesky, sklearn/gaussian_process/_gpr.py) and scipy's conjugate gradients on the dense K_hat."""
    from scipy.sparse.linalg import cg as scipy_cg
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern

    n, d = 3000, 6
    x, y = om.synthetic_problem(n, d, 3, torch.float32)
    xn, yn = x.double().numpy(), y.double().numpy()
    for kind, ls, osc, nz, sk in (("rbf", 0.9, 1.3, 0.1, ConstantKernel(1.3, "fixed") * RBF(0.9, "fixed")),
                                  ("matern52", 1.4, 0.7, 0.05, ConstantKernel(0.7, "fixed") * Matern(1.4, "fixed", nu=2.5))):
        gpr = GaussianProcessRegressor(kernel=sk, alpha=nz, optimizer=None).fit(xn, yn)
        lml = gpr.log_marginal_likelihood_value_          # log p(y), not divided by n
        Khat = sk(xn) + nz * np.eye(n)
        p = Plan(x.to(cuda_dev)).set_hypers(kind, ls, osc, nz)
        # kernel entries against sklearn's kernel matrix
        rows = p.rows(torch.arange(0, n, 97))
        assert np.abs(rows.double().cpu().numpy() - sk(xn)[::97]).max() < 3e-6
        # a tight CG solve against scipy's CG on the dense matrix
        sol_ref, info = scipy_cg(Khat, yn, rtol=1e-10, maxiter=5000)
        assert info == 0
        lt, piv, _ = p.pivoted_cholesky(50, 1e-3)
        w, _, _ = p.precond_build(lt)
        sol, _, cginfo = p.mbcg(y.to(cuda_dev).unsqueeze(-1), 0, 1e-5, 1000, 20, w)   # fp32 CG stalls near 2e-6 residual
        assert rel(sol[:, 0], torch.from_numpy(sol_ref)) < 1e-3
        # the stochastic MLL against sklearn's exact value: inv_quad is deterministic (tight), log det is SLQ with 10 probes
        pn = om.make_probe_noise(n, 50, 10, 5)
        res, _ = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, 50, 2000, 1e-3, 1e-4, 1000, 30)
        exact_iq = float(yn @ sol_ref)
        exact_ld = float(np.linalg.slogdet(Khat)[1])
        assert relf(res.inv_quad, exact_iq) < 1e-4
        assert relf(res.logdet, exact_ld) < 0.02
        assert lml == pytest.approx(-0.5 * (exact_iq + exact_ld + n * math.log(2 * math.pi)), rel=1e-9)   # sklearn == dense algebra
        assert relf(res.log_prob, lml) < 0.02
        p.close()


def test_inplace_input_update_repacks_the_plan(cuda_dev):
    """operators._get_plan caches plans by buffer address: an in-place update of X (x.copy_(new)) must invalidate the
    packed tiles (the cache is keyed on the tensor version counter)."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    g = torch.Generator().manual_seed(0)
    n, d = 1500, 4
    xa, xb = torch.rand(n, d, generator=g), torch.rand(n, d, generator=g)
    v = torch.randn(n, 3, generator=g)
    xdev = xa.clone().to(cuda_dev)
    k = gp.kernels.ScaleKernel(gp.kernels.RBFKernel()).to(cuda_dev)
    k.base_kernel.lengthscale = 0.7
    k.outputscale = 1.2
    with torch.no_grad(), settings.backend("tcgen05"):
        out_a = k(xdev).matmul(v.to(cuda_dev))
        xdev.copy_(xb.to(cuda_dev))          # same buffer, same shape, new contents
        out_b = k(xdev).matmul(v.to(cuda_dev))
    Ka = ok.kernel_matrix("rbf", xa.double(), xa.double(), 0.7, 1.2, True)
    Kb = ok.kernel_matrix("rbf", xb.double(), xb.double(), 0.7, 1.2, True)
    assert rel(out_a, Ka @ v.double()) < 5e-6
    assert rel(out_b, Kb @ v.double()) < 5e-6      # fails with a stale plan (it would still equal Ka @ v)
    # the same hazard through the training API: set_train_data with new inputs in the same buffer
    gp.operators.clear_plan_cache()


def test_cross_covariance_diagonal(cuda_dev):
    """kernel(x1, x2, diag=True) for x1 != x2 is k(x1_i, x2_i), not the constant outputscale."""
    import gpytorch_b200 as gp

    g = torch.Generator().manual_seed(2)
    x1, x2 = torch.rand(333, 5, generator=g), torch.rand(333, 5, generator=g)
    k = gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=1.5)).to(cuda_dev)
    k.base_kernel.lengthscale = 0.6
    k.outputscale = 2.0
    with torch.no_grad():
        dg = k(x1.to(cuda_dev), x2.to(cuda_dev), diag=True)
        dsame = k(x1.to(cuda_dev), diag=True)
    K = ok.kernel_matrix("matern32", x1.double(), x2.double(), 0.6, 2.0, False)
    assert (dg.double().cpu() - K.diagonal()).abs().max() < 3e-6
    assert torch.allclose(dsame.cpu(), torch.full((333,), 2.0))
    with pytest.raises(RuntimeError):
        with torch.no_grad():
            k(x1.to(cuda_dev), x2[:100].to(cuda_dev), diag=True)


def test_prediction_respects_active_dims(cuda_dev):
    """Posterior mean / variance go through the model's forward on the joint inputs (exact_gp.py:315-322), so kernels with
    active_dims see the same columns at test time as in training."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    g = torch.Generator().manual_seed(5)
    n, m = 1200, 50
    x = torch.rand(n, 5, generator=g)
    y = torch.sin(4 * x[:, 1]) + torch.cos(3 * x[:, 3]) + 0.05 * torch.randn(n, generator=g)
    xt = torch.rand(m, 5, generator=g)
    lik = gp.likelihoods.GaussianLikelihood()
    lik.noise = 0.01

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x.to(cuda_dev), y.to(cuda_dev), lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel(ard_num_dims=2, active_dims=[1, 3]))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    model.covar_module.base_kernel.lengthscale = torch.tensor([0.3, 0.4])
    model.mean_module.constant = 0.2
    model.eval(); lik.eval()
    with torch.no_grad(), settings.eval_cg_tolerance(1e-4), settings.max_preconditioner_size(30):
        pred = model(xt.to(cuda_dev))
    xs, xts = x[:, [1, 3]].double(), xt[:, [1, 3]].double()
    lsv = torch.tensor([0.3, 0.4], dtype=torch.float64)
    K = ok.kernel_matrix("rbf", xs, xs, lsv, 1.0, True) + 0.01 * torch.eye(n, dtype=torch.float64)
    Ks = ok.kernel_matrix("rbf", xts, xs, lsv, 1.0, False)
    Kss = ok.kernel_matrix("rbf", xts, xts, lsv, 1.0, True)
    mean_ref = 0.2 + Ks @ torch.linalg.solve(K, y.double() - 0.2)
    var_ref = (Kss - Ks @ torch.linalg.solve(K, Ks.t())).diagonal()
    assert (pred.mean.double().cpu() - mean_ref).abs().max() < 2e-3
    assert (pred.variance.double().cpu() - var_ref).abs().max() < 2e-3


def test_fixed_noise_likelihood_per_row_diagonal(Plan, cuda_dev):
    """FixedNoiseGaussianLikelihood (likelihoods/gaussian_likelihood.py:245-363): K_hat = K + diag(d) through the device path --
    products, the non-constant-diagonal preconditioner (log det P, P^-1, N(0, P) probes), mBCG and the MLL -- against the oracle's
    per-row branch and dense Cholesky; then the same through the public API with a learned additional noise."""
    n, d, kind, ls, rank = 3000, 5, "rbf", 0.8, 40
    x, y = om.synthetic_problem(n, d, 4, torch.float32)
    g = torch.Generator().manual_seed(3)
    dvec = 0.02 + 0.3 * torch.rand(n, generator=g)                       # heteroscedastic variances in [0.02, 0.32]
    K = ok.kernel_matrix(kind, x.double(), x.double(), ls, 1.3, True)
    p = Plan(x.to(cuda_dev)).set_hypers(kind, ls, 1.3, 0.0).set_noise_diag(dvec.to(cuda_dev))
    v = torch.randn(n, 6, generator=g)
    assert rel(p.kmv(v.to(cuda_dev), add_noise=True), K @ v.double() + dvec.double().unsqueeze(-1) * v.double()) < 5e-6
    # preconditioner of the non-constant diagonal: log det P and P^-1 against the oracle's QR form
    lt, piv, st = p.pivoted_cholesky(rank, 1e-3)
    L, piv_o = ol.pivoted_cholesky(torch.full((n,), 1.3, dtype=torch.float64), lambda i: K[i], rank)
    assert torch.equal(piv.cpu(), piv_o)
    pre = ol.build_preconditioner(L, dvec.double(), piv_o)
    w, logdet_p, st2 = p.precond_build(lt)
    assert st2 == 0 and logdet_p == pytest.approx(pre.logdet, rel=1e-6)
    wd = w.double().cpu()
    r = torch.randn(n, 3, generator=g, dtype=torch.float64)
    assert rel(r / dvec.double().unsqueeze(-1) - wd @ (wd.t() @ r), pre.apply(r)) < 1e-4
    # the MLL with identical probes
    pn = om.make_probe_noise(n, rank, 10, 7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm(kind, x.double(), y.double(), 0.0, ls, 1.3, dvec.double(), tuple(a.double() for a in pn), precond_size=rank, K=K)
        o32 = om.mll_bbmm(kind, x, y, 0.0, ls, 1.3, dvec, pn, precond_size=rank)
    res, sol = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000, want_solve=True)
    assert res.cg_iters == o64.iters
    assert abs(res.inv_quad - o64.inv_quad) <= max(1e-4 * abs(o64.inv_quad), 3 * abs(o32.inv_quad - o64.inv_quad))
    assert abs(res.logdet - o64.logdet) <= max(1e-4 * abs(o64.logdet), 3 * abs(o32.logdet - o64.logdet))
    dense = om.mll_cholesky(kind, x.double(), y.double(), 0.0, ls, 1.3, dvec.double())
    assert abs(res.mll - dense.mll) < 0.02 * abs(dense.mll) + 1e-3
    p.close()
    # public API: FixedNoiseGaussianLikelihood + learned second noise, gradient of the learned noise vs dense autograd
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=dvec.to(cuda_dev), learn_additional_noise=True).to(cuda_dev)
    lik.second_noise = 0.05

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x.to(cuda_dev), y.to(cuda_dev), lik)
            self.mean_module = gp.means.ZeroMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    model.covar_module.base_kernel.lengthscale = ls
    model.covar_module.outputscale = 1.3
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    model.train(); lik.train()
    with settings.max_preconditioner_size(rank), settings.probe_seed(7), settings.cg_tolerance(1e-3), settings.num_trace_samples(15):
        out = mll(model(x.to(cuda_dev)), y.to(cuda_dev))
        out.backward()
    dd = (dvec.double() + 0.05)
    Khat = K + torch.diag(dd)
    Lc = torch.linalg.cholesky(Khat)
    alpha = torch.cholesky_solve(y.double().unsqueeze(-1), Lc)[:, 0]
    exact = -0.5 * (float(y.double() @ alpha) + float(2 * Lc.diagonal().log().sum()) + n * math.log(2 * math.pi)) / n
    assert abs(out.item() - exact) < 0.02 * abs(exact) + 1e-3
    # d mll / d second_noise = 0.5 (alpha^T alpha - tr(Khat^-1)) / n ; chain rule through softplus of the raw parameter
    Kinv_tr = float(torch.cholesky_inverse(Lc).diagonal().sum())
    g_exact = 0.5 * (float(alpha @ alpha) - Kinv_tr) / n
    raw = lik.second_noise_covar.raw_noise
    g_gpu = raw.grad.item() / torch.sigmoid(raw).item()
    assert abs(g_gpu - g_exact) < 0.15 * abs(g_exact) + 1e-3     # stochastic trace estimate, 15 probes


def test_c4_batched_exact_gp_through_api(cuda_dev):
    """BASELINE config 4 shape (batch of independent exact GPs, own hyper-parameters per element, test/examples/
    test_batch_gp_regression.py:72-140): Kernel / ScaleKernel / GaussianLikelihood / ConstantMean with batch_shape, inputs
    [B, n, d], MultivariateNormal.log_prob -> [B].  Elements run concurrently (one engine plan and CUDA stream each); every
    element must equal its own stand-alone evaluation bit for bit, and the oracle within the Krylov tolerance rule."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    B, n, d, rank = 4, 2400, 8, 40
    g = torch.Generator().manual_seed(4)
    X = torch.rand(B, n, d, generator=g)
    Y = torch.sin(2 * X.sum(-1)) + 0.1 * torch.randn(B, n, generator=g)
    ls = torch.tensor([0.8 + 0.2 * i for i in range(B)])
    osc = torch.tensor([1.0 + 0.5 * i for i in range(B)])
    nz = torch.tensor([0.05 * (i + 1) for i in range(B)])
    bs = torch.Size([B])
    lik = gp.likelihoods.GaussianLikelihood(batch_shape=bs).to(cuda_dev)
    lik.noise = nz.unsqueeze(-1)

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(X.to(cuda_dev), Y.to(cuda_dev), lik)
            self.mean_module = gp.means.ConstantMean(batch_shape=bs)
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel(batch_shape=bs), batch_shape=bs)

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    model.covar_module.base_kernel.lengthscale = ls.reshape(B, 1, 1)
    model.covar_module.outputscale = osc
    assert tuple(model.covar_module.base_kernel.raw_lengthscale.shape) == (B, 1, 1)       # kernel.py:213-219
    assert tuple(lik.noise_covar.raw_noise.shape) == (B, 1)
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    model.train(); lik.train()
    with torch.no_grad(), settings.max_preconditioner_size(rank), settings.probe_seed(11):
        out = mll(model(X.to(cuda_dev)), Y.to(cuda_dev))
        out2 = mll(model(X.to(cuda_dev)), Y.to(cuda_dev))
    assert tuple(out.shape) == (B,)
    assert torch.equal(out, out2)                                  # concurrent execution is still deterministic
    # element by element: stand-alone model with the same hyper-parameters and probe seed
    for i in range(B):
        lik1 = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
        lik1.noise = float(nz[i])

        class M1(gp.models.ExactGP):
            def __init__(self):
                super().__init__(X[i].to(cuda_dev), Y[i].to(cuda_dev), lik1)
                self.mean_module = gp.means.ConstantMean()
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

            def forward(self, xx):
                return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

        m1 = M1().to(cuda_dev)
        m1.covar_module.base_kernel.lengthscale = float(ls[i])
        m1.covar_module.outputscale = float(osc[i])
        m1.train(); lik1.train()
        with torch.no_grad(), settings.max_preconditioner_size(rank), settings.probe_seed(11):
            o1 = gp.mlls.ExactMarginalLogLikelihood(lik1, m1)(m1(X[i].to(cuda_dev)), Y[i].to(cuda_dev))
        assert o1.item() == out[i].item()
        dense = om.mll_cholesky("rbf", X[i].double(), Y[i].double(), 0.0, float(ls[i]), float(osc[i]), float(nz[i]))
        assert abs(out[i].item() - dense.mll) < 0.02 * abs(dense.mll) + 2e-3
    # gradients flow to the batched parameters
    with settings.max_preconditioner_size(rank), settings.probe_seed(11):
        loss = -mll(model(X.to(cuda_dev)), Y.to(cuda_dev)).sum()
        loss.backward()
    gl = model.covar_module.base_kernel.raw_lengthscale.grad
    assert gl is not None and tuple(gl.shape) == (B, 1, 1) and torch.isfinite(gl).all() and (gl != 0).all()
    assert lik.noise_covar.raw_noise.grad is not None and torch.isfinite(lik.noise_covar.raw_noise.grad).all()


def test_solver_path_knobs_fast_computations_deterministic_probes_terminate_by_size(cuda_dev):
    """settings.fast_computations(log_prob=False, solves=False) forces the dense Cholesky branch above max_cholesky_size (MLL then
    equals the dense value); deterministic_probes re-uses one set of probes (bit-identical stochastic estimates); terminate_cg_by_size
    caps the iterations at n."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import ConstantDiagLinearOperator, KernelLinearOperator

    n, d = 1500, 3
    x, y = om.synthetic_problem(n, d, 3, torch.float32)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    lik.noise = 0.15

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(xd, yd, lik)
            self.mean_module = gp.means.ZeroMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    model.covar_module.base_kernel.lengthscale = 0.6
    model.covar_module.outputscale = 1.2
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    model.train(); lik.train()
    dense = om.mll_cholesky("rbf", x.double(), y.double(), 0.0, 0.6, 1.2, 0.15).mll
    with torch.no_grad(), settings.fast_computations(log_prob=False, solves=False):
        exact = mll(model(xd), yd).item()
    assert exact == pytest.approx(dense, rel=2e-4, abs=2e-5)
    with torch.no_grad(), settings.deterministic_probes(True):
        a = mll(model(xd), yd).item()
        b = mll(model(xd), yd).item()
    assert a == b and abs(a - dense) < 0.03          # 10 Rademacher probes, no preconditioner at n = 1500: stochastic log-det
    with torch.no_grad():
        c = mll(model(xd), yd).item()
        e = mll(model(xd), yd).item()
    assert c != e                                   # fresh probes every evaluation without the flag
    # terminate_cg_by_size: an unreachable tolerance stops at n iterations instead of max_cg_iterations
    m = 200
    op = KernelLinearOperator(xd[:m].contiguous(), None, "rbf", torch.tensor(0.6, device=cuda_dev), torch.tensor(1.2, device=cuda_dev))
    khat = op + ConstantDiagLinearOperator(torch.tensor(1e-3, device=cuda_dev), m)
    with torch.no_grad(), warnings.catch_warnings(), settings.max_cholesky_size(0), settings.cg_tolerance(1e-12), \
            settings.max_preconditioner_size(0), settings.terminate_cg_by_size(True):
        warnings.simplefilter("ignore")
        khat.inv_quad_logdet(yd[:m].unsqueeze(-1), logdet=True)
    assert khat.last_cg_iters <= m
