"""GPU checks of KISS-GP prediction on the grid: gp_ski_grid_matmul / gp_ski_interp_matmul (csrc/ski.cu) against the fp64 oracle
(oracle/ski_predict.py), and ExactGP with settings.ski_grid_prediction against the joint path and the oracle.

Bounds (u = 2^-24):
* gp_ski_grid_matmul: the SKI product bound of tests/test_gpu_ski.py, per column rel-l2 <= 2e-5 of |s K_uu W^T V|, the oracle in
  fp64 with fp64 interpolation weights (the fp32 grid coordinate and weights of the plan are part of the error).
* gp_ski_interp_matmul: W is the reference's interpolation of the fp32 data (oracle interp_dtype=float32: the same grid
  coordinate (x - u_0) / spacing rounded in fp32, hence the same first nodes as the plan) promoted to fp64.  The kernel sums
  sum_a w_0[a] (sum_b w_1[b] (...)) in fp32: every product of C with its d weights passes through at most 5 d <= 4^d + 2d roundings,
  so |out - W C| <= (4^d + 2d) u (|W| |C|).  The plan's 1-D weights and the reference's fp32 weights evaluate the same cubic
  polynomial of the same fp32 argument in a different rounding order (the compiler may fuse multiply-adds): intermediates are
  below 4 in magnitude and there are at most 6 roundings, so they differ by at most 32 u each; |w| <= 1, and the reference's
  product of d fp32 weights adds d - 1 roundings, so each of the 4^d product weights differs by at most 33 d u: the floor
  33 d u (S |C|), S the support pattern of W.
* LOVE covariance: U = W* C with C from 3xTF32 mode products (fp32 level, ~1e-6 relative) and K** from exact fp32 entries of the
  separable form: |Sigma - Sigma_ref|_ij <= 3e-5 sqrt(D_i D_j), D_i = K**_ii + |U_i|^2 (both terms are bounded by it, K** being
  positive semi-definite).
* CIQ sample covariance: tests/test_gpu_sampling.py's |C_hat - A|_F <= 3 sqrt((|A|_F^2 + tr(A)^2) / S)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mll as om, ski, ski_predict as osp  # noqa: E402

U32 = 2.0 ** -24


def _grid(sizes, bounds):
    axes = ski.create_grid(sizes, bounds, dtype=torch.float32)
    return axes, [float(a[0]) for a in axes], [float(a[1] - a[0]) for a in axes]


def _points(n, d, axes, lo, step, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g)
    x[:20] = torch.tensor(lo) + torch.rand(20, d, generator=g) * torch.tensor(step) * 0.999          # first cell: one-hot
    last = torch.tensor([float(a[-1]) for a in axes])
    x[20:40] = last - (0.001 + 0.998 * torch.rand(20, d, generator=g)) * torch.tensor(step)          # last cell
    # a quarter cell from the first / last node: one-hot on node 0 / node M - 1 (a point exactly on the last node of the fp32
    # linspace can fall outside the engine's fp32 bounds check)
    x[40] = torch.tensor(lo) + 0.25 * torch.tensor(step)
    x[41] = last - 0.25 * torch.tensor(step)
    x[42] = torch.tensor([float(a[3]) for a in axes])
    return x


CASES = [(1, [24]), (2, [20, 16]), (3, [12, 10, 9]), (4, [7, 6, 6, 5])]
TS = [1, 16, 17, 100, 129]


def _lib_call(fn, plan, a, lda, t, out, ldo):
    return fn(plan._h, C.c_void_p(a.data_ptr()), lda, t, C.c_void_p(out.data_ptr()), ldo)


@pytest.mark.parametrize("d,sizes", CASES)
def test_grid_matmul_matches_oracle(cuda_dev, d, sizes):
    from gpytorch_b200.engine import Plan

    n, ls, osc = 3000, 0.35, 1.4
    axes, lo, step = _grid(sizes, [(0.0, 1.0)] * d)
    x = _points(n, d, axes, lo, step, seed=d)
    p = Plan(x.to(cuda_dev)).set_ski(sizes, lo, step).set_hypers("rbf", ls, osc, 0.1)
    M = p.grid_points
    g = torch.Generator().manual_seed(100 + d)
    for t in TS:
        V = torch.randn(n, t + 3, generator=g)
        Vd = V.to(cuda_dev)[:, :t]                                  # ldv = t + 3
        out = torch.full((M, t + 5), float("nan"), device=cuda_dev)
        assert _lib_call(p.lib.gp_ski_grid_matmul, p, Vd, t + 3, t, out, t + 5) == 0
        ref = osp.grid_matmul("rbf", x.double(), [a.double() for a in axes], ls, osc, V[:, :t].double())
        o = out.double().cpu()
        assert torch.isnan(o[:, t:]).all()                          # the padding is not written
        err = (o[:, :t] - ref).norm(dim=0) / ref.norm(dim=0)
        assert float(err.max()) < 2e-5, (t, float(err.max()))
        # the Plan method on contiguous operands (the scatter adds tile blocks with atomics: equal up to their order)
        again = p.ski_grid_matmul(Vd.contiguous()).double().cpu()
        assert float(((again - ref).norm(dim=0) / ref.norm(dim=0)).max()) < 2e-5
    p.close()


@pytest.mark.parametrize("d,sizes", CASES)
def test_interp_matmul_matches_oracle_and_is_deterministic(cuda_dev, d, sizes):
    from gpytorch_b200.engine import Plan

    n = 3000
    axes, lo, step = _grid(sizes, [(0.0, 1.0)] * d)
    x = _points(n, d, axes, lo, step, seed=10 + d)
    p = Plan(x.to(cuda_dev)).set_ski(sizes, lo, step).set_hypers("matern52", 0.3, 1.0, 0.1)
    M = p.grid_points
    idx, val = osp._interp([a.double() for a in axes], x.double(), torch.float32)
    g = torch.Generator().manual_seed(200 + d)
    for t in TS + [32]:
        Cm = torch.randn(M, t + 3, generator=g)
        Cd = Cm.to(cuda_dev)
        out = torch.full((n, t + 2), float("nan"), device=cuda_dev)
        assert _lib_call(p.lib.gp_ski_interp_matmul, p, Cd, t + 3, t, out, t + 2) == 0       # strided: ldc = t + 3, ldo = t + 2
        o = out.double().cpu()
        assert torch.isnan(o[:, t:]).all()
        c64 = Cm[:, :t].double()
        ref = ski.left_interp(idx, val, c64)
        bound = (4 ** d + 2 * d) * U32 * ski.left_interp(idx, val.abs(), c64.abs()) \
            + 33 * d * U32 * ski.left_interp(idx, torch.ones_like(val), c64.abs())
        assert ((o[:, :t] - ref).abs() <= bound).all(), (t, float(((o[:, :t] - ref).abs() / bound).max()))
        # bit-identical: a repeated call, and contiguous operands (float4 staging for full aligned chunks)
        again = p.ski_interp_matmul(Cd[:, :t].contiguous())
        assert torch.equal(again, out[:, :t])
        assert torch.equal(p.ski_interp_matmul(Cd[:, :t].contiguous()), again)
    # the one-hot rows (first / last node): exactly the node's value
    Cm = torch.randn(M, 5, generator=g)
    o = p.ski_interp_matmul(Cm.to(cuda_dev)).cpu()
    for r, node in ((40, 0), (41, M - 1)):
        assert torch.equal(o[r], Cm[node]), r
    # a mean-sized call (t = 1) as a vector
    v = p.ski_interp_matmul(Cm[:, 0].contiguous().to(cuda_dev))
    assert v.shape == (n,) and torch.equal(v, p.ski_interp_matmul(Cm[:, :1].contiguous().to(cuda_dev))[:, 0])
    p.close()


def test_error_codes(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    n, sizes = 500, [16, 16]
    axes, lo, step = _grid(sizes, [(0.0, 1.0)] * 2)
    x = torch.rand(n, 2).to(cuda_dev)
    p = Plan(x).set_ski(sizes, lo, step).set_hypers("rbf", 0.3, 1.0, 0.1)
    V = torch.randn(n, 4, device=cuda_dev)
    G = torch.randn(256, 4, device=cuda_dev)
    out_m = torch.empty(256, 4, device=cuda_dev)
    out_n = torch.empty(n, 4, device=cuda_dev)
    for fn, a, o in ((p.lib.gp_ski_grid_matmul, V, out_m), (p.lib.gp_ski_interp_matmul, G, out_n)):
        assert _lib_call(fn, p, a, 4, 0, o, 4) == _lib.GP_E_SHAPE            # t < 1
        assert _lib_call(fn, p, a, 3, 4, o, 4) == _lib.GP_E_SHAPE            # ld < t
        assert _lib_call(fn, p, a, 4, 4, o, 3) == _lib.GP_E_SHAPE
        assert _lib_call(fn, p, a, 4, 4, o, 4) == _lib.GP_OK
    dense = Plan(x).set_hypers("rbf", 0.3, 1.0, 0.1)                          # not a SKI plan
    assert _lib_call(p.lib.gp_ski_grid_matmul, dense, V, 4, 4, out_m, 4) == _lib.GP_E_STATE
    assert _lib_call(p.lib.gp_ski_interp_matmul, dense, G, 4, 4, out_n, 4) == _lib.GP_E_STATE
    sharded = Plan(x, row_begin=0, row_count=n // 2).set_ski(sizes, lo, step)
    with pytest.raises(RuntimeError):
        sharded.set_hypers("rbf", 0.3, 1.0, 0.1)                              # the SKI backend refuses row shards
    assert _lib_call(p.lib.gp_ski_grid_matmul, sharded, V, 4, 4, out_m, 4) == _lib.GP_E_SHAPE
    assert _lib_call(p.lib.gp_ski_interp_matmul, sharded, G, 4, 4, out_n, 4) == _lib.GP_E_SHAPE
    for q in (p, dense, sharded):
        q.close()


# ---- API ---------------------------------------------------------------------------------------------------------------------
def _model(dev, x, y, kind="rbf", fixed_noise=None, G=24, ls=0.3, os_=1.1, noise=0.2):
    import gpytorch_b200 as gp

    lik = gp.likelihoods.GaussianLikelihood() if fixed_noise is None else gp.likelihoods.FixedNoiseGaussianLikelihood(noise=fixed_noise)
    base = gp.kernels.RBFKernel() if kind == "rbf" else gp.kernels.MaternKernel(nu=2.5)

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(base, grid_size=G, num_dims=x.size(-1),
                                                                                       grid_bounds=[(0.0, 1.0)] * x.size(-1)))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    lik = lik.to(dev)
    model.covar_module.base_kernel.base_kernel.lengthscale = ls
    model.covar_module.outputscale = os_
    model.mean_module.constant = 0.3
    if fixed_noise is None:
        lik.noise = noise
    model.eval(); lik.eval()
    return model, lik


def _hypers(model):
    k = model.covar_module
    return float(k.base_kernel.base_kernel.lengthscale.detach().cpu()), float(k.outputscale.detach().cpu())


@pytest.mark.parametrize("kind,fixed", [("rbf", False), ("matern52", True)])
def test_api_grid_mean_and_love_covariance(cuda_dev, kind, fixed):
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator

    n, m, d, G = 1500, 40, 2, 24
    x, y = om.synthetic_problem(n, d, 8, torch.float32)
    xt = torch.rand(m, d, generator=torch.Generator().manual_seed(2))
    nz = (0.1 + 0.2 * torch.rand(n, generator=torch.Generator().manual_seed(3))) if fixed else None
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), kind, None if nz is None else nz.to(cuda_dev), G)
    xtd = xt.to(cuda_dev)
    rows = []
    fwd = model.forward
    model.forward = lambda xx: rows.append(xx.size(-2)) or fwd(xx)
    with torch.no_grad(), settings.eval_cg_tolerance(1e-5), settings.probe_seed(4):
        joint = model(xtd)
        with settings.ski_grid_prediction(True):
            rows.clear()
            grid = model(xtd)
            assert rows == [n, m, n + m]            # exact mode: grid mean, the joint path's covariance
            with settings.fast_pred_var(True):
                rows.clear()
                love = model(xtd)
                assert rows == [n, m]                # LOVE on the grid: no joint operator
    rel = float((grid.mean - joint.mean).norm() / joint.mean.norm())
    assert rel < 1e-4, rel
    # the joint covariance recomputed: K** - K*x K_hat^-1 Kx* cancels down from the prior's scale s, its SKI products add tile
    # blocks with atomics and its solves stop at a CG tolerance of 1e-5, so two calls agree to ~1e-5 s
    osc_ = float(model.covar_module.outputscale.detach())
    assert float((grid.covariance_matrix - joint.covariance_matrix).abs().max()) <= 2e-4 * osc_
    axes = [a.double() for a in ski.create_grid([G] * d, [(0.0, 1.0)] * d, dtype=torch.float32)]
    ls, osc = _hypers(model)
    R = model._covar_cache.double().cpu()
    noise = nz.double() if fixed else float(lik.noise.detach().cpu())
    ref = osp.interpolated_prediction(kind, x.double(), xt.double(), y.double() - 0.3, axes, ls, osc, noise, R,
                                      interp_dtype=torch.float32)
    rel64 = float(((grid.mean.double().cpu() - 0.3) - ref["mean"]).norm() / ref["mean"].norm())
    assert rel64 < 2e-3, rel64
    op = love.lazy_covariance_matrix
    assert isinstance(op, LowRankUpdatedKernelLinearOperator)
    Dg = ref["Kss"].diagonal() + (ref["U"] ** 2).sum(-1)
    bound = 3e-5 * (Dg.unsqueeze(0) * Dg.unsqueeze(1)).sqrt()
    cov = love.covariance_matrix.double().cpu()
    assert ((cov - ref["covar"]).abs() <= bound).all(), float(((cov - ref["covar"]).abs() / bound).max())
    var = love.variance.double().cpu()
    assert ((var - ref["covar"].diagonal()).abs() <= 3e-5 * Dg).all()


def test_api_ciq_samples_of_the_grid_posterior(cuda_dev):
    from gpytorch_b200 import settings

    n, m, d, G, S = 1200, 64, 2, 20, 4096
    x, y = om.synthetic_problem(n, d, 9, torch.float32)
    xt = torch.rand(m, d, generator=torch.Generator().manual_seed(5))
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), G=G)
    with torch.no_grad(), settings.ski_grid_prediction(True), settings.fast_pred_samples(True), settings.ciq_samples(True), \
            settings.probe_seed(1):
        post = model(xt.to(cuda_dev))
        obs = lik(post)
        torch.manual_seed(3)
        smp = obs.sample(torch.Size([S])).double().cpu() - post.mean.double().cpu()
        Ud = post.lazy_covariance_matrix.U.double().cpu()
    axes = [a.double() for a in ski.create_grid([G] * d, [(0.0, 1.0)] * d, dtype=torch.float32)]
    ls, osc = _hypers(model)
    Kss = osp.dense_covariance("rbf", xt.double(), axes, ls, osc, torch.float32)
    A = Kss - Ud @ Ud.T + float(lik.noise.detach().cpu()) * torch.eye(m, dtype=torch.float64)
    Ch = smp.T @ smp / S
    assert float((Ch - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_api_caches_are_fresh_after_set_train_data_and_train(cuda_dev):
    from gpytorch_b200 import settings

    n, m, d = 1000, 30, 2
    x, y = om.synthetic_problem(n, d, 10, torch.float32)
    xt = torch.rand(m, d, generator=torch.Generator().manual_seed(6)).to(cuda_dev)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), G=20)
    with torch.no_grad(), settings.ski_grid_prediction(True), settings.fast_pred_var(True), settings.eval_cg_tolerance(1e-5), \
            settings.probe_seed(2):
        a = model(xt).mean
        assert model._grid_mean_cache is not None and model._grid_covar_cache is not None
        model.set_train_data(targets=(2 * y - 1).to(cuda_dev), strict=False)
        assert model._grid_mean_cache is None and model._grid_covar_cache is None
        b = model(xt).mean
        with settings.ski_grid_prediction(False):
            b_joint = model(xt).mean
        assert float((b - b_joint).norm() / b_joint.norm()) < 1e-4
        assert float((b - a).norm()) > 1e-2 * float(a.norm())
        model.train(); lik.train()
        assert model._grid_mean_cache is None and model._grid_covar_cache is None
        model.eval(); lik.eval()
        c = model(xt).mean
        with settings.ski_grid_prediction(False):
            c_joint = model(xt).mean
        assert float((c - c_joint).norm() / c_joint.norm()) < 1e-4
        # alpha solved again (CG to 1e-5 on products that add tile blocks with atomics): equal to b up to the solve's accuracy
        assert float((c - b).norm() / b.norm()) < 1e-3


def test_api_out_of_bounds_test_points_raise(cuda_dev):
    from gpytorch_b200 import settings

    x, y = om.synthetic_problem(800, 2, 11, torch.float32)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), G=16)
    xt = torch.rand(10, 2)
    xt[3, 0] = 1.5
    with torch.no_grad(), settings.ski_grid_prediction(True), pytest.raises(RuntimeError, match="out of bounds"):
        model(xt.to(cuda_dev)).mean


def test_api_large_test_set(cuda_dev):
    """N = 4000, d = 2, 64^2 grid, m = 200 000: the mean and LOVE variance complete without an m x m allocation (m^2 fp32 =
    160 GB) and without any forward() call over more than max(N, m) rows; on 500 of the points they agree with the joint path."""
    from gpytorch_b200 import settings

    n, m, d = 4000, 200_000, 2
    x, y = om.synthetic_problem(n, d, 12, torch.float32)
    xt = torch.rand(m, d, generator=torch.Generator().manual_seed(7)).to(cuda_dev)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), G=64, ls=0.15, noise=0.05)
    rows = []
    fwd = model.forward
    model.forward = lambda xx: rows.append(xx.size(-2)) or fwd(xx)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad(), settings.ski_grid_prediction(True), settings.fast_pred_var(True), settings.probe_seed(3):
        post = model(xt)
        mean, var = post.mean, post.variance
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"\nm = {m}: torch peak {peak / 2**20:.0f} MiB, forward rows {rows}")
    assert mean.shape == (m,) and var.shape == (m,) and torch.isfinite(mean).all() and torch.isfinite(var).all()
    assert max(rows) <= max(n, m)
    assert peak <= 1 * 2**30
    sel = torch.randperm(m, generator=torch.Generator().manual_seed(8))[:500].to(cuda_dev)
    U = post.lazy_covariance_matrix.U[sel]
    with torch.no_grad(), settings.fast_pred_var(True), settings.probe_seed(3):
        joint = model(xt[sel])
    assert float((mean[sel] - joint.mean).norm() / joint.mean.norm()) < 1e-4
    scale = float(model.covar_module.outputscale.detach()) + (U ** 2).sum(-1)
    assert ((var[sel] - joint.variance).abs() <= 1e-4 * scale).all()
