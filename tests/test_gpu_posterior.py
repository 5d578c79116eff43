"""Lazy LOVE posteriors: the low-rank correction of a plan (gp_plan_set_lowrank, csrc/lowrank.cu) and
settings.fast_pred_samples through the public API.

Bounds, derived, not tuned (u = 2^-24, r = rank of U, s K the plan's kernel operator, D its noise):
  * products.  The engine returns the backend's K.V slots plus slot nparts = -fl(U fl(U^T v)).  U^T v is summed in fp32 over
    the <= nc rows one CTA owns (nc = 64 ceil(ceil(n / 64) / (2 * 132))), then in fp64 over the CTAs and rounded to fp32:
    |c - U^T v| <= (nc + 2) u |U|^T |v|.  U c is an r-term fp32 sum: |fl(U c) - U c| <= (r + 1) u |U| |c|.  The finish kernels
    add each slot with one more rounding.  Per column, therefore
        |out - (s K - U U^T + D) v| <= e_K + (r + nc + 4) u | |U| |U|^T |v| | + 4 u (|s K v| + |U U^T v| + |D v|) ,
    with e_K = 1e-5 |s K|_2 |v| for the fused kernels (the 3xTF32 product bound of DESIGN section 2) and, for SKI, the rel-l2
    2e-5 |s K V|_F of tests/test_gpu_ski.py (fp32 interpolation weights, scatter atomics in arbitrary order).
  * entries.  gp_kdiag: the constant s minus an r-term fp32 sum of squares: |err_i| <= (r + 2) u sum_j U_ij^2.  gp_krows: one
    fp32 kernel entry (argument -|z_i - z_j|^2 / 2 in fp32, ex2.approx with relative error 2^-22; SKI: 4^d-term products of
    fp32 weights), bounded by 1e-5 s, plus (r + 2) u (|U| |U|^T)_ij for the correction.
  * CIQ on a low-rank plan: the per-column bound of tests/test_gpu_sampling.py with K_hat = s K - U U^T + D built in fp64 from the
    same fp32 U.
  * mBCG: the true residual of the fp32 solve departs from the recurrence by the residual gap, O(u k kappa |b|) (Greenbaum 1997);
    with k <= 200 that is <= 2e-5 kappa, so |b - A x| / |b| <= resid + min(1, 2e-5 kappa).
  * API, flag on: the lazy covariance and the dense fast_pred_var result share K** (the same krows kernel on the same packing)
    and U (the same engine product); they differ by the rounding of U U^T in two J-term sums (cuBLAS and the engine), at most
    (2 J + 4) u (|U| |U|^T)_ij + 2 u |K**_ij|.  The SLQ
    log-det has the Hutchinson standard deviation sd = sqrt(2 (|log A|_F^2 - sum_i (log A)_ii^2) / T) for T Rademacher probes;
    the test allows 4 sd plus 1e-3 |log det| for the Lanczos quadrature and fp32, and 1e-3 |r^T A^-1 r| at cg_tolerance 1e-5.
  * scale: m = 100 000 test points.  An m x m fp32 matrix would take 40 GB; the lazy path's largest buffers are the CIQ work
    blocks ((4 + 2 Q) m 16 fp32 = 218 MB at Q = 15) and the [m, J] factor, so the device memory it adds stays below 2 GB.
"""
import ctypes as C
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok, linalg as ol, ski  # noqa: E402

U32 = 2.0 ** -24
GP_E_SHAPE, GP_E_STATE = 1, 7


def _nystrom_u(x, z, kind, ls, os_, scale=0.9):
    """U [n, r] with U U^T = scale * K_xz K_zz^-1 K_zx <= s K (a Nystrom approximation): s K - U U^T stays PSD."""
    Kxz = ok.kernel_matrix(kind, x.double(), z.double(), ls, os_)
    Kzz = ok.kernel_matrix(kind, z.double(), z.double(), ls, os_, True) + 1e-6 * torch.eye(z.size(0), dtype=torch.float64)
    L = torch.linalg.cholesky(Kzz)
    return (math.sqrt(scale) * torch.linalg.solve_triangular(L, Kxz.T, upper=False).T).float()


def _rows_per_cta(n):
    return 64 * math.ceil(math.ceil(n / 64) / (2 * 132))


def _make(dev, backend, n, r, seed, noise=0.1, d=3):
    """(plan, sK fp64, U fp32 cpu, D fp64 diag vector, lengthscale / kind info)."""
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g)
    ls, os_ = 0.6, 1.3
    if backend == "sum":
        t1 = Plan(x.to(dev), backend="tcgen05").set_hypers("rbf", ls, os_, 0.0)
        t2 = Plan(x.to(dev), backend="simt").set_hypers("matern52", 1.1, 0.5, 0.0)
        p = Plan(x.to(dev)).set_hypers("rbf", [1.0], 1.0, noise).set_sum([t1, t2])
        sK = ok.kernel_matrix("rbf", x.double(), x.double(), ls, os_, True) + ok.kernel_matrix("matern52", x.double(), x.double(), 1.1, 0.5, True)
        p._keep = (t1, t2)
        z = x[torch.randperm(n, generator=g)[:r]]
        U = _nystrom_u(x, z, "rbf", ls, os_)
    elif backend == "ski":
        axes = ski.create_grid([24, 20, 16], [(0.0, 1.0)] * 3, dtype=torch.float32)
        lo, step = [float(a[0]) for a in axes], [float(a[1] - a[0]) for a in axes]
        p = Plan(x.to(dev)).set_ski([24, 20, 16], lo, step).set_hypers("rbf", ls, os_, noise)
        sK = ski.ski_matmul("rbf", x.double(), [a.double() for a in axes], ls, os_, torch.eye(n, dtype=torch.float64))
        sK = 0.5 * (sK + sK.T)
        e, V = torch.linalg.eigh(sK)
        U = (V[:, -r:] * (0.5 * e[-r:].clamp_min(0)).sqrt()).float()   # U U^T = half the top-r part of K_ski
    else:
        p = Plan(x.to(dev), backend=backend).set_hypers("rbf", ls, os_, noise)
        sK = ok.kernel_matrix("rbf", x.double(), x.double(), ls, os_, True)
        z = x[torch.randperm(n, generator=g)[:r]]
        U = _nystrom_u(x, z, "rbf", ls, os_)
    D = torch.full((n,), float(torch.tensor(noise, dtype=torch.float32)), dtype=torch.float64)
    return p, sK, U, D, g


def _product_bound(sK, U, D, v, r, n, ski_backend):
    Ud, vd = U.double(), v.double()
    corr = (Ud.abs() @ (Ud.abs().T @ vd.abs())).norm(dim=0)
    kv = (sK @ vd).norm(dim=0)
    uuv = (Ud @ (Ud.T @ vd)).norm(dim=0)
    dv = (D.unsqueeze(-1) * vd).norm(dim=0)
    rnd = (r + _rows_per_cta(n) + 4) * U32 * corr + 4 * U32 * (kv + uuv + dv)
    if ski_backend:
        return rnd, 2e-5 * float((sK @ vd).norm())
    return rnd + 1e-5 * float(torch.linalg.matrix_norm(sK, 2)) * vd.norm(dim=0), 0.0


@pytest.mark.parametrize("backend,r", [("tcgen05", 1), ("tcgen05", 100), ("simt", 37), ("simt", 128), ("sum", 64), ("ski", 20)])
def test_kmv_with_lowrank_matches_fp64(cuda_dev, backend, r):
    n, t = 3001, 11
    p, sK, U, D, g = _make(cuda_dev, backend, n, r, seed=r + len(backend))
    v = torch.randn(n, t, generator=g)
    Ug = U.to(cuda_dev)
    p.set_lowrank(Ug)
    A = sK - U.double() @ U.double().T
    for add_noise in (False, True):
        out = p.kmv(v.to(cuda_dev), add_noise=add_noise).cpu().double()
        Dn = D if add_noise else torch.zeros_like(D)
        ref = (A + torch.diag(Dn)) @ v.double()
        col, tot = _product_bound(sK, U, D if add_noise else Dn, v, r, n, backend == "ski")
        err = (out - ref).norm(dim=0)
        if backend == "ski":
            assert float((out - ref).norm()) <= tot + float(col.norm()), (float((out - ref).norm()), tot)
        else:
            assert (err <= col).all(), (err.max().item(), col.min().item())
    # per-row diagonal on a dense plan: the correction and D add
    if backend in ("tcgen05", "simt"):
        dv = 0.05 + 0.3 * torch.rand(n, generator=g)
        p.set_noise_diag(dv.to(cuda_dev))
        out = p.kmv(v.to(cuda_dev), add_noise=True).cpu().double()
        ref = (A + torch.diag(dv.double())) @ v.double()
        col, _ = _product_bound(sK, U, dv.double(), v, r, n, False)
        assert ((out - ref).norm(dim=0) <= col).all()
        p.set_noise_diag(None)


@pytest.mark.parametrize("backend", ["tcgen05", "simt", "sum", "ski"])
def test_kdiag_and_krows_with_lowrank_match_fp64(cuda_dev, backend):
    n, r = 2050, 48
    p, sK, U, D, g = _make(cuda_dev, backend, n, r, seed=7 + len(backend))
    p.set_lowrank(U.to(cuda_dev))
    Ud = U.double()
    A = sK - Ud @ Ud.T
    s = float(sK.diagonal().max())
    dg = p.diag().cpu().double()
    assert ((dg - A.diagonal()).abs() <= 1e-5 * s + (r + 2) * U32 * (Ud ** 2).sum(-1)).all()
    idx = torch.tensor([0, 5, 1999, n - 1, 1024])
    rows = p.rows(idx.to(cuda_dev)).cpu().double()
    bound = 1e-5 * s + (r + 2) * U32 * (Ud.abs()[idx] @ Ud.abs().T)
    assert ((rows - A[idx]).abs() <= bound).all()
    # an out-of-range index gives a NaN row, as without a correction
    bad = p.rows(torch.tensor([n + 3], device=cuda_dev))
    assert torch.isnan(bad).all()


@pytest.mark.parametrize("backend", ["tcgen05", "simt", "sum"])
def test_lowrank_products_are_deterministic_and_clearing_restores_the_plan(cuda_dev, backend):
    n, r, t = 4099, 100, 16
    p, sK, U, D, g = _make(cuda_dev, backend, n, r, seed=11)
    v = torch.randn(n, t, generator=g).to(cuda_dev)
    base = p.kmv(v, add_noise=True)
    base_diag = p.diag() if backend != "sum" else None
    p.set_lowrank(U.to(cuda_dev))
    a = p.kmv(v, add_noise=True)
    b = p.kmv(v, add_noise=True)
    assert torch.equal(a, b)
    # strided right-hand side and output: the same bits, padding untouched
    vp = torch.full((n, 20), float("nan"), device=cuda_dev)
    vp[:, :t] = v
    op = torch.full((n, 24), 7.0, device=cuda_dev)
    assert p.lib.gp_kmv(p._h, C.c_void_p(vp.data_ptr()), 20, t, C.c_void_p(op.data_ptr()), 24, 1) == 0
    assert torch.equal(op[:, :t], a) and (op[:, t:] == 7.0).all()
    # strided U (leading dimension > r) gives the same bits
    Upad = torch.zeros(n, r + 7, device=cuda_dev)
    Upad[:, :r] = U.to(cuda_dev)
    assert p.lib.gp_plan_set_lowrank(p._h, C.c_void_p(Upad.data_ptr()), r + 7, r) == 0
    assert torch.equal(p.kmv(v, add_noise=True), a)
    # clearing: the plan's previous outputs bit for bit (r = 0 with a pointer clears too)
    p.set_lowrank(None)
    assert torch.equal(p.kmv(v, add_noise=True), base)
    p.set_lowrank(U.to(cuda_dev))
    assert p.lib.gp_plan_set_lowrank(p._h, C.c_void_p(Upad.data_ptr()), r + 7, 0) == 0
    assert torch.equal(p.kmv(v, add_noise=True), base)
    if base_diag is not None:
        assert torch.equal(p.diag(), base_diag)


def test_lowrank_refusals_and_limits(cuda_dev):
    from gpytorch_b200.engine import Plan

    n, r = 600, 8
    p, sK, U, D, g = _make(cuda_dev, "tcgen05", n, r, seed=3)
    lib, h = p.lib, p._h
    Ug = U.to(cuda_dev)
    lt = p.pivoted_cholesky(10)[0].contiguous()
    w, _, _ = p.precond_build(lt)
    cu, _, _ = p.ciq_precond_build(lt)
    p.set_lowrank(Ug)
    P = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    k = lt.size(0)
    piv = torch.empty(k, dtype=torch.int64, device=cuda_dev)
    ro = C.c_int()
    dd = C.c_double()
    buf = torch.empty(n, 16, device=cuda_dev)
    e1 = torch.randn(k, 4, device=cuda_dev)
    e2 = torch.randn(n, 4, device=cuda_dev)
    it, js = C.c_int(), C.c_int()
    res = (C.c_float * 16)()
    ta, wa = (C.c_double * 1)(0.1), (C.c_double * 1)(1.0)
    gl, go = (C.c_double * 1)(), C.c_double()
    tmat = torch.zeros(1, 20, 20, device=cuda_dev)
    b = torch.randn(n, 4, device=cuda_dev)
    calls = {
        "pivoted_cholesky": lambda: lib.gp_pivoted_cholesky(h, k, 1e-3, P(buf), P(piv), C.byref(ro)),
        "precond_build": lambda: lib.gp_precond_build(h, P(lt), k, P(buf), C.byref(dd)),
        "precond_probes": lambda: lib.gp_precond_probes(h, P(lt), k, P(e1), P(e2), 4, P(buf)),
        "ciq_precond_build": lambda: lib.gp_ciq_precond_build(h, P(lt), k, P(buf), C.byref(dd)),
        "ciq_sqrt_matmul_precond": lambda: lib.gp_ciq_sqrt_matmul_precond(h, P(b), 4, 4, P(cu), k, ta, wa, 1, 1e-4, 10, P(buf), 16,
                                                                          C.byref(it), res),
        "bilinear_grad": lambda: lib.gp_bilinear_grad(h, P(b), 4, P(b), 4, 4, gl, C.byref(go)),
        "mbcg with W": lambda: lib.gp_mbcg(h, P(b), 4, 4, 1, 1.0, 20, 20, P(w), k, P(buf), 16, P(tmat), C.byref(it), C.byref(js), res),
    }
    l0 = p.launches()
    for name, fn in calls.items():
        assert fn() == GP_E_STATE, name
    assert p.launches() == l0
    # mBCG without W runs
    assert lib.gp_mbcg(h, P(b), 4, 4, 1, 1.0, 20, 20, None, 0, P(buf), 16, P(tmat), C.byref(it), C.byref(js), res) in (0, 4)
    # rank limits: 129 is rejected, 128 accepted
    U129 = torch.randn(n, 129, device=cuda_dev)
    assert lib.gp_plan_set_lowrank(h, P(U129), 129, 129) == GP_E_SHAPE
    assert lib.gp_plan_set_lowrank(h, P(U129), 129, 128) == 0
    assert lib.gp_plan_set_lowrank(h, P(U129), 100, 128) == GP_E_SHAPE   # ldu < r
    assert lib.gp_plan_set_lowrank(h, P(U129), 129, -1) == GP_E_SHAPE
    # non-square and row-sharded plans
    x = torch.rand(n, 3, device=cuda_dev)
    pc = Plan(x, torch.rand(n + 1, 3, device=cuda_dev)).set_hypers("rbf", 0.5, 1.0, 0.0)
    assert pc.lib.gp_plan_set_lowrank(pc._h, P(Ug), r, r) == GP_E_SHAPE
    ps = Plan(x, row_begin=0, row_count=n // 2).set_hypers("rbf", 0.5, 1.0, 0.0)
    assert ps.lib.gp_plan_set_lowrank(ps._h, P(Ug), r, r) == GP_E_SHAPE


def test_solvers_on_a_lowrank_plan_match_fp64(cuda_dev):
    from gpytorch_b200.sampling import contour_quadrature

    n, r = 2500, 60
    p, sK, U, D, g = _make(cuda_dev, "tcgen05", n, r, seed=21, noise=0.05)
    p.set_lowrank(U.to(cuda_dev))
    A = sK - U.double() @ U.double().T + torch.diag(D)
    e = torch.linalg.eigvalsh(A)
    lo, hi = float(e[0]), float(e[-1])
    # CIQ: the per-column bound of test_gpu_sampling.py
    tau, w = contour_quadrature(lo, hi * 1.01, 15)
    b = torch.randn(n, 16, generator=g)
    out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, w, tol=1e-6, max_iter=600, warn=False)
    bd = b.double()
    eye = torch.eye(n, dtype=torch.float64)
    zs = sum(wq * torch.linalg.solve(A + tq * eye, bd) for tq, wq in zip(tau, w))
    ref = A @ zs
    res = torch.tensor(info.residual_norms, dtype=torch.float64)
    for c in range(16):
        gap = sum(wq * (float(res[q, c]) + min(1.0, 2e-5 * (hi + tq) / (lo + tq))) for q, (tq, wq) in enumerate(zip(tau, w)))
        bound = float(bd[:, c].norm()) * gap + 1e-5 * hi * float(zs[:, c].norm())
        assert float((out[:, c].cpu().double() - ref[:, c]).norm()) <= bound, c
    # mBCG without a preconditioner
    rhs = torch.randn(n, 8, generator=g)
    sol, _, mi = p.mbcg(rhs.to(cuda_dev), tolerance=1e-6, max_iter=1000, warn=False)
    kappa = hi / lo
    resid = (rhs.double() - A @ sol.cpu().double()).norm(dim=0) / rhs.double().norm(dim=0)
    for c in range(8):
        assert float(resid[c]) <= mi.residual_norms[c] + min(1.0, 2e-5 * kappa), (c, float(resid[c]), mi.residual_norms[c])
    # Lanczos: the extreme Ritz values against the fp64 Lanczos of the same operator from the same start vector
    init = torch.randn(n, generator=g)
    _, T = p.lanczos(init.to(cuda_dev), 30)
    _, To = ol.lanczos_tridiag(lambda v: A @ v, 30, init.double().unsqueeze(-1))
    ritz = torch.linalg.eigvalsh(T.cpu().double())
    ritz_o = torch.linalg.eigvalsh(To[0])
    assert ritz.numel() == ritz_o.numel()
    # the top Ritz values converge first; fp32 Lanczos with full re-orthogonalisation keeps them to ~1e-5 of |A|
    assert ((ritz[-5:] - ritz_o[-5:]).abs() <= 1e-4 * hi).all()
    assert float(ritz[0]) >= lo - 1e-4 * hi


# ---- API ---------------------------------------------------------------------------------------------------------------------
def _model(dev, x, y, noise=0.1, ls=0.5, os_=1.2, additive=False):
    import gpytorch_b200 as gp

    lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            if additive:
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel()) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))
            else:
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    lik = lik.to(dev)
    if additive:
        a, b = model.covar_module.kernels
        a.base_kernel.lengthscale = ls; a.outputscale = os_
        b.base_kernel.lengthscale = 2 * ls; b.outputscale = 0.3
    else:
        model.covar_module.base_kernel.lengthscale = ls
        model.covar_module.outputscale = os_
    model.mean_module.constant = 0.3
    lik.noise = noise
    model.eval(); lik.eval()
    return model, lik


def _data(n, m, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 2, generator=g)
    y = torch.sin(6 * x[:, 0]) + torch.cos(4 * x[:, 1]) + 0.1 * torch.randn(n, generator=g)
    xs = torch.rand(m, 2, generator=g)
    ys = torch.sin(6 * xs[:, 0]) + torch.cos(4 * xs[:, 1]) + 0.1 * torch.randn(m, generator=g)
    return x, y, xs, ys


@pytest.mark.parametrize("additive", [False, True])
def test_api_fast_pred_samples_covariance_and_variance(cuda_dev, additive):
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator

    x, y, xs, _ = _data(2600, 2000, seed=1 + additive)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), additive=additive)
    xsd = xs.to(cuda_dev)
    with torch.no_grad(), settings.probe_seed(4):
        with settings.fast_pred_var(True):
            dense = model(xsd)
        with settings.fast_pred_samples(True):
            lazy = model(xsd)
    op = lazy.lazy_covariance_matrix
    assert isinstance(op, LowRankUpdatedKernelLinearOperator) and torch.is_tensor(dense.lazy_covariance_matrix)
    assert torch.equal(lazy.mean, dense.mean)
    C_lazy = lazy.covariance_matrix.double().cpu()
    C_dense = dense.covariance_matrix.double().cpu()
    Ud = op.U.double().cpu()
    J = Ud.size(-1)
    bound = (2 * J + 4) * U32 * (Ud.abs() @ Ud.abs().T) + 2 * U32 * (C_dense + Ud @ Ud.T).abs()
    assert ((C_lazy - C_dense).abs() <= bound).all()
    var = lazy.variance.double().cpu()
    assert ((var - C_lazy.diagonal()).abs() <= 2 * U32 * C_lazy.diagonal().abs().clamp_min(1e-3)).all()
    # the flag changes nothing where it does not apply: fast_pred_var alone keeps its dense result
    with torch.no_grad(), settings.probe_seed(4), settings.fast_pred_var(True):
        again = model(xsd)
    assert torch.equal(again.covariance_matrix, dense.covariance_matrix)


def test_api_ciq_samples_logprob_and_lanczos_default(cuda_dev, monkeypatch):
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator, _SamplingMixin

    n, m = 2600, 2000
    x, y, xs, ys = _data(n, m, seed=9)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev))
    xsd = xs.to(cuda_dev)
    with torch.no_grad(), settings.fast_pred_samples(True), settings.probe_seed(2):
        post = model(xsd)
        obs = lik(post)
        op = post.lazy_covariance_matrix
        Ud = op.U.double().cpu()
        K = ok.kernel_matrix("rbf", xs.double(), xs.double(), 0.5, float(model.covar_module.outputscale.detach().cpu()), True)
        s2 = float(lik.noise.detach().cpu())
        A = K - Ud @ Ud.T + s2 * torch.eye(m, dtype=torch.float64)
        # CIQ samples of the observed posterior against the fp64 eigh square root, same xi
        with settings.ciq_samples(True):
            torch.manual_seed(31)
            s = obs.rsample(torch.Size([16]))
        torch.manual_seed(31)
        xi = torch.randn(m, 16, device=cuda_dev).cpu().double()
        e, V = torch.linalg.eigh(A)
        ref = ((V * e.clamp_min(0).sqrt()) @ V.T @ xi).T
        mean = post.mean.double().cpu()
        err = ((s.double().cpu() - mean - ref).norm(dim=-1) / ref.norm(dim=-1)).max().item()
        assert err <= 1e-3, err
        # log_prob(test_y): unpreconditioned mBCG + SLQ on the device against a dense fp64 Cholesky
        T = 15
        with settings.num_trace_samples(T), settings.cg_tolerance(1e-5), settings.eval_cg_tolerance(1e-5), \
                settings.max_lanczos_quadrature_iterations(100):
            lp = float(obs.log_prob(ys.to(cuda_dev)))
        r = ys.double() - mean
        L = torch.linalg.cholesky(A)
        iq = float(r @ torch.cholesky_solve(r.unsqueeze(-1), L).squeeze(-1))
        ld = float(2 * L.diagonal().log().sum())
        lp64 = -0.5 * (iq + ld + m * math.log(2 * math.pi))
        logA = (V * e.log()) @ V.T
        sd = math.sqrt(2 * (float((logA ** 2).sum()) - float((logA.diagonal() ** 2).sum())) / T)
        assert abs(lp - lp64) <= 0.5 * (4 * sd + 1e-3 * abs(ld) + 1e-3 * abs(iq)), (lp, lp64, sd)
        # m > max_cholesky_size without CIQ: the device Lanczos root
        calls = []
        orig = _SamplingMixin._lanczos_root
        monkeypatch.setattr(_SamplingMixin, "_lanczos_root", lambda self, init=None: calls.append(type(self)) or orig(self, init))
        assert m > settings.max_cholesky_size.value()
        sl = obs.rsample(torch.Size([3]))
        assert sl.shape == (3, m) and torch.isfinite(sl).all() and calls
        assert isinstance(op, LowRankUpdatedKernelLinearOperator)


def test_api_sample_covariance_of_the_lazy_posterior(cuda_dev):
    """m = 64 test points, S = 4096 CIQ draws of the observed posterior: |C_hat - A|_F <= 3 sqrt((|A|_F^2 + tr(A)^2) / S)."""
    from gpytorch_b200 import settings

    n, m, S = 800, 64, 4096
    x, y, xs, _ = _data(n, m, seed=13)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev))
    with torch.no_grad(), settings.fast_pred_samples(True), settings.ciq_samples(True), settings.probe_seed(1):
        post = model(xs.to(cuda_dev))
        obs = lik(post)
        torch.manual_seed(3)
        smp = obs.sample(torch.Size([S])).double().cpu() - post.mean.double().cpu()
        Ud = post.lazy_covariance_matrix.U.double().cpu()
    K = ok.kernel_matrix("rbf", xs.double(), xs.double(), 0.5, float(model.covar_module.outputscale.detach().cpu()), True)
    A = K - Ud @ Ud.T + float(lik.noise.detach().cpu()) * torch.eye(m, dtype=torch.float64)
    Ch = smp.T @ smp / S
    assert float((Ch - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_api_large_test_set_allocates_nothing_m_by_m(cuda_dev):
    from gpytorch_b200 import NumericalWarning, settings

    n, m = 500, 100_000
    x, y, xs, _ = _data(n, m, seed=17)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev))
    xsd = xs.to(cuda_dev)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    torch.cuda.reset_peak_memory_stats()
    base, reserved0 = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
    with torch.no_grad(), settings.fast_pred_samples(True), settings.ciq_samples(True), settings.max_cg_iterations(40), \
            warnings.catch_warnings():
        warnings.simplefilter("ignore", NumericalWarning)     # the capped msMINRES may stop above its tolerance
        post = model(xsd)
        var = post.variance
        s = lik(post).rsample(torch.Size([16]))
    torch.cuda.synchronize()
    assert var.shape == (m,) and s.shape == (16, m)
    assert torch.isfinite(var).all() and torch.isfinite(s).all()
    assert (var > -1e-4).all()
    torch_peak = torch.cuda.max_memory_allocated() - base
    engine = max(0, free0 - torch.cuda.mem_get_info()[0] - (torch.cuda.memory_reserved() - reserved0))   # cudaMalloc outside torch
    print(f"\nm = {m}: torch peak {torch_peak / 2**20:.0f} MiB, engine buffers ~{engine / 2**20:.0f} MiB")
    assert torch_peak + engine <= 2 * 2**30


# ---- plan lifetime, stale corrections, gp_mll ------------------------------------------------------------------------------
def test_destroying_lowrank_plans_frees_their_device_memory(cuda_dev):
    """Create, use and close low-rank plans: the device's free memory returns to where it started (the U^T V workspace of one
    plan is 264 x 16 r fp32 + 16 r fp64 = 2.1 MB at r = 128, so five leaked plans would show as > 10 MB)."""
    from gpytorch_b200.engine import Plan

    n, r = 40_000, 128
    g = torch.Generator().manual_seed(2)
    x = torch.rand(n, 3, generator=g).to(cuda_dev)
    U = (0.01 * torch.randn(n, r, generator=g)).to(cuda_dev)
    v = torch.randn(n, 4, generator=g).to(cuda_dev)

    def cycle():
        p = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1).set_lowrank(U)
        out = p.kmv(v, add_noise=True)
        d = p.diag()
        torch.cuda.synchronize()
        del out, d
        p.close()

    cycle()                                   # module loading and first-launch allocations happen here
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        cycle()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 <= 2 * 2**20, (free0 - free1) / 2**20


def test_a_stale_correction_is_refused_after_the_data_changes(cuda_dev):
    from gpytorch_b200.engine import Plan

    n, r = 3000, 16
    g = torch.Generator().manual_seed(5)
    x = torch.rand(n, 3, generator=g).to(cuda_dev)
    U = (0.1 * torch.randn(n, r, generator=g)).to(cuda_dev)
    v = torch.randn(n, 2, generator=g).to(cuda_dev)
    p = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1).set_lowrank(U)
    ref = p.kmv(v)
    lib, h = p.lib, p._h
    P = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    out = torch.empty(n, 2, device=cuda_dev)
    diag = torch.empty(n, device=cuda_dev)
    idx = torch.tensor([0, 7], device=cuda_dev)
    rows = torch.empty(2, n, device=cuda_dev)
    # fewer rows: U [n, r] no longer matches the operator
    assert lib.gp_plan_set_data(h, P(x), n - 10, 3, None, n - 10, 3, 3, 0, 0) == 0
    assert lib.gp_kmv(h, P(v), 2, 2, P(out), 2, 0) == GP_E_STATE
    assert lib.gp_kdiag(h, P(diag)) == GP_E_STATE
    assert lib.gp_krows(h, P(idx), 2, P(rows), n) == GP_E_STATE
    # a row shard of the original size
    assert lib.gp_plan_set_data(h, P(x), n, 3, None, n, 3, 3, 0, n // 2) == 0
    assert lib.gp_kmv(h, P(v), 2, 2, P(out), 2, 0) == GP_E_STATE
    # the same operator again: the correction applies as before
    assert lib.gp_plan_set_data(h, P(x), n, 3, None, n, 3, 3, 0, 0) == 0
    assert lib.gp_kmv(h, P(v), 2, 2, P(out), 2, 0) == 0
    assert torch.equal(out, ref)
    # a U that is not on the plan's device is refused by the binding
    with pytest.raises(RuntimeError, match="device"):
        p.set_lowrank(U.cpu())


def test_mll_on_a_lowrank_plan_runs_unpreconditioned(cuda_dev):
    from oracle import mll as om

    n, r = 3000, 32
    p, sK, U, D, g = _make(cuda_dev, "tcgen05", n, r, seed=41)
    p.set_lowrank(U.to(cuda_dev))
    y = torch.randn(n, generator=g).to(cuda_dev)
    rad = (torch.randint(0, 2, (n, 10), generator=g).float() * 2 - 1).to(cuda_dev)
    eps1, eps2, _ = om.make_probe_noise(n, 15, 10, 3)
    res0, _ = p.mll(y, None, None, rad, 10, 0, 2000, warn=False)
    res1, _ = p.mll(y, eps1.to(cuda_dev), eps2.to(cuda_dev), rad, 10, 15, 2000, warn=False)   # a preconditioner is asked for
    assert res1.precond_rank == 0
    assert (res1.log_prob, res1.cg_iters, res1.logdet) == (res0.log_prob, res0.cg_iters, res0.logdet)
    assert math.isfinite(res1.log_prob)


def test_api_rank_above_128_falls_back_to_dense_love(cuda_dev):
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator

    x, y, xs, _ = _data(1500, 300, seed=23)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), noise=0.01, ls=0.05)
    with torch.no_grad(), settings.fast_pred_samples(True), settings.probe_seed(6):
        with settings.max_root_decomposition_size(150):
            post = model(xs.to(cuda_dev))
            J = model._covar_cache.size(-1)
        assert J > 128, J                                    # the Lanczos cache really is wider than a correction may be
        assert torch.is_tensor(post.lazy_covariance_matrix)  # today's dense LOVE covariance
        model._covar_cache = None
        post = model(xs.to(cuda_dev))                        # the default 100 steps: lazy
        assert isinstance(post.lazy_covariance_matrix, LowRankUpdatedKernelLinearOperator)


@pytest.mark.parametrize("dense_branch", [True, False])
def test_api_latent_posterior_log_prob(cuda_dev, dense_branch):
    """log_prob of the noise-free posterior K** - U U^T (dense Cholesky, or mBCG + SLQ) against fp64 from the engine's own U.
    Test points on a 5 x 5 grid 0.2 apart with lengthscale 0.08 keep K** - U U^T well conditioned (kappa < 1e3), so fp32
    Cholesky / CG lose < 1e-3 relative; SLQ gets the Hutchinson allowance of the header (20 Lanczos steps of the 25-dimensional
    operator at kappa < 1e3 leave a quadrature error far below 1e-3 |log det|)."""
    from gpytorch_b200 import settings

    g = torch.Generator().manual_seed(29)
    x = torch.rand(200, 2, generator=g)
    y = torch.sin(6 * x[:, 0]) + 0.1 * torch.randn(200, generator=g)
    grid = torch.linspace(0.1, 0.9, 5)
    xs = torch.stack(torch.meshgrid(grid, grid, indexing="ij"), -1).reshape(-1, 2)
    ys = torch.sin(6 * xs[:, 0])
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), ls=0.08)
    T = 15
    with torch.no_grad(), settings.fast_pred_samples(True), settings.probe_seed(8), settings.num_trace_samples(T), \
            settings.cg_tolerance(1e-5), settings.max_lanczos_quadrature_iterations(20), \
            settings.max_cholesky_size(800 if dense_branch else 10):
        post = model(xs.to(cuda_dev))
        lp = float(post.log_prob(ys.to(cuda_dev)))
        Ud = post.lazy_covariance_matrix.U.double().cpu()
        mean = post.mean.double().cpu()
    K = ok.kernel_matrix("rbf", xs.double(), xs.double(), 0.08, float(model.covar_module.outputscale.detach().cpu()), True)
    A = K - Ud @ Ud.T
    e, V = torch.linalg.eigh(A)
    assert float(e[-1] / e[0]) < 1e3
    r = ys.double() - mean
    iq = float(r @ torch.linalg.solve(A, r))
    ld = float(e.log().sum())
    lp64 = -0.5 * (iq + ld + 25 * math.log(2 * math.pi))
    tol = 1e-3 * (abs(iq) + abs(ld)) + 1e-3
    if not dense_branch:
        logA = (V * e.log()) @ V.T
        tol += 0.5 * 4 * math.sqrt(2 * (float((logA ** 2).sum()) - float((logA.diagonal() ** 2).sum())) / T)
    assert abs(lp - lp64) <= tol, (lp, lp64, tol)
