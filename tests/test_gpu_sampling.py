"""Sampling on the device: gp_ciq_sqrt_matmul (csrc/minres.cu, multi-shift MINRES) against fp64, and MultivariateNormal.rsample /
sample through the public API (CIQ, Cholesky and Lanczos roots).

Bound of the engine-vs-fp64 comparison (test_ciq_engine_matches_fp64), derived, not tuned.  Let A_q = K_hat + tau_q I and
OUT* = K_hat sum_q w_q A_q^-1 b in fp64 with the same tau, w.  The engine returns fl(K_hat Z), Z = sum_q w_q x_q, where x_q has
the true residual r_q = b - A_q x_q.  Then
    K_hat Z - OUT* = - sum_q w_q K_hat A_q^-1 r_q ,   |K_hat A_q^-1|_2 = max_i lam_i / (lam_i + tau_q) <= 1,
so |K_hat Z - OUT*| <= sum_q w_q |r_q|.  MINRES reports |r_q| through its recurrence, resid_q = |phibar_q| / |b| (resid_out); in
fp32 the true residual departs from the recurrence by the residual gap, which for a Lanczos-based solver stays at
O(u k |A_q| |x_q|) = O(u k kappa_q |b|) per step (Greenbaum 1997); with k <= 200 steps and u = 2^-24 that is g_q = 2e-5 kappa_q'
where kappa_q' = |A_q|/lam_min(A_q), capped at the |b| scale.  The final product adds the fp32 error of one fused K.V plus the
noise term, 1e-5 |K_hat|_2 |Z| (3xTF32 product, Table in DESIGN section 2).  Together, per column:
    |OUT - OUT*| <= |b| sum_q w_q (resid_q + min(1, 2e-5 kappa_q')) + 1e-5 |K_hat|_2 |Z*| .
"""
import ctypes as C
import math
import time
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok, linalg as ol, ski  # noqa: E402
from test_sampling_host import msminres64  # noqa: E402

U32 = 2.0 ** -24


def _kdense(kind, x, ls, os_):
    return ok.kernel_matrix(kind, x.double(), x.double(), ls, os_, True)


def _sqrt_psd(A):
    e, V = torch.linalg.eigh(A)
    return (V * e.clamp_min(0).sqrt()) @ V.T


def _bounds64(A):
    e = torch.linalg.eigvalsh(A)
    return float(e[0]), float(e[-1])


def _case_list():
    # (backend, kind, n, t, Q, noise) -- every value of every axis appears at least once
    return [
        ("tcgen05", "rbf", 64, 1, 1, 0.1), ("simt", "rbf", 64, 16, 8, 1e-2), ("tcgen05", "matern12", 1000, 11, 15, 0.1),
        ("simt", "matern12", 1000, 16, 32, 1.0), ("tcgen05", "matern52", 4099, 16, 15, 1e-2), ("simt", "matern52", 4099, 11, 8, 0.1),
        ("tcgen05", "rbf", 1000, 16, 32, "diag"), ("simt", "matern52", 64, 11, 15, "diag"), ("tcgen05", "matern12", 4099, 1, 32, 1.0),
        ("simt", "rbf", 4099, 1, 1, 1e-2), ("tcgen05", "matern52", 1000, 1, 8, 1.0), ("simt", "matern12", 64, 16, 15, 0.1),
        ("tcgen05", "rbf", 7, 11, 15, 0.1), ("simt", "matern52", 7, 1, 32, 1e-2),
    ]


def _setup(cuda_dev, kind, n, noise, seed, backend="auto", d=3):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g)
    ls, os_ = 0.6, 1.3
    K = _kdense(kind, x, ls, os_)
    p = Plan(x.to(cuda_dev), backend=backend)
    if noise == "diag":
        dv = 0.02 + 0.3 * torch.rand(n, generator=g)
        p.set_hypers(kind, ls, os_, 0.0).set_noise_diag(dv.to(cuda_dev))
        A = K + torch.diag(dv.double())
    else:
        p.set_hypers(kind, ls, os_, noise)
        A = K + float(torch.tensor(noise, dtype=torch.float32)) * torch.eye(n, dtype=torch.float64)
    return p, x, A, g


@pytest.mark.parametrize("backend,kind,n,t,Q,noise", _case_list())
def test_ciq_engine_matches_fp64(cuda_dev, backend, kind, n, t, Q, noise):
    from gpytorch_b200.sampling import contour_quadrature

    p, x, A, g = _setup(cuda_dev, kind, n, noise, seed=n + t + Q, backend=backend)
    lo, hi = _bounds64(A)
    tau, w = contour_quadrature(lo, hi * 1.01, Q)
    b = torch.randn(n, t, generator=g)
    out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, w, tol=1e-6, max_iter=400, warn=False)
    assert torch.isfinite(out).all()
    bd = b.double()
    eye = torch.eye(n, dtype=torch.float64)
    zs = sum(wq * torch.linalg.solve(A + tq * eye, bd) for tq, wq in zip(tau, w))
    ref = A @ zs
    A2 = hi
    res = torch.tensor(info.residual_norms, dtype=torch.float64)   # [Q][t]
    for c in range(t):
        bn = float(bd[:, c].norm())
        gap = sum(wq * (float(res[q, c]) + min(1.0, 2e-5 * (A2 + tq) / (lo + tq))) for q, (tq, wq) in enumerate(zip(tau, w)))
        bound = bn * gap + 1e-5 * A2 * float(zs[:, c].norm())
        err = float((out[:, c].cpu().double() - ref[:, c]).norm())
        assert err <= bound, (c, err, bound, info.iters)
    # the fp64 restatement of the solver reaches the same answer in a comparable number of steps
    if n <= 1000 and t == 1:
        xo, _, it64 = msminres64(A.numpy(), bd[:, 0].numpy(), tau, 1e-6, 400)
        zo = (np.array(w)[:, None] * xo).sum(0)
        assert np.linalg.norm(A.numpy() @ zo - ref[:, 0].numpy()) <= 1e-6 * np.linalg.norm(ref[:, 0].numpy())
        assert info.iters <= 2 * it64 + 10
    p.close()


def test_ciq_zero_column_padding_and_strides(cuda_dev):
    from gpytorch_b200.sampling import contour_quadrature

    n, t = 1000, 11
    p, x, A, g = _setup(cuda_dev, "rbf", n, 0.1, seed=5)
    lo, hi = _bounds64(A)
    tau, w = contour_quadrature(lo, hi * 1.01, 15)
    b = torch.randn(n, t, generator=g)
    b[:, 3] = 0
    bd = b.to(cuda_dev)
    out, info = p.ciq_sqrt_matmul(bd, tau, w, tol=1e-5, max_iter=400)
    assert (out[:, 3] == 0).all()
    assert all(info.residual_norms[q][3] == 0 for q in range(15))
    # padded pitches: the padding of OUT is never written, the values are bit-identical
    bp = torch.full((n, 20), float("nan"), device=cuda_dev)
    bp[:, :t] = bd
    op = torch.full((n, 24), 7.0, device=cuda_dev)
    lib = p.lib
    ta = (C.c_double * 15)(*tau); wa = (C.c_double * 15)(*w)
    it = C.c_int(); rs = (C.c_float * (15 * t))()
    st = lib.gp_ciq_sqrt_matmul(p._h, C.c_void_p(bp.data_ptr()), 20, t, ta, wa, 15, 1e-5, 400, C.c_void_p(op.data_ptr()), 24,
                                C.byref(it), rs)
    assert st == 0
    assert torch.equal(op[:, :t], out)
    assert (op[:, t:] == 7.0).all()
    assert it.value == info.iters
    p.close()


def test_ciq_exhausts_krylov_space_without_nan(cuda_dev):
    """N = 7: after 7 steps the Krylov space is exhausted and every shifted residual is near rounding level.  With tol = 1e-5 the
    loop stops within a few steps of that; with tol = 1e-12 (below fp32 reach) it runs on past the exhausted space -- fp32 Lanczos does not see an exact
    zero beta -- and must stay finite and accurate."""
    from gpytorch_b200.sampling import contour_quadrature

    for noise in (1e-2, 1.0):
        p, x, A, g = _setup(cuda_dev, "matern52", 7, noise, seed=7)
        lo, hi = _bounds64(A)
        tau, w = contour_quadrature(lo, hi * 1.01, 15)
        b = torch.randn(7, 16, generator=g)
        ref = A @ sum(wq * torch.linalg.solve(A + tq * torch.eye(7, dtype=torch.float64), b.double()) for tq, wq in zip(tau, w))
        out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, w, tol=1e-5, max_iter=50)
        assert info.iters <= 7 + 3      # the 7-dimensional space, plus the few steps fp32 rounding costs to reach 1e-5
        assert float((out.cpu().double() - ref).norm() / ref.norm()) < 1e-4
        out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, w, tol=1e-12, max_iter=50, warn=False)
        assert torch.isfinite(out).all()
        assert float((out.cpu().double() - ref).norm() / ref.norm()) < 1e-4
        p.close()


def _model(cuda_dev, x, y, kind="rbf", noise=0.1, ls=0.5, os_=1.2, lik=None):
    import gpytorch_b200 as gp

    lik = lik if lik is not None else gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            base = gp.kernels.RBFKernel() if kind == "rbf" else gp.kernels.MaternKernel(nu=2.5)
            self.covar_module = gp.kernels.ScaleKernel(base)

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    lik = lik.to(cuda_dev)
    model.covar_module.base_kernel.lengthscale = ls
    model.covar_module.outputscale = os_
    model.mean_module.constant = 0.3
    if isinstance(lik, gp.likelihoods.GaussianLikelihood):
        lik.noise = noise
    return model, lik


@pytest.mark.parametrize("n,kind", [(2000, "rbf"), (4099, "matern52")])
def test_rsample_ciq_end_to_end(cuda_dev, n, kind):
    """likelihood(model(x)).rsample with ciq_samples on equals mean + K_hat^{1/2} xi (fp64 eigh) for the same xi."""
    from gpytorch_b200 import settings

    g = torch.Generator().manual_seed(n)
    x = torch.rand(n, 2, generator=g)
    y = torch.randn(n, generator=g)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), kind=kind)
    model.train(); lik.train()
    t0 = time.perf_counter()
    with settings.ciq_samples(True):
        torch.manual_seed(123)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.rsample(torch.Size([16]))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert s.shape == (16, n)
    torch.manual_seed(123)
    xi = torch.randn(n, 16, device=cuda_dev).cpu().double()
    A = _kdense(kind, x, 0.5, 1.2) + float(lik.noise.detach().cpu()) * torch.eye(n, dtype=torch.float64)
    ref = (_sqrt_psd(A) @ xi).T + 0.3
    err = ((s.cpu().double() - ref).norm(dim=-1) / (ref - 0.3).norm(dim=-1)).max().item()
    m, M, infos = dist.lazy_covariance_matrix.last_ciq
    print(f"\nCIQ n={n} {kind}: iters {[i.iters for i in infos]}, m={m:.4g} M={M:.4g}, max rel err {err:.2e}, {wall * 1e3:.1f} ms")
    assert err <= 1e-3


def test_rsample_moments_match_covariance(cuda_dev):
    """N = 64, S = 4096 CIQ samples: |C_hat - K_hat|_F <= 3 sqrt((|K_hat|_F^2 + tr(K_hat)^2) / S) (Wishart variance)."""
    from gpytorch_b200 import settings

    n, S = 64, 4096
    g = torch.Generator().manual_seed(64)
    x = torch.rand(n, 2, generator=g)
    model, lik = _model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev))
    model.train(); lik.train()
    with settings.ciq_samples(True), torch.no_grad():
        torch.manual_seed(5)
        s = lik(model(x.to(cuda_dev))).sample(torch.Size([S])).cpu().double() - 0.3
    A = _kdense("rbf", x, 0.5, 1.2) + float(lik.noise.detach().cpu()) * torch.eye(n, dtype=torch.float64)
    Ch = s.T @ s / S
    assert float((Ch - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_default_paths_cholesky_lanczos_and_posterior(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.sampling import psd_safe_cholesky

    # Cholesky root at n <= max_cholesky_size: samples are L xi with the same xi
    n = 500
    g = torch.Generator().manual_seed(3)
    x = torch.rand(n, 2, generator=g)
    model, lik = _model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev))
    model.train(); lik.train()
    dist = lik(model(x.to(cuda_dev)))
    torch.manual_seed(9)
    s = dist.rsample(torch.Size([5]))
    L = psd_safe_cholesky(dist.lazy_covariance_matrix.to_dense())
    torch.manual_seed(9)
    ref = (L @ torch.randn(n, 5, device=cuda_dev)).T + 0.3
    assert torch.allclose(s, ref, rtol=0, atol=1e-5)
    # ... and with covar_root_decomposition=False at a size above the Cholesky limit
    n2 = 1200
    x2 = torch.rand(n2, 2, generator=g)
    model2, lik2 = _model(cuda_dev, x2.to(cuda_dev), torch.zeros(n2, device=cuda_dev))
    model2.train(); lik2.train()
    with settings.fast_computations(covar_root_decomposition=False):
        dist2 = lik2(model2(x2.to(cuda_dev)))
        torch.manual_seed(4)
        s2 = dist2.rsample(torch.Size([3]))
    L2 = psd_safe_cholesky(dist2.lazy_covariance_matrix.to_dense())
    torch.manual_seed(4)
    assert torch.allclose(s2, (L2 @ torch.randn(n2, 3, device=cuda_dev)).T + 0.3, rtol=0, atol=1e-5)

    # Lanczos root at n = 2000 against the oracle's Lanczos from the same start vector
    n3 = 2000
    x3 = torch.rand(n3, 2, generator=g)
    model3, lik3 = _model(cuda_dev, x3.to(cuda_dev), torch.zeros(n3, device=cuda_dev))
    model3.train(); lik3.train()
    op = lik3(model3(x3.to(cuda_dev))).lazy_covariance_matrix
    init = torch.randn(n3, generator=g)
    R = op._lanczos_root(init.to(cuda_dev)).cpu().double()
    A = _kdense("rbf", x3, 0.5, 1.2) + float(lik3.noise.detach().cpu()) * torch.eye(n3, dtype=torch.float64)
    Qo, To = ol.lanczos_tridiag(lambda v: A @ v, settings.max_root_decomposition_size.value(), init.double().unsqueeze(-1))
    Qo, To = Qo[0], To[0]
    e, V = torch.linalg.eigh(To)
    Ro = Qo @ (V * e.clamp_min(0).sqrt())
    assert float((R @ R.T - Ro @ Ro.T).norm() / (Ro @ Ro.T).norm()) < 1e-3
    # a default-path sample at n = 2000 runs the Lanczos root
    with torch.no_grad():
        assert op.zero_mean_mvn_samples(4).shape == (4, n3)

    # eval-mode posterior: a dense covariance, sampled by its Cholesky factor
    y = torch.sin(3 * x[:, 0]).to(cuda_dev)
    model4, lik4 = _model(cuda_dev, x.to(cuda_dev), y)
    model4.eval(); lik4.eval()
    xt = torch.rand(40, 2, generator=g).to(cuda_dev)
    with torch.no_grad():
        post = model4(xt)
        torch.manual_seed(21)
        sp = post.rsample(torch.Size([8]))
    assert sp.shape == (8, 40)
    Lp = psd_safe_cholesky(post.covariance_matrix)
    torch.manual_seed(21)
    assert torch.allclose(sp, (Lp @ torch.randn(40, 8, device=cuda_dev)).T + post.mean, rtol=0, atol=1e-5)
    # base_samples: the root path, reproducible
    base = torch.randn(6, 40, device=cuda_dev)
    with torch.no_grad():
        sb = post.rsample(base_samples=base)
    assert torch.allclose(sb, (Lp @ base.T).T + post.mean, rtol=0, atol=1e-5)


def test_ciq_other_operators(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import AddedDiagLinearOperator, ConstantDiagLinearOperator

    g = torch.Generator().manual_seed(17)
    # AdditiveKernel
    n = 2000
    x = torch.rand(n, 3, generator=g)
    xd = x.to(cuda_dev)
    k = (gp.kernels.ScaleKernel(gp.kernels.RBFKernel(active_dims=[0, 1])) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))).to(cuda_dev)
    ka, kb = k.kernels
    ka.base_kernel.lengthscale = 0.5; ka.outputscale = 0.9
    kb.base_kernel.lengthscale = 1.3; kb.outputscale = 0.6
    op = AddedDiagLinearOperator(k(xd), ConstantDiagLinearOperator(torch.tensor(0.05, device=cuda_dev), n))
    A = (ok.kernel_matrix("rbf", x[:, :2].double(), x[:, :2].double(), 0.5, 0.9, True)
         + ok.kernel_matrix("matern52", x.double(), x.double(), 1.3, 0.6, True) + float(torch.tensor(0.05)) * torch.eye(n, dtype=torch.float64))
    with settings.ciq_samples(True):
        torch.manual_seed(1)
        s = op.zero_mean_mvn_samples(8)
    torch.manual_seed(1)
    ref = (_sqrt_psd(A) @ torch.randn(n, 8, device=cuda_dev).cpu().double()).T
    assert float(((s.cpu().double() - ref).norm(dim=-1) / ref.norm(dim=-1)).max()) <= 1e-3

    # SKI: GridInterpolationKernel, d = 2, grid 64^2, n = 4000, against the dense operator of oracle/ski.py
    n = 4000
    x = torch.rand(n, 2, generator=g)
    kern = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), grid_size=64, num_dims=2,
                                                                     grid_bounds=[(0.0, 1.0)] * 2)).to(cuda_dev)
    kern.base_kernel.base_kernel.lengthscale = 0.3
    kern.outputscale = 1.1
    sop = AddedDiagLinearOperator(kern(x.to(cuda_dev)), ConstantDiagLinearOperator(torch.tensor(0.1, device=cuda_dev), n))
    lo, step = kern.base_kernel._grid()
    axes = [torch.tensor(l0, dtype=torch.float64) + torch.tensor(s0, dtype=torch.float64) * torch.arange(64, dtype=torch.float64)
            for l0, s0 in zip(lo, step)]
    Ks = ski.ski_matmul("rbf", x.double(), axes, 0.3, float(kern.outputscale.detach().cpu()), torch.eye(n, dtype=torch.float64))
    As = 0.5 * (Ks + Ks.T) + float(torch.tensor(0.1)) * torch.eye(n, dtype=torch.float64)
    with settings.ciq_samples(True):
        torch.manual_seed(2)
        s = sop.zero_mean_mvn_samples(4)
    torch.manual_seed(2)
    ref = (_sqrt_psd(As) @ torch.randn(n, 4, device=cuda_dev).cpu().double()).T
    assert float(((s.cpu().double() - ref).norm(dim=-1) / ref.norm(dim=-1)).max()) <= 1e-3

    # FixedNoiseGaussianLikelihood: per-row noise
    n = 1500
    x = torch.rand(n, 2, generator=g)
    dv = 0.05 + 0.2 * torch.rand(n, generator=g)
    lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=dv.to(cuda_dev))
    model, lik = _model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev), lik=lik)
    model.train(); lik.train()
    with settings.ciq_samples(True):
        torch.manual_seed(3)
        s = lik(model(x.to(cuda_dev))).rsample(torch.Size([4]))
    A = _kdense("rbf", x, 0.5, 1.2) + torch.diag(dv.double())
    s = s.detach()
    torch.manual_seed(3)
    ref = (_sqrt_psd(A) @ torch.randn(n, 4, device=cuda_dev).cpu().double()).T + 0.3
    assert float(((s.cpu().double() - ref).norm(dim=-1) / (ref - 0.3).norm(dim=-1)).max()) <= 1e-3


def test_ciq_batch_matches_single(cuda_dev):
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import (AddedDiagLinearOperator, BatchLinearOperator, ConstantDiagLinearOperator,
                                         KernelLinearOperator)

    B, n = 4, 1200
    g = torch.Generator().manual_seed(4)
    xs = [torch.rand(n, 2, generator=g).to(cuda_dev) for _ in range(B)]
    ops = [AddedDiagLinearOperator(KernelLinearOperator(x, None, "rbf", torch.tensor(0.3 + 0.1 * b, device=cuda_dev),
                                                        torch.tensor(1.0, device=cuda_dev)),
                                   ConstantDiagLinearOperator(torch.tensor(0.1, device=cuda_dev), n)) for b, x in enumerate(xs)]
    bop = BatchLinearOperator(ops)
    with settings.ciq_samples(True):
        torch.manual_seed(8)
        s = bop.zero_mean_mvn_samples(5)
        assert s.shape == (5, B, n)
        torch.manual_seed(8)
        xi = torch.randn(B, n, 5, device=cuda_dev)
        for b in range(B):
            single = ops[b]._ciq_samples(xi[b])[0].t()
            assert torch.equal(s[:, b], single)


def test_ciq_errors(cuda_dev):
    from gpytorch_b200 import NanError, NumericalWarning, settings
    from gpytorch_b200.engine import Plan
    from gpytorch_b200.operators import AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator

    n = 300
    x = torch.rand(n, 2, device=cuda_dev)
    p = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    b = torch.randn(n, 17, device=cuda_dev)
    l0 = p.launches()
    for bb, tau, w in [(b, [0.1], [1.0]), (b[:, :4], [], []), (b[:, :4], [0.1] * 33, [1.0] * 33), (b[:, :4], [-1.0], [1.0]),
                       (b[:, :4], [float("inf")], [1.0]), (b[:, :4], [0.1], [float("nan")])]:
        with pytest.raises(RuntimeError, match="shape"):
            p.ciq_sqrt_matmul(bb, tau, w)
    assert p.launches() == l0
    # non-finite inputs
    xb = x.clone()
    xb[5, 1] = float("nan")
    pb = Plan(xb).set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(NanError):
        pb.ciq_sqrt_matmul(b[:, :4].contiguous(), [0.1, 1.0], [0.5, 0.5])
    # the iteration cap warns
    op = AddedDiagLinearOperator(KernelLinearOperator(x, None, "rbf", torch.tensor(0.5, device=cuda_dev), torch.tensor(1.0, device=cuda_dev)),
                                 ConstantDiagLinearOperator(torch.tensor(0.01, device=cuda_dev), n))
    with settings.ciq_samples(True), settings.max_cg_iterations(2), warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        s = op.zero_mean_mvn_samples(3)
    assert s.shape == (3, n) and torch.isfinite(s).all()
    assert any(issubclass(r.category, NumericalWarning) for r in rec)
    p.close(); pb.close()
