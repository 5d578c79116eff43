"""The preconditioned CIQ sampler on the device: gp_ciq_precond_build (csrc/pivchol.cu) and gp_ciq_sqrt_matmul_precond
(csrc/minres.cu) against fp64 with the engine's own L and U, and settings.ciq_preconditioner through the public API.

Bound of the factor test (test_precond_build_matches_fp64).  With W = I - U U^T and Pw = D^-1/2 P D^-1/2 = I + M M^T, the fp64
factor W0 satisfies W0 Pw W0 = I, so for the engine's W = W0 + dW
    |W Pw W - I|_2 <= 2 |dW|_2 |Pw|_2^1/2 + |dW|_2^2 |Pw|_2      (|W0 Pw|_2 = |Pw|_2^1/2).
dW has two sources: fp32 storage of U, |dW| <= 2 u |U|_F^2 <= 2 u k (U U^T <= I), and the fp32 Gram chunks (<= 64 terms each, fp64
across chunks), a relative error <= 64 u of G = M^T M; W depends on G through s -> s h(s)^2, and a relative change eps of s moves
1 - s h(s)^2 = (1 + s)^-1/2 by eps s / (2 (1 + s)^3/2) <= eps / 2.  So |dW| <= eta = u (2 k + 32), u = 2^-24.

Bound of the product test (test_ciq_precond_engine_matches_fp64), as test_gpu_sampling.py derives its own with A = F^-1 K_hat F^-T
in place of K_hat.  OUT* = K_hat F^-T sum_q w_q (A + tau_q I)^-1 b = F A sum_q w_q (A + tau_q I)^-1 b; with the true residuals r_q
of A's shifted systems, OUT - OUT* = F sum_q w_q A (A + tau_q I)^-1 r_q, |A (A + tau_q I)^-1|_2 <= 1, so per column
    |OUT - OUT*| <= |F|_2 |b| sum_q w_q (resid_q + min(1, 2e-5 kappa_q')) + 1e-5 |K_hat|_2 |F^-T Z*| ,
kappa_q' = (lam_max(A) + tau_q) / (lam_min(A) + tau_q), |F|_2 = max(d)^1/2 / lam_min(I - U U^T)."""
import ctypes as C
import math
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok  # noqa: E402
from test_gpu_sampling import _model, _sqrt_psd  # noqa: E402
from test_sampling_host import msminres64  # noqa: E402

U32 = 2.0 ** -24


def _setup(cuda_dev, kind, n, noise, seed, backend="auto", k=15, tol=1e-3):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g)
    ls, os_ = 0.6, 1.3
    K = ok.kernel_matrix(kind, x.double(), x.double(), ls, os_, True)
    p = Plan(x.to(cuda_dev), backend=backend)
    if noise == "diag":
        dv = (0.02 + 0.3 * torch.rand(n, generator=g)).double()
        p.set_hypers(kind, ls, os_, 0.0).set_noise_diag(dv.float().to(cuda_dev))
        d = dv.float().double()
    else:
        p.set_hypers(kind, ls, os_, noise)
        d = torch.full((n,), float(torch.tensor(noise, dtype=torch.float32)), dtype=torch.float64)
    lt, _, st = p.pivoted_cholesky(k, tol)
    assert st == 0
    return p, K, d, lt, g


def _factor64(K, d, lt, u, dev):
    """fp64 (on the device) F^-T, A, |F|_2 from the engine's L and U."""
    n = K.shape[0]
    L = lt.double().t()
    U = u.double()
    dd = d.to(dev)
    W = torch.eye(n, dtype=torch.float64, device=dev) - U @ U.T
    finv_t = W / dd.sqrt()[:, None]                           # F^-T = D^-1/2 (I - U U^T)
    Khat = K.to(dev) + torch.diag(dd)
    A = finv_t.T @ Khat @ finv_t
    A = 0.5 * (A + A.T)
    smax = float(torch.linalg.matrix_norm(U, 2))
    fnorm = math.sqrt(float(dd.max())) / (1.0 - smax * smax)
    return L, W, finv_t, Khat, A, fnorm


@pytest.mark.parametrize("kind,n,k,noise,tol", [
    ("matern12", 4099, 1, 0.05, 0.0), ("matern12", 4099, 15, "diag", 0.0), ("matern12", 2000, 64, 0.05, 0.0),
    ("matern12", 4099, 100, "diag", 0.0), ("matern12", 1000, 128, 1e-2, 0.0), ("matern52", 3000, 128, "diag", 0.0),
    ("rbf", 4099, 128, 0.05, 0.5)])                           # the last one stops early
def test_precond_build_matches_fp64(cuda_dev, kind, n, k, noise, tol):
    p, K, d, lt, g = _setup(cuda_dev, kind, n, noise, seed=n + k, k=k, tol=tol)
    kk = lt.size(0)
    if tol > 0:
        assert kk < k
    else:
        assert kk == k
    u, tr_e, st = p.ciq_precond_build(lt)
    assert st == 0 and u.shape == (n, kk) and torch.isfinite(u).all()
    _check_factor(cuda_dev, K, d, lt, u, tr_e, n * float(np.float32(1.3)))
    p.close()


def _check_factor(dev, K, d, lt, u, tr_e, tr_k):
    """tr_k: n times the engine's fp32 outputscale (sum), the diagonal gp_ciq_precond_build sums"""
    L, W, _, _, _, _ = _factor64(K, d, lt, u, dev)
    dd = d.to(dev)
    Pw = (L @ L.T) / dd.sqrt()[:, None] / dd.sqrt()[None, :] + torch.eye(K.shape[0], dtype=torch.float64, device=dev)
    err = float(torch.linalg.matrix_norm(W @ Pw @ W - torch.eye(K.shape[0], dtype=torch.float64, device=dev), 2))
    npw = float(torch.linalg.matrix_norm(Pw, 2))
    eta = U32 * (2 * L.shape[1] + 32)
    bound = 2 * eta * math.sqrt(npw) + eta * eta * npw
    print(f"\nk={L.shape[1]}: |W Pw W - I| {err:.3g} bound {bound:.3g} (|Pw| {npw:.3g})")
    assert err <= bound
    tr_ref = tr_k - float((lt.double() ** 2).sum())
    assert abs(tr_e - tr_ref) <= 1e-9 * tr_k


def test_precond_build_kernel_sum(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200.operators import AddedDiagLinearOperator, ConstantDiagLinearOperator

    n = 3000
    g = torch.Generator().manual_seed(11)
    x = torch.rand(n, 3, generator=g)
    k = (gp.kernels.ScaleKernel(gp.kernels.RBFKernel(active_dims=[0, 1])) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=0.5))).to(cuda_dev)
    ka, kb = k.kernels
    ka.base_kernel.lengthscale = 0.5; ka.outputscale = 0.9
    kb.base_kernel.lengthscale = 1.3; kb.outputscale = 0.6
    op = AddedDiagLinearOperator(k(x.to(cuda_dev)), ConstantDiagLinearOperator(torch.tensor(0.05, device=cuda_dev), n))
    K = (ok.kernel_matrix("rbf", x[:, :2].double(), x[:, :2].double(), 0.5, 0.9, True)
         + ok.kernel_matrix("matern12", x.double(), x.double(), 1.3, 0.6, True))
    plan = op._plan()
    lt, _, st = plan.pivoted_cholesky(64, 0.0)
    assert st == 0 and lt.size(0) == 64
    u, tr_e, st = plan.ciq_precond_build(lt)
    assert st == 0
    _check_factor(cuda_dev, K, torch.full((n,), float(torch.tensor(0.05)), dtype=torch.float64), lt, u, tr_e,
                  n * (float(ka.outputscale.detach()) + float(kb.outputscale.detach())))


def _cases():
    # (backend, kind, n, t, Q, noise, k): every value of every axis at least once
    return [
        ("tcgen05", "rbf", 64, 1, 1, 0.1, 15), ("simt", "matern12", 1000, 11, 8, "diag", 64),
        ("tcgen05", "matern52", 4099, 16, 15, 1e-2, 100), ("simt", "rbf", 4099, 1, 32, "diag", 15),
        ("tcgen05", "matern12", 1000, 16, 32, 1.0, 128), ("simt", "matern52", 64, 11, 15, 0.1, 64),
        ("tcgen05", "rbf", 1000, 1, 15, "diag", 100), ("simt", "matern52", 1000, 16, 8, 1e-2, 1),
    ]


@pytest.mark.parametrize("backend,kind,n,t,Q,noise,k", _cases())
def test_ciq_precond_engine_matches_fp64(cuda_dev, backend, kind, n, t, Q, noise, k):
    from gpytorch_b200.sampling import contour_quadrature

    p, K, d, lt, g = _setup(cuda_dev, kind, n, noise, seed=n + t + Q, backend=backend, k=k)
    u, tr_e, st = p.ciq_precond_build(lt)
    assert st == 0
    m, M = 0.5, 2.0 * (1.0 + max(tr_e, 1e-6 * float(K.trace())) / float(d.min()))
    tau, w = contour_quadrature(m, M, Q)
    b = torch.randn(n, t, generator=g)
    out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, w, tol=1e-6, max_iter=400, warn=False, precond_u=u)
    assert torch.isfinite(out).all() and info.precond_rank == lt.size(0)
    L, W, finv_t, Khat, A, fnorm = _factor64(K, d, lt, u, cuda_dev)
    e, V = torch.linalg.eigh(A)
    lo, hi = float(e[0]), float(e[-1])
    assert 0.5 <= lo and hi <= M
    bd = b.double().to(cuda_dev)
    filt = sum(wq / (e + tq) for tq, wq in zip(tau, w))
    zs = V @ (filt[:, None] * (V.T @ bd))
    fz = finv_t @ zs
    ref = Khat @ fz
    nk = float(torch.linalg.matrix_norm(Khat, 2))
    res = torch.tensor(info.residual_norms, dtype=torch.float64)
    outd = out.double()
    for c in range(t):
        gap = sum(wq * (float(res[q, c]) + min(1.0, 2e-5 * (hi + tq) / (lo + tq))) for q, (tq, wq) in enumerate(zip(tau, w)))
        bound = fnorm * float(bd[:, c].norm()) * gap + 1e-5 * nk * float(fz[:, c].norm())
        err = float((outd[:, c] - ref[:, c]).norm())
        assert err <= bound, (c, err, bound, info.iters)
    xo, _, it64 = msminres64(A.cpu().numpy(), bd[:, 0].cpu().numpy(), tau, 1e-6, 400)
    assert info.iters <= 2 * it64 + 10, (info.iters, it64)
    if kind == "matern52" and n == 4099 and noise == 1e-2:
        lo_k, hi_k = (float(v) for v in torch.linalg.eigvalsh(Khat)[[0, -1]])
        tau0, w0 = contour_quadrature(lo_k, hi_k * 1.01, Q)
        _, info0 = p.ciq_sqrt_matmul(b.to(cuda_dev), tau0, w0, tol=1e-6, max_iter=400, warn=False)
        print(f"\nN=4099 Matern-5/2 sigma^2=1e-2, k={lt.size(0)}: {info.iters} iterations preconditioned, {info0.iters} without "
              f"(kappa(A) {hi / lo:.3g}, kappa(K_hat) {hi_k / lo_k:.3g})")
        assert info.iters < info0.iters
    p.close()


def test_ciq_precond_zero_columns_strides_and_repeats(cuda_dev):
    from gpytorch_b200.sampling import contour_quadrature

    n, t = 1000, 11
    p, K, d, lt, g = _setup(cuda_dev, "rbf", n, 0.1, seed=5, k=30)
    u, tr_e, _ = p.ciq_precond_build(lt)
    k = u.size(1)
    tau, w = contour_quadrature(0.5, 2.0 * (1.0 + tr_e / 0.1), 15)
    b = torch.randn(n, t, generator=g)
    b[:, 3] = 0
    bd = b.to(cuda_dev)
    out, info = p.ciq_sqrt_matmul(bd, tau, w, tol=1e-5, max_iter=400, precond_u=u)
    assert (out[:, 3] == 0).all()
    assert all(info.residual_norms[q][3] == 0 for q in range(15))
    out2, info2 = p.ciq_sqrt_matmul(bd, tau, w, tol=1e-5, max_iter=400, precond_u=u)
    assert torch.equal(out, out2) and info2.iters == info.iters
    bp = torch.full((n, 20), float("nan"), device=cuda_dev)
    bp[:, :t] = bd
    op = torch.full((n, 24), 7.0, device=cuda_dev)
    ta = (C.c_double * 15)(*tau); wa = (C.c_double * 15)(*w)
    it = C.c_int(); rs = (C.c_float * (15 * t))()
    st = p.lib.gp_ciq_sqrt_matmul_precond(p._h, C.c_void_p(bp.data_ptr()), 20, t, C.c_void_p(u.data_ptr()), k, ta, wa, 15, 1e-5,
                                          400, C.c_void_p(op.data_ptr()), 24, C.byref(it), rs)
    assert st == 0
    assert torch.equal(op[:, :t], out)
    assert (op[:, t:] == 7.0).all()
    assert it.value == info.iters
    p.close()


def _fp64_precond_sample(op, K, d, xi):
    """F A^{1/2} xi in fp64 with F from the operator's cached L (U rebuilt in fp64 from that L)."""
    lt = op._preconditioner()[1]
    L = lt.double().cpu().t()
    M = L / d.sqrt()[:, None]
    s, V = torch.linalg.eigh(M.T @ M)
    r1 = (1 + s.clamp_min(0)).sqrt()
    U = (M @ V) / (r1 * (1 + r1)).sqrt()[None, :]
    n = K.shape[0]
    W = torch.eye(n, dtype=torch.float64) - U @ U.T
    finv_t = W / d.sqrt()[:, None]
    Khat = K + torch.diag(d)
    A = finv_t.T @ Khat @ finv_t
    F = torch.linalg.solve(W, torch.diag(d.sqrt())).T         # F = D^1/2 W^-1  (W symmetric)
    return F @ (_sqrt_psd(0.5 * (A + A.T)) @ xi)


@pytest.mark.parametrize("n,kind", [(2000, "rbf"), (4099, "matern52")])
def test_rsample_ciq_precond_end_to_end(cuda_dev, n, kind, monkeypatch):
    from gpytorch_b200 import settings
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(n)
    x = torch.rand(n, 2, generator=g)
    y = torch.randn(n, generator=g)
    model, lik = _model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), kind=kind)
    model.train(); lik.train()
    calls = []
    orig = Plan.lanczos
    monkeypatch.setattr(Plan, "lanczos", lambda self, *a, **kw: calls.append(1) or orig(self, *a, **kw))
    with settings.ciq_samples(True), settings.ciq_preconditioner(True):
        torch.manual_seed(123)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.rsample(torch.Size([16]))
    assert not calls
    op = dist.lazy_covariance_matrix
    m, M, infos = op.last_ciq
    assert all(i.precond_rank > 0 for i in infos) and m == 0.5
    torch.manual_seed(123)
    xi = torch.randn(n, 16, device=cuda_dev).cpu().double()
    noise = float(lik.noise.detach().cpu())
    K = ok.kernel_matrix(kind, x.double(), x.double(), 0.5, 1.2, True)
    ref = _fp64_precond_sample(op, K, torch.full((n,), noise, dtype=torch.float64), xi).T + 0.3
    err = ((s.detach().cpu().double() - ref).norm(dim=-1) / (ref - 0.3).norm(dim=-1)).max().item()
    print(f"\nCIQ precond n={n} {kind}: k={infos[0].precond_rank} iters {[i.iters for i in infos]}, M={M:.4g}, max rel err {err:.2e}")
    assert err <= 1e-3


def test_rsample_precond_moments_match_covariance(cuda_dev):
    from gpytorch_b200 import settings

    n, S = 64, 4096
    g = torch.Generator().manual_seed(64)
    x = torch.rand(n, 2, generator=g)
    model, lik = _model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev))
    model.train(); lik.train()
    with settings.ciq_samples(True), settings.ciq_preconditioner(True), settings.min_preconditioning_size(0), torch.no_grad():
        torch.manual_seed(5)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.sample(torch.Size([S])).cpu().double() - 0.3
        assert dist.lazy_covariance_matrix.last_ciq[2][0].precond_rank > 0
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 0.5, 1.2, True) + float(lik.noise.detach().cpu()) * torch.eye(n, dtype=torch.float64)
    Ch = s.T @ s / S
    assert float((Ch - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_flag_is_inert_where_no_preconditioner_applies(cuda_dev, monkeypatch):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.engine import Plan
    from gpytorch_b200.operators import AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator

    g = torch.Generator().manual_seed(23)

    def both(make, num=4, exact=True):
        op = make()
        outs = []
        for flag in (False, True):
            with settings.ciq_samples(True), settings.ciq_preconditioner(flag):
                torch.manual_seed(7)
                outs.append(op.zero_mean_mvn_samples(num))
                assert all(i.precond_rank == 0 for i in op.last_ciq[2])
        if exact:
            assert torch.equal(outs[0], outs[1])
        else:   # same path, but the SKI product is not bit-reproducible from call to call: agreement to the solver's accuracy
            assert float(((outs[0] - outs[1]).norm(dim=-1) / outs[0].norm(dim=-1)).max()) <= 1e-3

    calls = []
    orig = Plan.pivoted_cholesky
    monkeypatch.setattr(Plan, "pivoted_cholesky", lambda self, *a, **kw: calls.append(1) or orig(self, *a, **kw))

    n = 3000
    x = torch.rand(n, 2, generator=g).to(cuda_dev)
    ls, os_ = torch.tensor(0.4, device=cuda_dev), torch.tensor(1.0, device=cuda_dev)
    noise = ConstantDiagLinearOperator(torch.tensor(0.1, device=cuda_dev), n)
    both(lambda: KernelLinearOperator(x, None, "rbf", ls, os_))                                   # prior without noise
    small = x[:1500]
    both(lambda: AddedDiagLinearOperator(KernelLinearOperator(small, None, "rbf", ls, os_),
                                         ConstantDiagLinearOperator(torch.tensor(0.1, device=cuda_dev), 1500)))   # n < 2000
    with settings.max_preconditioner_size(0):
        both(lambda: AddedDiagLinearOperator(KernelLinearOperator(x, None, "rbf", ls, os_), noise))
    kern = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), grid_size=64, num_dims=2,
                                                                     grid_bounds=[(0.0, 1.0)] * 2)).to(cuda_dev)
    kern.base_kernel.base_kernel.lengthscale = 0.3
    both(lambda: AddedDiagLinearOperator(kern(x), noise), exact=False)                            # SKI
    assert not calls


def test_ciq_precond_other_operators(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import (AddedDiagLinearOperator, BatchLinearOperator, ConstantDiagLinearOperator,
                                         KernelLinearOperator)

    g = torch.Generator().manual_seed(29)
    # AdditiveKernel
    n = 2500
    x = torch.rand(n, 3, generator=g)
    k = (gp.kernels.ScaleKernel(gp.kernels.RBFKernel(active_dims=[0, 1])) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))).to(cuda_dev)
    ka, kb = k.kernels
    ka.base_kernel.lengthscale = 0.5; ka.outputscale = 0.9
    kb.base_kernel.lengthscale = 1.3; kb.outputscale = 0.6
    op = AddedDiagLinearOperator(k(x.to(cuda_dev)), ConstantDiagLinearOperator(torch.tensor(0.05, device=cuda_dev), n))
    K = (ok.kernel_matrix("rbf", x[:, :2].double(), x[:, :2].double(), 0.5, 0.9, True)
         + ok.kernel_matrix("matern52", x.double(), x.double(), 1.3, 0.6, True))
    with settings.ciq_samples(True), settings.ciq_preconditioner(True):
        torch.manual_seed(1)
        s = op.zero_mean_mvn_samples(8)
    assert op.last_ciq[2][0].precond_rank > 0
    torch.manual_seed(1)
    xi = torch.randn(n, 8, device=cuda_dev).cpu().double()
    ref = _fp64_precond_sample(op, K, torch.full((n,), float(torch.tensor(0.05)), dtype=torch.float64), xi).T
    assert float(((s.cpu().double() - ref).norm(dim=-1) / ref.norm(dim=-1)).max()) <= 1e-3

    # FixedNoiseGaussianLikelihood: per-row noise
    n = 2200
    x = torch.rand(n, 2, generator=g)
    dv = 0.05 + 0.2 * torch.rand(n, generator=g)
    lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=dv.to(cuda_dev))
    model, lik = _model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev), lik=lik)
    model.train(); lik.train()
    with settings.ciq_samples(True), settings.ciq_preconditioner(True):
        torch.manual_seed(3)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.rsample(torch.Size([4])).detach()
    fop = dist.lazy_covariance_matrix
    assert fop.last_ciq[2][0].precond_rank > 0
    torch.manual_seed(3)
    xi = torch.randn(n, 4, device=cuda_dev).cpu().double()
    ref = _fp64_precond_sample(fop, ok.kernel_matrix("rbf", x.double(), x.double(), 0.5, 1.2, True), dv.float().double(), xi).T + 0.3
    assert float(((s.cpu().double() - ref).norm(dim=-1) / (ref - 0.3).norm(dim=-1)).max()) <= 1e-3

    # a batch of 4 matches per-element calls
    B, n = 4, 2100
    xs = [torch.rand(n, 2, generator=g).to(cuda_dev) for _ in range(B)]
    ops = [AddedDiagLinearOperator(KernelLinearOperator(xb, None, "rbf", torch.tensor(0.3 + 0.1 * b, device=cuda_dev),
                                                        torch.tensor(1.0, device=cuda_dev)),
                                   ConstantDiagLinearOperator(torch.tensor(0.1, device=cuda_dev), n)) for b, xb in enumerate(xs)]
    bop = BatchLinearOperator(ops)
    with settings.ciq_samples(True), settings.ciq_preconditioner(True):
        torch.manual_seed(8)
        s = bop.zero_mean_mvn_samples(5)
        assert s.shape == (5, B, n)
        torch.manual_seed(8)
        xi = torch.randn(B, n, 5, device=cuda_dev)
        for b in range(B):
            single = ops[b]._ciq_samples(xi[b])
            assert single[1][0].precond_rank > 0
            assert torch.equal(s[:, b], single[0].t())


def test_ciq_precond_errors(cuda_dev):
    from gpytorch_b200 import NanError, NumericalWarning, settings
    from gpytorch_b200.engine import Plan
    from gpytorch_b200.operators import AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator

    n = 300
    x = torch.rand(n, 2, device=cuda_dev)
    p = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    lt, _, _ = p.pivoted_cholesky(10, 0.0)
    u, _, _ = p.ciq_precond_build(lt)
    b = torch.randn(n, 4, device=cuda_dev)
    ta = (C.c_double * 2)(0.1, 1.0); wa = (C.c_double * 2)(0.5, 0.5)
    it = C.c_int(); rs = (C.c_float * 8)()
    out = torch.empty(n, 4, device=cuda_dev)

    def call(plan, uu, k):
        return plan.lib.gp_ciq_sqrt_matmul_precond(plan._h, C.c_void_p(b.data_ptr()), 4, 4, C.c_void_p(uu), k, ta, wa, 2, 1e-4, 100,
                                                  C.c_void_p(out.data_ptr()), 4, C.byref(it), rs)

    from gpytorch_b200 import _lib
    p0 = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)                 # noise 0
    ps = Plan(x, row_begin=0, row_count=n // 2).set_hypers("rbf", 0.5, 1.0, 0.1)   # row-sharded
    l0 = [q.launches() for q in (p, p0, ps)]
    big = torch.zeros(n, 129, device=cuda_dev)
    for uu, k in [(u.data_ptr(), 0), (big.data_ptr(), 129), (0, 10)]:
        assert call(p, uu, k) == _lib.GP_E_SHAPE
    assert call(p0, u.data_ptr(), 10) == _lib.GP_E_SHAPE
    for bad in (0, 129):
        with pytest.raises(RuntimeError, match="shape"):
            p.ciq_precond_build(torch.zeros(bad, n, device=cuda_dev) if bad else torch.zeros(0, n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="shape"):
        p0.ciq_precond_build(lt)
    assert call(ps, u.data_ptr(), 10) == _lib.GP_E_SHAPE
    with pytest.raises(RuntimeError, match="shape"):
        ps.ciq_precond_build(lt)
    assert [q.launches() for q in (p, p0, ps)] == l0
    # non-finite inputs
    xb = x.clone()
    xb[5, 1] = float("nan")
    pb = Plan(xb).set_hypers("rbf", 0.5, 1.0, 0.1)
    with pytest.raises(NanError):
        pb.ciq_sqrt_matmul(b, [0.1, 1.0], [0.5, 0.5], precond_u=u)
    # the iteration cap warns
    op = AddedDiagLinearOperator(KernelLinearOperator(x, None, "rbf", torch.tensor(0.5, device=cuda_dev), torch.tensor(1.0, device=cuda_dev)),
                                 ConstantDiagLinearOperator(torch.tensor(0.01, device=cuda_dev), n))
    with settings.ciq_samples(True), settings.ciq_preconditioner(True), settings.min_preconditioning_size(0), \
            settings.max_cg_iterations(2), warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        s = op.zero_mean_mvn_samples(3)
    assert s.shape == (3, n) and torch.isfinite(s).all()
    assert op.last_ciq[2][0].precond_rank > 0
    assert any(issubclass(r.category, NumericalWarning) for r in rec)
    for q in (p, p0, ps, pb):
        q.close()
