"""Host side of the preconditioned CIQ sampler, no GPU: an fp64 restatement of the split factor that gp_ciq_precond_build computes
(csrc/pivchol.cu, the math in the csrc/minres.cu header), its trace interval, and multi-shift MINRES on the preconditioned
operator mapped back through K_hat F^-T (the product gp_ciq_sqrt_matmul_precond returns).

P = L L^T + D, M = D^-1/2 L, (V, s) = eigh(M^T M), U = M V diag(h), h_j = (sqrt(1 + s_j) (1 + sqrt(1 + s_j)))^-1/2,
F^-1 = (I - U U^T) D^-1/2, A = F^-1 K_hat F^-T.  The identities are checked to 1e-12 relative to the norm of the matrix they
hold for (fp64 rounding grows with that norm)."""
import math

import numpy as np
import pytest
import torch

from gpytorch_b200.sampling import contour_quadrature
from oracle import kernels as ok, linalg as ol
from test_sampling_host import msminres64


def h_of(s):
    r1 = np.sqrt(1.0 + np.maximum(s, 0.0))
    return 1.0 / np.sqrt(r1 * (1.0 + r1))


def build64(L, d):
    """U [n, k] of the split factor from L [n, k] and the diagonal d [n] (fp64)."""
    M = L / np.sqrt(d)[:, None]
    s, V = np.linalg.eigh(M.T @ M)
    return (M @ V) * h_of(s)[None, :]


def _problem(kind, n, k, per_row, seed, deficient=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g, dtype=torch.float64)
    K = ok.kernel_matrix(kind, x, x, 0.5, 1.3, True)
    L, _ = ol.pivoted_cholesky(K.diagonal().clone(), lambda i: K[i], k)
    L = L.numpy()
    if L.shape[0] != n:
        L = L.T
    if deficient and L.shape[1] > 1:   # L Pr with an orthogonal projector Pr of rank k/2: L Pr Pr L^T <= L L^T keeps E >= 0
        Qr, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((L.shape[1], max(1, L.shape[1] // 2))))
        L = L @ (Qr @ Qr.T)
    d = (0.02 + 0.3 * torch.rand(n, generator=g, dtype=torch.float64)).numpy() if per_row else np.full(n, 0.05)
    return K.numpy(), L, d


CASES = [(kind, k, per_row, deficient) for kind in ("rbf", "matern12", "matern52") for k in (1, 15, 64, 128)
         for per_row in (False, True) for deficient in (False, True) if not (deficient and k == 1)]


@pytest.mark.parametrize("kind,k,per_row,deficient", CASES)
def test_split_factor_whitens_the_preconditioner(kind, k, per_row, deficient):
    n = 300
    K, L, d = _problem(kind, n, k, per_row, seed=k + 7 * per_row, deficient=deficient)
    U = build64(L, d)
    W = np.eye(n) - U @ U.T                                  # (I + M M^T)^-1/2
    Dm = 1.0 / np.sqrt(d)
    Pw = Dm[:, None] * (L @ L.T + np.diag(d)) * Dm[None, :]  # D^-1/2 P D^-1/2 = I + M M^T
    err = np.abs(W @ Pw @ W - np.eye(n)).max()
    assert err <= 1e-12 * np.linalg.norm(Pw, 2), err
    # the interval: every eigenvalue of A in [1 - 1e-10, 1 + tr E / min d], inside the [m, M] the operator uses
    Khat = K + np.diag(d)
    A = W @ (Dm[:, None] * Khat * Dm[None, :]) @ W
    ev = np.linalg.eigvalsh(A)
    tr_e = np.trace(K) - (L * L).sum()
    hi = 1.0 + tr_e / d.min()
    assert ev[0] >= 1.0 - 1e-10 and ev[-1] <= hi * (1 + 1e-10), (ev[0], ev[-1], hi)
    m, M = 0.5, 2.0 * (1.0 + max(tr_e, 1e-6 * np.trace(K)) / d.min())
    assert m <= ev[0] and ev[-1] <= M


def test_h_is_finite_at_zero_and_bounded():
    s = np.array([0.0, -1e-17, 1e-300, 1e-16, 1e-8, 1.0, 1e8, 1e300])
    h = h_of(s)
    assert np.isfinite(h).all()
    assert h[0] == h[1] == 1.0 / math.sqrt(2.0) and (h <= 1.0 / math.sqrt(2.0)).all()
    assert (np.diff(h) <= 0).all()
    # h^2 = (1 - (1 + s)^-1/2) / s, the form with the cancellation, where that form is accurate
    big = s[5:7]
    assert np.allclose(h_of(big) ** 2, (1 - 1 / np.sqrt(1 + big)) / big, rtol=1e-14)


@pytest.mark.parametrize("kind,k,per_row", [("rbf", 15, False), ("matern12", 64, True), ("matern52", 100, False),
                                            ("matern52", 30, True)])
def test_msminres_on_the_preconditioned_operator(kind, k, per_row):
    n, Q = 300, 15
    K, L, d = _problem(kind, n, k, per_row, seed=3 * k)
    Khat = K + np.diag(d)
    U = build64(L, d)
    W = np.eye(n) - U @ U.T
    Dm = 1.0 / np.sqrt(d)
    Finv_t = Dm[:, None] * W                                  # F^-T = D^-1/2 (I - U U^T)
    F = np.sqrt(d)[:, None] * np.linalg.inv(W)               # F = D^1/2 (I + M M^T)^1/2
    A = Finv_t.T @ Khat @ Finv_t
    assert np.abs(F @ A @ F.T - Khat).max() <= 1e-12 * np.linalg.norm(Khat, 2)
    tr_e = np.trace(K) - (L * L).sum()
    m, M = 0.5, 2.0 * (1.0 + max(tr_e, 1e-6 * np.trace(K)) / d.min())
    tau, w = contour_quadrature(m, M, Q)
    b = np.random.default_rng(k).standard_normal(n)
    X, _, it_a = msminres64(A, b, tau, 1e-10, 4 * n)
    out = Khat @ (Finv_t @ (np.array(w)[:, None] * X).sum(0))
    ev, V = np.linalg.eigh(A)
    ref = F @ ((V * np.sqrt(ev)) @ (V.T @ b))
    qerr = 5 * math.exp(-2 * math.pi ** 2 * Q / (math.log(M / m) + 3))
    assert np.linalg.norm(out - ref) <= (qerr + 1e-9) * np.linalg.norm(ref) * 10
    # fewer iterations than on K_hat itself whenever the preconditioner cuts the condition number tenfold
    ek = np.linalg.eigvalsh(Khat)
    tau_k, _ = contour_quadrature(ek[0], ek[-1], Q)
    _, _, it_k = msminres64(Khat, b, tau_k, 1e-10, 4 * n)
    kappa_a, kappa_k = ev[-1] / ev[0], ek[-1] / ek[0]
    print(f"\n{kind} k={k} per_row={per_row}: kappa(A) {kappa_a:.3g} kappa(K_hat) {kappa_k:.3g}, iterations {it_a} vs {it_k}")
    if kappa_a <= kappa_k / 10:
        assert it_a < it_k


def test_ciq_preconditioner_defaults_off():
    from gpytorch_b200 import settings

    assert settings.ciq_preconditioner.off()
    with settings.ciq_preconditioner(True):
        assert settings.ciq_preconditioner.on()
    assert settings.ciq_preconditioner.off()
