"""Host side of sampling, no GPU: the contour quadrature (gpytorch_b200/sampling.py) against scipy, its accuracy bound, an fp64
restatement of multi-shift MINRES (the algorithm of csrc/minres.cu) against dense solves, the CIQ product against eigh square
roots, the psd-safe Cholesky, and MultivariateNormal.rsample / sample on dense CPU covariances (which never touch the engine)."""
import math
import warnings

import numpy as np
import pytest
import torch

from gpytorch_b200.sampling import contour_quadrature, psd_safe_cholesky


def msminres64(A, b, tau, tol, max_iter):
    """fp64 multi-shift MINRES, the recurrences of csrc/minres.cu: one Lanczos process on A from b / |b|, one Givens QR of
    T_k + tau_q I per shift.  Returns (sum_q w_q x_q is NOT formed here: X [Q, n] with X_q ~= (A + tau_q I)^-1 b),
    |phibar| per shift, iterations."""
    n = b.shape[0]
    Q = len(tau)
    tau = np.asarray(tau, dtype=np.float64)
    bn = np.linalg.norm(b)
    X = np.zeros((Q, n))
    if bn == 0:
        return X, np.zeros(Q), 0
    q, qprev, beta = b / bn, np.zeros(n), 0.0
    c1, s1, c2, s2 = np.ones(Q), np.zeros(Q), np.ones(Q), np.zeros(Q)
    pb = np.ones(Q)
    d1, d2 = np.zeros((Q, n)), np.zeros((Q, n))
    k = 0
    for k in range(max_iter):
        v = A @ q - beta * qprev
        alpha = q @ v
        v = v - alpha * q
        bn1 = np.linalg.norm(v)
        brk = not (bn1 > 1e-12 * math.sqrt(alpha * alpha + beta * beta + bn1 * bn1))
        if brk:
            bn1 = 0.0
        a = alpha + tau
        eps, dbar = s2 * beta, c2 * beta
        delta = c1 * dbar + s1 * a
        gbar = -s1 * dbar + c1 * a
        gamma = np.hypot(gbar, bn1)
        cn, sn = gbar / gamma, bn1 / gamma
        phi = cn * pb
        pb = -sn * pb
        dn = (q[None, :] - delta[:, None] * d1 - eps[:, None] * d2) / gamma[:, None]
        X += phi[:, None] * dn
        d2, d1 = d1, dn
        c2, s2, c1, s1 = c1, s1, cn, sn
        if brk or np.max(np.abs(pb)) <= tol:
            break
        qprev, q, beta = q, v / bn1, bn1
    return X * bn, np.abs(pb), k + 1


def _spd(n, kappa, seed):
    rng = np.random.default_rng(seed)
    Qm, _ = np.linalg.qr(rng.standard_normal((n, n)))
    e = np.geomspace(1.0, kappa, n)
    return (Qm * e) @ Qm.T, e


@pytest.mark.parametrize("kappa", [10.0, 1e3, 2e5, 1e6, 1e7])
def test_quadrature_matches_scipy(kappa):
    """tau and w against scipy.special.ellipj / ellipk, rel <= 1e-12, Q = 1..32.  (At kappa = 1e8 scipy's own dn near u = K' is off
    by 2e-10 against mpmath while the AGM here is within 4e-12, so that modulus is covered by the accuracy test below instead.)"""
    sp = pytest.importorskip("scipy.special")
    m, M = 0.1, 0.1 * kappa
    for Q in range(1, 33):
        tau, w = contour_quadrature(m, M, Q)
        k2 = 1.0 - m / M
        Kp = sp.ellipk(k2)
        u = (np.arange(1, Q + 1) - 0.5) * Kp / Q
        sn, cn, dn, _ = sp.ellipj(u, k2)
        t_ref = m * (sn / cn) ** 2
        w_ref = 2 * Kp * math.sqrt(m) / (math.pi * Q) * dn / cn ** 2
        assert np.max(np.abs(np.array(tau) - t_ref) / t_ref) <= 1e-12
        assert np.max(np.abs(np.array(w) - w_ref) / w_ref) <= 1e-12


@pytest.mark.parametrize("kappa", [10.0, 1e2, 1e4, 2e5, 1e6, 1e7, 1e8])
def test_quadrature_accuracy_bound(kappa):
    """max over [m, M] of |sqrt(lam) sum_q w_q / (lam + tau_q) - 1| <= 5 exp(-2 pi^2 Q / (ln kappa + 3)) + 1e-12 for Q = 2..32
    (at Q = 1 the error is O(1) and the bound, being > 1 only for small kappa, says nothing)."""
    m, M = 0.37, 0.37 * kappa
    lam = np.geomspace(m, M, 4000)
    for Q in range(2, 33):
        tau, w = contour_quadrature(m, M, Q)
        approx = (np.array(w)[None, :] / (lam[:, None] + np.array(tau)[None, :])).sum(1)
        err = np.max(np.abs(approx * np.sqrt(lam) - 1.0))
        assert err <= 5 * math.exp(-2 * math.pi ** 2 * Q / (math.log(kappa) + 3)) + 1e-12, (Q, err)


def test_quadrature_rejects_bad_interval():
    for m, M, Q in [(0.0, 1.0, 5), (1.0, 0.5, 5), (1.0, float("inf"), 5), (0.1, 1.0, 0)]:
        with pytest.raises(RuntimeError):
            contour_quadrature(m, M, Q)


@pytest.mark.parametrize("n,kappa,Q", [(200, 1e2, 1), (200, 1e4, 8), (300, 1e3, 15), (7, 50.0, 15)])
def test_oracle_msminres_matches_dense_solves(n, kappa, Q):
    A, e = _spd(n, kappa, n + Q)
    b = np.random.default_rng(1).standard_normal(n)
    tau, _ = contour_quadrature(e[0], e[-1], Q)
    X, res, it = msminres64(A, b, tau, 1e-11, 3 * n)
    for q in range(Q):
        xs = np.linalg.solve(A + tau[q] * np.eye(n), b)
        assert np.linalg.norm(X[q] - xs) <= 1e-7 * np.linalg.norm(xs) * math.sqrt(kappa)
        # the recurrence residual is the true residual
        tr = np.linalg.norm(b - (A + tau[q] * np.eye(n)) @ X[q]) / np.linalg.norm(b)
        assert abs(tr - res[q]) <= 1e-9
    if n == 7:
        assert it <= 8


@pytest.mark.parametrize("kappa", [1e2, 1e4])
def test_oracle_ciq_matches_eigh_sqrt(kappa):
    n, Q = 200, 15
    A, e = _spd(n, kappa, 3)
    b = np.random.default_rng(2).standard_normal(n)
    tau, w = contour_quadrature(e[0], e[-1], Q)
    X, _, _ = msminres64(A, b, tau, 1e-12, 4 * n)
    out = A @ (np.array(w)[:, None] * X).sum(0)
    ev, V = np.linalg.eigh(A)
    ref = (V * np.sqrt(ev)) @ (V.T @ b)
    qerr = 5 * math.exp(-2 * math.pi ** 2 * Q / (math.log(kappa) + 3))
    assert np.linalg.norm(out - ref) <= (qerr + 1e-9) * np.linalg.norm(ref) * 10


def test_psd_safe_cholesky_jitter_schedule_and_errors():
    from gpytorch_b200 import NanError, NotPSDError, NumericalWarning

    A = torch.tensor([[1.0, 1.0], [1.0, 1.0]])           # singular psd: one retry with 1e-6 is enough
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        L = psd_safe_cholesky(A)
    msgs = [str(r.message) for r in rec if issubclass(r.category, NumericalWarning)]
    assert msgs[0] == "A not p.d., added jitter of 1.0e-06 to the diagonal"
    assert len(msgs) == 1 and torch.allclose(L @ L.T, A + 1e-6 * torch.eye(2), atol=1e-6)
    B = torch.tensor([[1.0, 0.0], [0.0, -1.0]])          # indefinite: three warnings, then NotPSDError
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        with pytest.raises(NotPSDError, match="after repeatedly adding jitter up to 1.0e-04"):
            psd_safe_cholesky(B)
    assert [str(r.message) for r in rec] == [f"A not p.d., added jitter of {j:.1e} to the diagonal" for j in (1e-6, 1e-5, 1e-4)]
    with pytest.raises(NanError):
        psd_safe_cholesky(torch.tensor([[float("nan"), 0.0], [0.0, 1.0]]))
    with warnings.catch_warnings(record=True) as rec:       # fp64 schedule starts at 1e-8
        warnings.simplefilter("always")
        psd_safe_cholesky(A.double())
    assert str(rec[0].message) == "A not p.d., added jitter of 1.0e-08 to the diagonal"


def test_dense_rsample_shapes_and_base_samples():
    from gpytorch_b200.distributions import MultivariateNormal

    torch.manual_seed(0)
    n = 6
    X = torch.randn(n, n)
    C = X @ X.T + 0.5 * torch.eye(n)
    mu = torch.randn(n, requires_grad=True)
    d = MultivariateNormal(mu, C)
    assert d.rsample().shape == (n,)
    assert d.rsample(torch.Size([3, 2])).shape == (3, 2, n)
    assert d.sample(torch.Size([4])).shape == (4, n) and not d.sample(torch.Size([4])).requires_grad
    s = d.rsample(torch.Size([5]))
    s.sum().backward()
    assert torch.allclose(mu.grad, torch.full((n,), 5.0))
    # reseeded draws are mean + L eps
    torch.manual_seed(3)
    s = d.rsample(torch.Size([4]))
    torch.manual_seed(3)
    L = torch.linalg.cholesky(C)
    assert torch.allclose(s, (L @ torch.randn(n, 4)).T + mu, atol=1e-5)
    # base samples: sample shape taken from them
    base = torch.randn(7, 2, n)
    sb = d.rsample(base_samples=base)
    assert sb.shape == (7, 2, n)
    assert torch.allclose(sb, base @ L.T + mu, atol=1e-5)
    # batch of dense covariances
    Cb = torch.stack([C, 2 * C, 3 * C])
    mb = torch.zeros(3, n)
    db = MultivariateNormal(mb, Cb)
    assert db.rsample(torch.Size([5])).shape == (5, 3, n)
    bb = torch.randn(5, 3, n)
    out = db.rsample(base_samples=bb)
    Lb = torch.linalg.cholesky(Cb)
    assert torch.allclose(out, torch.einsum("bij,sbj->sbi", Lb, bb), atol=1e-4)
    # a covariance that gradients reach through torch's Cholesky
    Cg = C.clone().requires_grad_(True)
    MultivariateNormal(torch.zeros(n), Cg).rsample(torch.Size([2])).pow(2).sum().backward()
    assert Cg.grad is not None and torch.isfinite(Cg.grad).all()


def test_dense_rsample_low_rank_root_truncates_base_samples():
    from gpytorch_b200.distributions import MultivariateNormal
    from gpytorch_b200.operators import RootLinearOperator

    class LowRank:
        """A covariance operator whose root has rank 2 < n."""

        def __init__(self, R):
            self.R = R
            self.shape = torch.Size([R.shape[0], R.shape[0]])

        def root_decomposition(self):
            return RootLinearOperator(self.R)

    n = 5
    R = torch.randn(n, 2)
    d = MultivariateNormal(torch.zeros(n), LowRank(R))
    base = torch.randn(3, n)
    assert torch.allclose(d.rsample(base_samples=base), base[:, :2] @ R.T, atol=1e-6)


def test_settings_defaults():
    from gpytorch_b200 import settings

    assert settings.ciq_samples.off()
    assert settings.num_contour_quadrature.value() == 15
    assert settings.minres_tolerance.value() == 1e-4
    with settings.ciq_samples(True), settings.num_contour_quadrature(8):
        assert settings.ciq_samples.on() and settings.num_contour_quadrature.value() == 8


def test_minres_kernels_use_no_stack():
    """Every kernel of csrc/minres.cu compiles for sm_90a without stack / local memory (no spills)."""
    import os
    import re
    import shutil
    import subprocess

    from gpytorch_b200 import build

    build.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", os.path.join(build.OBJDIR, "minres.o")], capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*ms_\w+?_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    names = {re.search(r"ms_\w+?_kernel", f[0]).group(0) for f in found}
    assert names == {"ms_init_kernel", "ms_finish_kernel", "ms_orth_kernel", "ms_update_kernel", "ms_scale_kernel"}
    for fn, reg, stack, local in found:
        assert stack == "0" and local == "0", (fn, reg, stack, local)
