"""Host helpers of the sampling path: the contour-integral quadrature for K^{1/2}, the eigenvalue interval it needs, and a
psd-safe dense Cholesky.

CIQ (Pleiss et al. 2020, arXiv 2006.11267) writes  K^{1/2} b = K K^{-1/2} b ~= K sum_q w_q (K + tau_q I)^{-1} b  with the
shifts / weights of Hale, Higham & Trefethen 2008 (method 3) for z^{-1/2} on [m, M]; the shifted solves run on the device
(csrc/minres.cu).  Everything here is fp64 and pure Python: the package imports only torch.
"""
from __future__ import annotations

import math
import warnings

import torch

from ._lib import NanError, NotPSDError, NumericalWarning


def _agm_chain(m: float):
    """Arithmetic-geometric mean chain from (1, sqrt(1 - m)): the lists a_i, c_i of the descending Landen transformation."""
    a, b, c = [1.0], math.sqrt(1.0 - m), [math.sqrt(m)]
    while abs(c[-1] / a[-1]) > 1.1102230246251565e-16 and len(a) < 64:
        ai = a[-1]
        c.append((ai - b) / 2.0)
        a.append((ai + b) / 2.0)
        b = math.sqrt(ai * b)
    return a, c


def _ellipk(m: float) -> float:
    """Complete elliptic integral of the first kind K(m) (parameter m = k^2): pi / (2 AGM(1, sqrt(1 - m)))."""
    a, _ = _agm_chain(m)
    return math.pi / (2.0 * a[-1])


def _ellipj(u: float, m: float):
    """Jacobi elliptic functions (sn, cn, dn) of u at parameter m in [0, 1) by the AGM / descending Landen method."""
    a, c = _agm_chain(m)
    i = len(a) - 1
    phi = (2.0 ** i) * a[i] * u
    b = phi
    while i > 0:
        t = c[i] * math.sin(phi) / a[i]
        b = phi
        phi = (math.asin(t) + phi) / 2.0
        i -= 1
    return math.sin(phi), math.cos(phi), math.cos(phi) / math.cos(phi - b)


def contour_quadrature(m: float, M: float, Q: int):
    """Shifts tau_q and weights w_q (q = 1..Q) with  sum_q w_q / (lam + tau_q) ~= lam^{-1/2}  for lam in [m, M].

    Hale, Higham & Trefethen 2008, method 3: with k'^2 = 1 - m/M, K' = K(k'^2), u_q = (q - 1/2) K'/Q and
    (sn, cn, dn) = ellipj(u_q, k'^2):  tau_q = m (sn/cn)^2,  w_q = 2 K' sqrt(m) / (pi Q) * dn / cn^2.
    The relative error decays like exp(-2 pi^2 Q / (ln(M/m) + 3)) inside [m, M]; below m it grows fast, so m must bound the
    spectrum from below."""
    if not (m > 0.0 and M >= m and math.isfinite(M)):
        raise RuntimeError(f"contour quadrature needs 0 < m <= M < inf (m={m}, M={M})")
    if Q < 1:
        raise RuntimeError(f"contour quadrature needs Q >= 1 (Q={Q})")
    k2 = 1.0 - m / M
    Kp = _ellipk(k2)
    tau, w = [], []
    for q in range(1, Q + 1):
        sn, cn, dn = _ellipj((q - 0.5) * Kp / Q, k2)
        tau.append(m * (sn / cn) ** 2)
        w.append(2.0 * Kp * math.sqrt(m) / (math.pi * Q) * dn / cn ** 2)
    return tau, w


def psd_safe_cholesky(A: torch.Tensor, jitter=None, max_tries: int = 3) -> torch.Tensor:
    """Lower Cholesky factor of A; on failure adds jitter 1e-6, 1e-5, 1e-4 (fp32; 1e-8, 1e-7, 1e-6 in fp64) to the diagonal with
    a NumericalWarning per retry, then raises NotPSDError (linear_operator.utils.cholesky.psd_safe_cholesky)."""
    L, info = torch.linalg.cholesky_ex(A)
    if not torch.any(info):
        return L
    isnan = torch.isnan(A)
    if isnan.any():
        raise NanError(f"cholesky_cpu: {isnan.sum().item()} of {A.numel()} elements of the {tuple(A.shape)} tensor are NaN.")
    if jitter is None:
        jitter = 1e-6 if A.dtype == torch.float32 else 1e-8
    Aprime = A.clone()
    jitter_prev = 0.0
    for i in range(max_tries):
        jitter_new = jitter * (10 ** i)
        Aprime.diagonal(dim1=-2, dim2=-1).add_(jitter_new - jitter_prev)
        jitter_prev = jitter_new
        warnings.warn(f"A not p.d., added jitter of {jitter_new:.1e} to the diagonal", NumericalWarning)
        L, info = torch.linalg.cholesky_ex(Aprime)
        if not torch.any(info):
            return L
    raise NotPSDError(f"Matrix not positive definite after repeatedly adding jitter up to {jitter_new:.1e}. "
                      f"Original error on first attempt: {int(info.max())}-th leading minor not positive-definite")
