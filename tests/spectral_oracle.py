"""fp64 oracle of the spectral mixture operator (csrc/spectral.cu) and a per-entry bound for its K.V.

K(x, x') = S prod_c s_c,   s_c = sum_q w_q e_qc cos_qc,   e_qc = exp(-2 pi^2 v_qc^2 tau_c^2),   cos_qc = cos(2 pi mu_qc tau_c),
tau = x - x'  (the reference sums the components of each dimension, then multiplies over the dimensions).

Bound.  The engine works on the fp32 inputs x and, per (q, c), the reduced phase p_qc = mu_qc x_c - round(mu_qc x_c) in
[-1/2, 1/2), formed in fp64 (mu x is exact there) and rounded once to fp32.  Per pair, with u = 2^-24:

  * tau_c = fl(x_c - x'_c) has relative error u, so t2 = fl(tau_c^2) has relative error 3u;  beta_qc = -2 pi^2 v^2 log2 e is
    rounded to fp32 (u), and the argument a = fl(beta t2) carries a relative error of 5u.  ex2.approx adds a relative 2^-22 and
    flushes results below 2^-126 to zero, so |de_qc| <= e_qc (2^-22 + 5u ln2 |a|) + 2^-126: the exponent's relative error, which
    depends on tau alone, and the underflow floor;
  * the phase difference fl(p - p') is within 2^-24 of p - p' (two roundings of |p| <= 1/2 to fp32, one of a difference below 1),
    the multiplication by 2 pi (the constant rounded to fp32, the product rounded to fp32, |2 pi dp| < 2 pi) adds 2 pi u + 2^-22,
    and __cosf's reduction to revolutions one more 2 pi u: an absolute phase error dphi = 2 pi 2^-24 + 2 pi u + 2^-22 + 2 pi u
    radians, of order u, whatever |x|;
  * MUFU.COS has an absolute error of at most 2^-20.5 over -100 pi .. 100 pi (PTX ISA, cos.approx.f32), so
    |dcos_qc| <= dphi + 2^-20.5;
  * a term a_qc = w_q e_qc cos_qc rounds once more (u) and the Q-term FMA chain of s_c adds Q u sum_q |a_qc|:
    ds_c = sum_q w_q (|de_qc| + e_qc |dcos_qc| + 2u e_qc) + Q u sum_q w_q e_qc;
  * k = S prod_c s_c (d - 1 products, and the multiplication by S where a row or the diagonal applies it):
    dk <= S (sum_c ds_c prod_{c' != c} (|s_c'| + ds_c') + d u prod_c |s_c|).

The product: every row sum of one split is a chain of fp32 FMAs over its columns, the splits are then added and scaled by S,
so with n2 columns |(K V)_ic - exact| <= sum_j (dk_ij + (n2 + 2) u |k_ij|) |V_jc|.  Nothing in the bound grows with |x|: the
reference's fp32 argument 2 pi (mu x - mu x') instead has an absolute error of order 2 pi u |mu x|.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
EX2_REL = 2.0 ** -22
COS_ABS = 2.0 ** -20.5
FTZ = 2.0 ** -126
DPHI = 2 * math.pi * 2.0 ** -24 + 2 * math.pi * U + 2.0 ** -22 + 2 * math.pi * U


def _params(w, mu, v, d):
    w = torch.as_tensor(w, dtype=torch.float64).reshape(-1)
    mu = torch.as_tensor(mu, dtype=torch.float64).reshape(w.numel(), d)
    v = torch.as_tensor(v, dtype=torch.float64).reshape(w.numel(), d)
    return w, mu, v


def _terms(x1, x2, w, mu, v, diag=False):
    """Per (q, c) fp64 exponents e and cosines [Q, n1, n2, d] (or [Q, n, d] for diag) and tau."""
    x1, x2 = x1.double(), x2.double()
    d = x1.size(-1)
    w, mu, v = _params(w, mu, v, d)
    dev = x1.device
    w, mu, v = w.to(dev), mu.to(dev), v.to(dev)
    tau = (x1 - x2) if diag else (x1.unsqueeze(-2) - x2.unsqueeze(-3))
    shp = (-1,) + (1,) * (tau.dim() - 1) + (d,)
    mu_ = mu.reshape(mu.size(0), *shp[1:])
    v_ = v.reshape(v.size(0), *shp[1:])
    e = torch.exp(-2 * math.pi ** 2 * v_ ** 2 * tau.unsqueeze(0) ** 2)
    # the phase in fp64 from the reduced products, as exact as fp64 allows for fp32 inputs and means
    if diag:
        ph = _frac(mu_ * x1.unsqueeze(0)) - _frac(mu_ * x2.unsqueeze(0))
    else:
        ph = _frac(mu_ * x1.unsqueeze(-2).unsqueeze(0)) - _frac(mu_ * x2.unsqueeze(-3).unsqueeze(0))
    cs = torch.cos(2 * math.pi * ph)
    return w, e, cs, tau


def _frac(t):
    return t - torch.floor(t + 0.5)


def covariance(x1, x2, w, mu, v, S=1.0, diag=False):
    """K(x1, x2) in fp64: [n1, n2], or [n] with diag=True (x1, x2 of equal sizes)."""
    w, e, cs, _ = _terms(x1, x2, w, mu, v, diag)
    s = (w.reshape(-1, *([1] * (e.dim() - 1))) * e * cs).sum(0)
    return S * s.prod(-1)


def covariance_torch(x1, x2, w, mu, v, S=1.0):
    """The same covariance written with torch operations on differentiable fp64 parameter tensors (for autograd checks)."""
    d = x1.size(-1)
    tau = x1.double().unsqueeze(-2) - x2.double().unsqueeze(-3)           # [n1, n2, d]
    w_ = w.reshape(-1, 1, 1, 1)
    mu_ = mu.reshape(-1, 1, 1, d)
    v_ = v.reshape(-1, 1, 1, d)
    terms = w_ * torch.exp(-2 * math.pi ** 2 * v_ ** 2 * tau ** 2) * torch.cos(2 * math.pi * mu_ * tau)
    return S * terms.sum(0).prod(-1)


def entry_bound(x1, x2, w, mu, v, S=1.0, diag=False):
    """Per-entry bound |k_engine - k| (before the product's accumulation), fp64, same shape as covariance()."""
    w, e, cs, tau = _terms(x1, x2, w, mu, v, diag)
    Q = w.numel()
    d = tau.size(-1)
    vv = _params(w, mu, v, d)[2].to(tau.device)
    a = (-2 * math.pi ** 2 * vv.reshape(Q, *([1] * (tau.dim() - 1)), d) ** 2 * tau.unsqueeze(0) ** 2) / math.log(2.0)
    wq = w.reshape(-1, *([1] * (e.dim() - 1)))
    de = e * (EX2_REL + 5 * U * math.log(2.0) * a.abs()) + FTZ
    dc = DPHI + COS_ABS
    ds = (wq * (de + e * dc + 2 * U * e)).sum(0) + Q * U * (wq * e).sum(0)     # [..., d]
    s = (wq * e * cs).sum(0)
    sa = s.abs()
    dk = torch.zeros_like(s[..., 0])
    for c in range(d):
        other = torch.ones_like(dk)
        for c2 in range(d):
            if c2 != c:
                other = other * (sa[..., c2] + ds[..., c2])
        dk = dk + ds[..., c] * other
    dk = dk + d * U * sa.prod(-1)
    return S * dk


def kmv_bound(x1, x2, w, mu, v, V, S=1.0):
    """Per-entry bound of the engine's K V against the fp64 product, [n1, t]."""
    K = covariance(x1, x2, w, mu, v, S)
    dk = entry_bound(x1, x2, w, mu, v, S)
    n2 = x2.size(0)
    return (dk + (n2 + 2) * U * K.abs()) @ V.double().abs()
