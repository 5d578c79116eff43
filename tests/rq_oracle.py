"""fp64 restatement of the rational quadratic kernel, the per-entry bound of the engine's K.V on an RQ plan, and fp32 emulations
of the device formulas (gp_common.cuh: rq_lg2_1p, rq_phi).

    K(x, x') = S (1 + t)^-alpha,   t = r^2 / (2 alpha),   r^2 = |(x - x') / l|^2

Bound derivation.  The engine packs z = (x - mean) / l (C = 1, alpha stays out of the packing) and forms a = -r^2 / 2 as for RBF;
then t = max(-a, 0) (1/alpha)_fp32, L = log2(1 + t) and k = ex2(-alpha L).  Per pair, with m = r^2 / 2:
  (1) packing and GEMM1: tests/bilinear_oracle.py's pair_arg (the model of tests/kmv_oracle.py) gives |da|; since
      |dk/dm| = k / (1 + t) <= 1, the value moves by at most da times the largest k / (1 + t) over [m - da, m + da];
  (2) t: 1/alpha rounded once and one multiply, relative 2u (u = 2^-24), so |dL| <= 2u t / ((1 + t) ln 2);
  (3) L itself: below t = 1/16 the degree-6 polynomial (truncation t^7 / 7 log2 e, Horner and the log2 e multiply: 8u L); above,
      the rounding of 1 + t (u / ln 2) and lg2.approx's absolute error 2^-22;
  (4) the product -alpha L (u |E|) and ex2.approx (2^-21 relative);
  (2)-(4) change the exponent E = -alpha L by dE and k by k ln2 dE.  Every dE is either relative to E (so k |E| 2^-|E| <= 1/(e ln 2)
  keeps it bounded) or alpha times an error of L that only the MUFU branch has, where alpha L >= alpha log2(17/16) makes k
  vanish faster than alpha grows.  At fixed r no term grows with alpha.
  (5) the fp32 row sums and the tensor-core split of P: kmv_oracle's terms, as periodic_oracle.kmv_bound uses them.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import bilinear_oracle as bo
import kmv_oracle as ko

U32 = 2.0 ** -24
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2


def kernel(x1, x2, ls, alpha, S=1.0):
    """K [n1, n2] in fp64."""
    x1, x2 = x1.double(), x2.double()
    ls = torch.as_tensor(ls, dtype=torch.float64).reshape(-1)
    d2 = (((x1[:, None, :] - x2[None, :, :]) / ls) ** 2).sum(-1)
    return S * torch.pow(1.0 + d2 / (2.0 * float(alpha)), -float(alpha))


def packed(x, ref, ls):
    """fp32 packed rows z = (x - mean(ref)) / l in fp64 (pack.cu with C = 1)."""
    ls = torch.as_tensor(ls, dtype=torch.float64).reshape(-1)
    mean = ref.double().mean(0)
    return ((x.double() - mean) / ls).float().double()


def _lg2_err(t, alpha):
    """Bound on |dL| of terms (2) and (3) above, per pair."""
    L = torch.log2(1.0 + t)
    small = 8 * U32 * L + t ** 7 / 7 * LOG2E
    big = U32 * LOG2E + 2.0 ** -22
    return torch.where(t < 0.0625, small, big) + 2 * U32 * t / ((1 + t) * LN2)


def kmv_bound(x1, x2, ls, alpha, V, S, path, nsplit, T, same=False):
    """Per-entry bound [n1, t] of |engine K.V - kernel(x1, x2) S V| on path "tc" or "simt" with nsplit partial slots and T tiles
    per split (kmv_oracle.geometry); see the module docstring."""
    d = x1.size(-1)
    alpha = float(np.float32(alpha))
    zr = packed(x1, x1, ls)
    zc = zr if same else packed(x2, x1, ls)
    DP, KP = bo.dp_of(d), bo.kp_of(d)
    n2 = zc.size(0)
    if path == "tc":
        eps = ko.TC_CHAIN * (1 + 2.0 ** -11 + 2.0 ** -10) + 2 * U32 + T * U32
    else:
        eps = min(T * ko.TILE_J, n2) * U32
    eps += (nsplit + 1) * U32
    _, _, _, _, m, da = bo.pair_arg(zr, zc, (zc * zc).sum(1), path, DP, KP)
    if same:
        idx = torch.arange(zr.size(0))
        m[idx, idx] = 0.0
        da[idx, idx] = 0.0
    t = m / alpha
    k = torch.pow(1.0 + t, -alpha)
    tlo = (m - da).clamp_min(0.0) / alpha
    q_hi = torch.pow(1.0 + tlo, -alpha - 1.0)                   # the largest k / (1 + t) over the interval of m
    E = alpha * torch.log2(1.0 + t)
    khi = torch.pow(1.0 + tlo, -alpha)
    dE = alpha * _lg2_err(t, alpha) + U32 * E
    dk = da * q_hi + khi * LN2 * dE * (1 + 2 * LN2 * dE)
    rel = 2.0 ** -21 + 2 * U32
    kabs = khi * (1 + rel) + dk
    pair = khi * rel + dk
    if path == "tc":
        pair = pair + 2.0 ** -19 * kabs
    Va = V.double().abs()
    Sf = float(bo.f32(S))
    return Sf * (pair @ Va + eps * (kabs @ Va))


def grads(x1, x2, ls, alpha, W, S=1.0):
    """(dF/dl, dF/dalpha, dF/dS) of F = sum(W * K) by fp64 autograd; ls of the given shape (1 or d values)."""
    ls = torch.as_tensor(ls, dtype=torch.float64).clone().requires_grad_(True)
    al = torch.tensor(float(alpha), dtype=torch.float64, requires_grad=True)
    Sv = torch.tensor(float(S), dtype=torch.float64, requires_grad=True)
    d2 = (((x1.double()[:, None, :] - x2.double()[None, :, :]) / ls.reshape(-1)) ** 2).sum(-1)
    K = Sv * torch.pow(1.0 + d2 / (2.0 * al), -al)
    (K * W.double()).sum().backward()
    return ls.grad, al.grad, Sv.grad


# ---- fp32 emulation of the device formulas (numpy float32 rounds every operation, as the FMA pipe does up to its fused adds) ----
def lg2_1p_f32(t):
    """rq_lg2_1p below t = 1/16 (the polynomial; the MUFU branch is not emulated)."""
    t = np.float32(t)
    p = np.float32(t * np.float32(-0.16666667) + np.float32(0.2))
    for c in (-0.25, 0.33333334, -0.5, 1.0):
        p = np.float32(t * p + np.float32(c))
    return np.float32(np.float32(LOG2E) * np.float32(t * p))


def phi_f32(t):
    """rq_phi: the series to n = 9 below 1/8, the difference of log1p and t / (1 + t) above."""
    t = np.float32(t)
    if t < 0.125:
        s = np.float32(t * np.float32(-0.88888889) + np.float32(0.875))
        for c in (-0.85714286, 0.83333333, -0.8, 0.75, -0.66666667, 0.5):
            s = np.float32(t * s + np.float32(c))
        return np.float32(np.float32(t * t) * s)
    return np.float32(np.log1p(t) - np.float32(t / np.float32(1 + t)))


def phi_exact(t):
    t = float(t)
    return math.log1p(t) - t / (1 + t)
