"""fp64 restatement of the polynomial kernel and the per-entry bound of the engine's K.V on a polynomial plan.

    K(x, x') = S (x . x' + c)^p      (raw inputs: no lengthscale, no centring)

Bound derivation.  The bound is stated in m_ij = sum_c |x_ic| |x_jc| + c, not in |k_ij|: where x_i . x_j cancels c, k is tiny
but the rounding of a is not, so a bound in |k| would not hold there.
  (1) the argument a = x_i . x_j + c.  Tensor cores (pack.cu): 3xTF32 operands, the offset split c = c_hi + c_lo in the spare
      columns; each product drops lo * lo and the tf32 residuals (3 2^-22 |x_ic| |x_jc|), the fp32 accumulation over the KP
      columns of GEMM1 adds at most KP 2^-23 times the running sum of magnitudes, and c_hi + c_lo is c to 2^-22 c.  So
      |da| <= gamma m with gamma = (2 + KP) 2^-22.  CUDA cores: a chain of DP fmas and one add, gamma = (DP + 2) 2^-24.
  (2) the power by squaring (gp_common.cuh poly_pow): any product tree that forms a^p carries at most p - 1 roundings, relative
      (p - 1) u (u = 2^-24).  |a^p - (a + da)^p| <= p |da| (m + |da|)^(p-1) <= p gamma (1 + gamma)^(p-1) m^p.
  So |dk| <= S m^p [p gamma (1 + gamma)^(p-1) + (p - 1) u (1 + gamma)^p] =: pair, and |k| <= S (m (1 + gamma))^p =: kabs.
  (3) the fp32 row sums and the tensor-core split of P: kmv_oracle's terms, as rq_oracle.kmv_bound uses them.
"""
from __future__ import annotations

import torch

import bilinear_oracle as bo
import kmv_oracle as ko

U32 = 2.0 ** -24


def kernel(x1, x2, power, offset, S=1.0):
    """K [n1, n2] in fp64."""
    return S * torch.pow(x1.double() @ x2.double().T + float(offset), int(power))


def diag(x, power, offset, S=1.0):
    return S * torch.pow((x.double() ** 2).sum(-1) + float(offset), int(power))


def gamma(d, path):
    return (2 + bo.kp_of(d)) * 2.0 ** -22 if path == "tc" else (bo.dp_of(d) + 2) * U32


def entry_bound(x1, x2, power, offset, path):
    """(pair, kabs) [n1, n2]: the per-entry error bound and magnitude bound of S = 1 (see the module docstring)."""
    p = int(power)
    m = x1.double().abs() @ x2.double().abs().T + float(offset)
    g = gamma(x1.size(1), path)
    mp = m ** p
    pair = mp * (p * g * (1 + g) ** (p - 1) + (p - 1) * U32 * 1.01 * (1 + g) ** p)
    kabs = mp * (1 + g) ** p
    return pair, kabs


def kmv_bound(x1, x2, power, offset, V, S, path, nsplit, T):
    """Per-entry bound [n1, t] of |engine K.V - kernel(x1, x2) V| on path "tc" or "simt" with nsplit partial slots and T tiles
    per split (kmv_oracle.geometry)."""
    n2 = x2.size(0)
    if path == "tc":
        eps = ko.TC_CHAIN * (1 + 2.0 ** -11 + 2.0 ** -10) + 2 * U32 + T * U32
    else:
        eps = min(T * ko.TILE_J, n2) * U32
    eps += (nsplit + 1) * U32
    pair, kabs = entry_bound(x1, x2, power, float(torch.tensor(offset, dtype=torch.float32)), path)
    if path == "tc":
        pair = pair + 2.0 ** -19 * kabs
    Va = V.double().abs()
    return float(bo.f32(S)) * (pair @ Va + eps * (kabs @ Va))


def grads(x1, x2, power, offset, W, S=1.0):
    """(dF/dc, dF/dS) of F = sum(W * K) by fp64 autograd."""
    c = torch.tensor(float(offset), dtype=torch.float64, requires_grad=True)
    Sv = torch.tensor(float(S), dtype=torch.float64, requires_grad=True)
    K = Sv * torch.pow(x1.double() @ x2.double().T + c, int(power))
    (K * W.double()).sum().backward()
    return c.grad, Sv.grad


def input_grads(x1, x2, power, offset, W, S=1.0):
    """(dF/dx1, dF/dx2) of F = sum(W * K) by fp64 autograd; x2 None: the square plan (one set of points, both arguments)."""
    a = x1.double().clone().requires_grad_(True)
    b = a if x2 is None else x2.double().clone().requires_grad_(True)
    K = S * torch.pow(a @ b.T + float(offset), int(power))
    (K * W.double()).sum().backward()
    return a.grad, (None if x2 is None else b.grad)
