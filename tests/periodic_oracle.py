"""fp64 restatement of the periodic kernel and the per-entry bound of the engine's K.V on a periodic plan (csrc/periodic.cu).

    K(x, x') = S exp(-2 sum_d sin^2(pi tau_d / p_d) / l_d),   tau = x - x'

Bound derivation.  The engine packs z_d(x) = a_d (cos, sin)(2 pi r_d(x)), a_d = sqrt(log2 e / l_d), with r the reduced phase
x/p - round(x/p) formed in fp64 and rounded once to fp32, then runs the plain RBF K.V on z: k = 2^A, A = -|z - z'|^2 / 2.  The
terms of the bound, per pair:
  (1) rounding r to fp32: |dr| <= 2^-25 (|r| <= 1/2), so each endpoint's unit vector e moves by at most 2 pi 2^-25;
  (2) sincospi of the exact phase: at most 2 ulp per component, so |de| <= 2^-22 per endpoint;
      with delta = 2 (2 pi 2^-25 + 2^-22) for the two endpoints and |e - e'| <= 2, |d |e - e'|^2| <= 4 delta + delta^2, so
      |dA| <= sum_d a_d^2 (2 delta + delta^2 / 2);
  (3) the packing multiply a_d (cos, sin) and (4) GEMM1: tests/bilinear_oracle.py's pair_arg -- the model tests/kmv_oracle.py
      uses for the plain plans -- applied to the uncentred packed rows z themselves ((1 + KP/4) 2^-21 (|z_i|^2 + |z_j|^2) on
      tensor cores, with |z|^2 = sum_d a_d^2 for every point);
  (5) ex2.approx and the fp32 row sums: kmv_oracle's pair_rel and sums terms, as in kmv_oracle.bound.
Every term is a function of the lengthscales, the width and the product's size: nothing grows with |x|.
"""
from __future__ import annotations

import math

import torch

import bilinear_oracle as bo
import kmv_oracle as ko

U32 = 2.0 ** -24

LOG2E = 1.4426950408889634


def _params(ls, per, d):
    ls = torch.as_tensor(ls, dtype=torch.float64).reshape(-1).expand(d)
    per = torch.as_tensor(per, dtype=torch.float64).reshape(-1).expand(d)
    return ls, per


def kernel(x1, x2, ls, per, S=1.0):
    """K [n1, n2] in fp64 from the exact (fp64-reduced) phases: 4 sin^2(pi tau / p) = |e(x) - e(x')|^2."""
    x1, x2 = x1.double(), x2.double()
    ls, per = _params(ls, per, x1.size(-1))
    tau = x1[:, None, :] - x2[None, :, :]
    s2 = torch.sin(math.pi * tau / per) ** 2
    return S * torch.exp(-2.0 * (s2 / ls).sum(-1))


def embed(x, ls, per):
    """u(x) [n, 2d] in fp64: (cos, sin)(2 pi x / p) / sqrt(l), interleaved per dimension (the engine's packed layout, without the
    log2 e factor)."""
    x = x.double()
    ls, per = _params(ls, per, x.size(-1))
    t = x / per
    r = t - torch.floor(t + 0.5)
    ph = 2 * math.pi * r
    u = torch.stack([torch.cos(ph), torch.sin(ph)], -1) / ls.sqrt()[:, None]
    return u.reshape(x.size(0), -1)


def packed(x, ls, per):
    """The engine's packed rows [n, 2d] in fp64: sqrt(log2 e) u(x)."""
    return embed(x, ls, per) * math.sqrt(LOG2E)


def kmv_bound(x1, x2, ls, per, V, S, path, nsplit, T, same=False):
    """Per-entry bound [n1, t] of |engine K.V - kernel(x1, x2) S V| on path "tc" or "simt" with nsplit partial slots and T tiles
    per split (kmv_oracle.geometry of the packed width 2d); see the module docstring."""
    d = x1.size(-1)
    lsv, _ = _params(ls, per, d)
    zr = packed(x1, ls, per)
    zc = zr if same else packed(x2, ls, per)
    DP, KP = bo.dp_of(2 * d), bo.kp_of(2 * d)
    delta = 2 * (2 * math.pi * 2.0 ** -25 + 2.0 ** -22)
    e_phase = float((LOG2E / lsv).sum()) * (2 * delta + 0.5 * delta * delta)
    n2 = zc.size(0)
    if path == "tc":
        eps = ko.TC_CHAIN * (1 + 2.0 ** -11 + 2.0 ** -10) + 2 * U32 + T * U32
    else:
        eps = min(T * ko.TILE_J, n2) * U32
    eps += (nsplit + 1) * U32
    _, _, _, _, m, da = bo.pair_arg(zr, zc, (zc * zc).sum(1), path, DP, KP)
    da = da + e_phase
    if same:   # exact diagonal: a = 0 on both paths
        idx = torch.arange(zr.size(0))
        m[idx, idx] = 0.0
        da[idx, idx] = 0.0
    k, _ = bo._kg("rbf", m)
    dk, _ = bo._dev("rbf", m, da)
    rel = bo.pair_rel(m)
    kabs = k * (1 + rel) + dk
    pair = k * rel + dk
    if path == "tc":
        pair = pair + 2.0 ** -19 * kabs
    Va = V.double().abs()
    Sf = float(bo.f32(S))
    return Sf * (pair @ Va + eps * (kabs @ Va))


def grads(x1, x2, ls, per, W, S=1.0):
    """(dF/dl, dF/dp, dF/dS) of F = sum(W * K) by fp64 autograd, with ls / per of the given shapes (1 or d values)."""
    ls = torch.as_tensor(ls, dtype=torch.float64).clone().requires_grad_(True)
    per = torch.as_tensor(per, dtype=torch.float64).clone().requires_grad_(True)
    Sv = torch.tensor(float(S), dtype=torch.float64, requires_grad=True)
    d = x1.size(-1)
    K = Sv * kernel_t(x1.double(), x2.double(), ls.reshape(-1).expand(d), per.reshape(-1).expand(d))
    (K * W.double()).sum().backward()
    return ls.grad, per.grad, Sv.grad


def kernel_t(x1, x2, ls, per):
    tau = x1[:, None, :] - x2[None, :, :]
    return torch.exp(-2.0 * (torch.sin(math.pi * tau / per) ** 2 / ls).sum(-1))
