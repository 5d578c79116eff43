"""fp64 closed form of the kernel input gradient and the fp32 error bound of the engine's gp_kmv_input_grad /
gp_kdense_input_grad (test infrastructure; imported by test_xgrad_host.py and test_gpu_input_grad.py).

For k(x, x') = s f(r^2), r^2 = sum_c ((x_c - x'_c) / l_c)^2 (kernels/rbf_kernel.py:68-85, kernels/matern_kernel.py:86-107):
    dk(x_i, x_j)/dx_i = -s h(r^2) (x_i - x_j) / l^2,   h = -2 f'(r^2)
    RBF  e^{-r^2/2} ;  Matern-1/2  e^{-r}/r ;  Matern-3/2  3 e^{-sqrt3 r} ;  Matern-5/2  (5/3)(1 + sqrt5 r) e^{-sqrt5 r}
A pair at distance 0 contributes 0 (the clamps of kernels/kernel.py:52-60).  Differences are formed directly, in row blocks.
"""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -24
_C = {"rbf": 1.0 / math.log(2.0), "matern12": 2.0, "matern32": 6.0, "matern52": 10.0}   # pack.cu: z = (x - mean) sqrt(C) / l


def _h(kind, r2):
    r = r2.sqrt()
    if kind == "rbf":
        h = torch.exp(-0.5 * r2)
    elif kind == "matern12":
        h = torch.exp(-r) / r
    elif kind == "matern32":
        h = 3.0 * torch.exp(-math.sqrt(3.0) * r)
    elif kind == "matern52":
        h = (5.0 / 3.0) * (1.0 + math.sqrt(5.0) * r) * torch.exp(-math.sqrt(5.0) * r)
    else:
        raise ValueError(kind)
    return torch.where(r2 > 0, h, torch.zeros_like(h))


def _ls(lengthscale, d):
    ls = torch.as_tensor(lengthscale, dtype=torch.float64).reshape(-1)
    return ls.expand(d) if ls.numel() == 1 else ls


def _blocks(n, size=128):
    for i0 in range(0, n, size):
        yield slice(i0, min(n, i0 + size))


def input_grad(kind, x1, x2, lengthscale, outputscale, W, same=False):
    """(dF/dx1 [n1, d], dF/dx2 [n2, d]) of F = sum_ij W_ij s k(x1_i, x2_j) in fp64; with same=True (x2 is x1) one array, the
    total gradient of F(x, x)."""
    x1, x2, W = x1.double(), x2.double(), W.double()
    ls = _ls(lengthscale, x1.size(1))
    il2 = float(outputscale) / ls**2
    dx1 = torch.zeros_like(x1)
    dx2 = torch.zeros_like(x2)
    for b in _blocks(x1.size(0)):
        diff = x1[b, None, :] - x2[None, :, :]                         # [bi, n2, d]
        coef = W[b] * _h(kind, ((diff / ls) ** 2).sum(-1))             # [bi, n2]
        dx1[b] = -il2 * (coef.unsqueeze(-1) * diff).sum(1)
        dx2 += il2 * (coef.unsqueeze(-1) * diff).sum(0)
    return dx1 + dx2 if same else (dx1, dx2)


def input_grad_bound(kind, x1, x2, lengthscale, outputscale, Wabs, t, same=False):
    """Entry-wise bound of |engine - input_grad| for the same fp32 inputs, with Wabs_ij >= |w_ij| + |fl(w_ij) - w_ij| / (t u)
    (sum_c |G_ic| |V_jc| for the product form, |W_ij| (+ |W_ji|) for the dense form) and t the dot length (0: dense).

    Per pair (z = (x - mean) sqrt(C) / l packed in fp32, a = -|z_i - z_j|^2 / 2, q = df/da):
      w       t-term fp32 dot: relative t u of Wabs
      z       two roundings per entry: |dz| <= 2 u |z|, so the direction z_i - z_j is off by E = 2 u (|z_i| + |z_j|) and
              a by  da <= (DP + 3) u |a| + E |z_i - z_j| ;  q then by |d ln q / da| da
              (RBF ln 2 ; Matern-1/2 (1 + 1/rho) / (2 rho) ; Matern-3/2, -5/2 1 / (2 rho), rho = sqrt(-a))
      q       ex2.approx 2^-22, sqrt.approx 2^-22, the fp32 product -log2(e) rho: 2 u (1 + rho)
      sums    fp32 accumulation over the reduced side (nt terms per split, then nsplit <= nt partials in order): 2 nt u
              of the sum of magnitudes; the final -s sqrt(C)/l scaling 3 u.
    The bound sums the magnitudes |w q (z_i - z_j)| (s sqrt(C)/l_c) times these relative errors plus Wabs q E.  It is a
    worst-case bound (every rounding at its extreme, same sign), not an estimate."""
    x1, x2, Wabs = x1.double(), x2.double(), Wabs.double()
    d = x1.size(1)
    DP = next(o for o in (4, 8, 12, 16, 24, 32, 48, 64) if d <= o)
    ls = _ls(lengthscale, d)
    sc = math.sqrt(_C[kind]) / ls
    mean = x1.mean(0)
    z1, z2 = (x1 - mean) * sc, (x2 - mean) * sc
    out1 = torch.zeros_like(x1)
    out2 = torch.zeros_like(x2)
    rel_sum = 2.0 * max(x1.size(0), x2.size(0)) * U32 + 3 * U32 + t * U32

    def q_and_l(a):
        rho = (-a).clamp_min(0).sqrt()
        if kind == "rbf":
            q = math.log(2.0) * torch.exp2(a)
            lq = torch.full_like(a, math.log(2.0))
        else:
            e = torch.exp(-rho)
            q = {"matern12": 0.5 * e / rho, "matern32": 0.5 * e, "matern52": (1 + rho) * e / 6}[kind]
            lq = (1 + 1 / rho) / (2 * rho) if kind == "matern12" else 1 / (2 * rho)
        return q, lq, rho

    for b in _blocks(x1.size(0)):
        dz = z1[b, None, :] - z2[None, :, :]
        nz = dz.norm(dim=-1)
        a = -0.5 * nz**2
        E = 2 * U32 * (z1[b, None, :].abs() + z2[None, :, :].abs())             # [bi, n2, d]
        q, lq, rho = q_and_l(a)
        da = (DP + 3) * U32 * a.abs() + E.norm(dim=-1) * nz
        eps = rel_sum + 2.0 ** -21 + 2 * U32 * (1 + rho) + lq * da
        mask = (a < 0).double()
        term = (Wabs[b] * q * mask).unsqueeze(-1) * (dz.abs() * eps.unsqueeze(-1) + E)
        term = torch.nan_to_num(term, nan=0.0, posinf=0.0)
        out1[b] = term.sum(1)
        out2 += term.sum(0)
    scale = float(outputscale) * sc
    if same:
        return (out1 + out2) * scale
    return out1 * scale, out2 * scale
