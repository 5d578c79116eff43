"""fp64 oracle of the additive operator (csrc/additive.cu) and a per-entry bound for its K.V.

K(x, x') = sum_{m=1}^{M} e_m(c_1 .. c_D),  c_i = s_i k_i(x_i, x'_i) of one kind over column i with lengthscale l_i.

Bound.  The engine packs z_i = (x_i - mean_i) sqrt(C) / l_i in fp32 (pack.cu; C = log2 e for RBF, 2 nu * 2 for Matern as in
kmv_oracle) and forms per pair, per component:

  * df = z_i - z'_i in fp32.  The packing rounds z to within 3u (|z| + |mean_i| sqrt(C) / l_i) (subtract, multiply, scale), so
    |df - df_exact| <= dz_i = 3u (|z_i| + |z'_i| + 2 |mean_i| sqrt(C) / l_i) + u |df|  (u = 2^-24);
  * k_i from a = -df^2 / 2 through ex2.approx (relative error <= 2^-22) and, for Matern, sqrt.approx and the polynomial: the
    pair model of kmv_oracle / bilinear_oracle gives |k - k_exact| <= (2^-21 + 8u (1 + |a|)) k + L dz_i with the Lipschitz constant
    of k in df, L = ln2 |df| for RBF (dk/ddf = -ln2 df k, k <= 1) and L = 1 for Matern (dk/drho <= 1, rho = |df| / sqrt 2);
  * c_i = s_i k_i adds u c_i, so |dc_i| <= s_i ((2^-21 + 9u (1 + |a|)) k_i + L dz_i).

The positive recurrence combines non-negative terms: an error dc_i moves K by at most dK/dc_i dc_i with dK/dc_i =
sum_{m=1}^{M} e_{m-1}(c without c_i) <= P := sum_{m=0}^{M-1} e_m(c), and the recurrence's own D M FMAs and the final M - 1 adds
round every partial sum of positive terms, (2 D M + M) u relative in all.  So per entry

  dK_ij <= P_ij sum_i |dc_i| + (2 D M + M) u K_ij.

The product: every row sum of one split is a chain of fp32 FMAs over its columns, the splits are then added and scaled by 1, so
with n2 columns |(K V)_ic - exact| <= sum_j (dK_ij + (n2 + 2) u K_ij) |V_jc|.  The bound is returned in fp64 for each entry.
"""
from __future__ import annotations

import itertools
import math

import torch

U = 2.0 ** -24
CONST = {"rbf": 1.0 / math.log(2.0), "matern12": 2.0, "matern32": 6.0, "matern52": 10.0}   # pack.cu: C (RBF: log2 e)
NU = {"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}


def component_cov(kind: str, a: torch.Tensor, b: torch.Tensor, ls: float) -> torch.Tensor:
    """k(a_i, b_j) of one component in fp64 (the reference's covariance functions, one input dimension)."""
    r = (a.reshape(-1, 1).double() - b.reshape(1, -1).double()).abs() / ls
    if kind == "rbf":
        return torch.exp(-0.5 * r * r)
    nu = NU[kind]
    d = math.sqrt(2.0 * nu) * r
    e = torch.exp(-d)
    if nu == 0.5:
        return e
    if nu == 1.5:
        return (1.0 + d) * e
    return (1.0 + d + d * d / 3.0) * e


def esym_sum(cs, M: int) -> torch.Tensor:
    """sum_{m=1}^{M} e_m(c_1 .. c_D) entry by entry, positive recurrence in the inputs' dtype."""
    M = min(M, len(cs))
    e = [torch.ones_like(cs[0])] + [torch.zeros_like(cs[0]) for _ in range(M)]
    for c in cs:
        for m in range(M, 0, -1):
            e[m] = e[m] + c * e[m - 1]
    return sum(e[1:])


def brute_force(cs, M: int) -> torch.Tensor:
    """The same sum over itertools.combinations (small D only)."""
    out = torch.zeros_like(cs[0])
    for m in range(1, min(M, len(cs)) + 1):
        for S in itertools.combinations(range(len(cs)), m):
            t = torch.ones_like(cs[0])
            for i in S:
                t = t * cs[i]
            out = out + t
    return out


def newton_girard(cs, M: int) -> torch.Tensor:
    """The reference's formula (alternating power sums), fp64, for cross-checks only."""
    p = [sum(c ** (k + 1) for c in cs) * (-1.0) ** k for k in range(M)]
    E = [p[0]]
    for deg in range(1, M):
        s = p[deg]
        for k in range(deg):
            s = s + p[k] * E[deg - 1 - k]
        E.append(s / (deg + 1))
    return sum(E)


def components(kind, X1, X2, ls, scales):
    """[c_i] (fp64, n1 x n2 each) over the columns of X1 / X2."""
    return [float(scales[i]) * component_cov(kind, X1[:, i], X2[:, i], float(ls[i])) for i in range(X1.size(1))]


def additive_dense(kind, X1, X2, ls, scales, M) -> torch.Tensor:
    return esym_sum(components(kind, X1, X2, ls, scales), M)


def kmv_bound(kind, X1, X2, ls, scales, M, V) -> torch.Tensor:
    """Per-entry bound of |engine K.V - exact| (module docstring), fp64 [n1, t]."""
    X1, X2, V = X1.double(), X2.double(), V.double()
    D = X1.size(1)
    M = min(M, D)
    mean = X1.mean(0)
    C = CONST[kind]
    dK = torch.zeros(X1.size(0), X2.size(0), dtype=torch.float64, device=X1.device)
    cs = []
    for i in range(D):
        sc = math.sqrt(C) / float(ls[i])
        z1 = (X1[:, i] - mean[i]) * sc
        z2 = (X2[:, i] - mean[i]) * sc
        df = z1.reshape(-1, 1) - z2.reshape(1, -1)
        a = 0.5 * df * df
        dz = 3 * U * (z1.abs().reshape(-1, 1) + z2.abs().reshape(1, -1) + 2 * abs(float(mean[i])) * sc) + U * df.abs()
        k = component_cov(kind, X1[:, i], X2[:, i], float(ls[i]))
        L = math.log(2.0) * df.abs() if kind == "rbf" else torch.ones_like(df)
        dK = dK + float(scales[i]) * ((2.0 ** -21 + 9 * U * (1 + a)) * k + L * dz)
        cs.append(float(scales[i]) * k)
    P = 1.0 + (esym_sum(cs, M - 1) if M > 1 else 0.0)
    K = esym_sum(cs, M)
    dK = P * dK + (2 * D * M + M) * U * K
    n2 = X2.size(0)
    return (dK + (n2 + 2) * U * K) @ V.abs()
