"""fp64 restatement of the piecewise polynomial kernel, of the compact-support backend's schedule (Morton order, tile boxes, tile-pair
lists) and the per-entry bound of its K.V.

    K(x, x') = S (1 - r)_+^(j+q) poly_q(r),   r = |(x - x') / l|,   j = floor(D / 2) + q + 1

with the reference module's polynomials (kernels/piecewise_polynomial_kernel.py), whose q = 2 coefficient is (j + 4 j + 3) / 3 where
R&W eq. 4.21 has (j^2 + 4 j + 3) / 3.

Bound derivation (u = 2^-24).  The engine packs z = (x - mean) * fp32(1 / l): each coordinate carries a relative error of at most 3u,
and both points of a pair share the mean, so a difference df_c = z_ic - z_jc is off by at most 4u (|z_ic| + |z_jc|) + u |df_c|.  By
the triangle inequality r moves by at most the sum of those, and the fp32 sum of squares and the IEEE sqrt add (D + 3) u r.  An
entry then moves by at most max|k'| dr; its evaluation (1 - r rounded, e - 1 multiplies, the Horner polynomial of positive terms with
fp32 coefficients) adds (e + 12) u k.  A pair with r >= 1 + dr is an exact 0 on both sides.  The row sum over m evaluated columns
adds (m + 4) u sum_j k |v_j| (fp32 sums in any order, the slots, the outputscale).  The bound is doubled.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U32 = 2.0 ** -24
PP_TI, PP_TJ = 128, 64
PP_REACH2 = 1.0 + 1.0 / 1048576.0


def coeffs(q: int, D: int, textbook: bool = False):
    """(e, [c1, c2, c3]) of poly_q(r) = 1 + c1 r + c2 r^2 + c3 r^3; textbook=True gives R&W's q = 2 coefficient."""
    j = D // 2 + q + 1
    c = [0.0, 0.0, 0.0]
    if q == 1:
        c[0] = j + 1.0
    elif q == 2:
        c[0] = j + 2.0
        c[1] = (j * j + 4 * j + 3) / 3.0 if textbook else (j + 4 * j + 3) / 3.0
    elif q == 3:
        c[0] = j + 3.0
        c[1] = (6 * j * j + 36 * j + 45) / 15.0
        c[2] = (j ** 3 + 9 * j * j + 23 * j + 15) / 15.0
    return j + q, c


def kernel_r(r, q: int, D: int):
    e, c = coeffs(q, D)
    m = torch.clamp(1.0 - r, min=0.0)
    return m ** e * (1.0 + r * (c[0] + r * (c[1] + r * c[2])))


def dist(x1, x2, ls):
    ls = torch.as_tensor(ls, dtype=torch.float64, device=x1.device).reshape(-1)
    return torch.cdist(x1.double() / ls, x2.double() / ls)


def kernel(x1, x2, ls, q: int, S=1.0):
    """K [n1, n2] in fp64 (direct differences: the diagonal of K(x, x) is exactly S)."""
    x1, x2 = x1.double(), x2.double()
    ls = torch.as_tensor(ls, dtype=torch.float64, device=x1.device).reshape(-1)
    d = (x1[:, None, :] - x2[None, :, :]) / ls
    r = torch.sqrt((d * d).sum(-1))
    return S * kernel_r(r, q, x1.size(1))


def max_slope(q: int, D: int) -> float:
    """max over [0, 1] of |k'(r)| (fp64 grid, 10 % margin)."""
    r = torch.linspace(0.0, 1.0, 20001, dtype=torch.float64, requires_grad=True)
    k = kernel_r(r, q, D)
    (g,) = torch.autograd.grad(k.sum(), r)
    return 1.1 * float(g.abs().max())


def kmv_bound(x1, x2, ls, q: int, S: float, v, mean=None):
    """Per-entry bound [n1, t] of the engine's S K V against the fp64 product (module docstring)."""
    x1, x2, v = x1.double(), x2.double(), v.double()
    D = x1.size(1)
    ls = torch.as_tensor(ls, dtype=torch.float64, device=x1.device).reshape(-1)
    if mean is None:
        mean = x1.mean(0)
    z1, z2 = (x1 - mean) / ls, (x2 - mean) / ls
    dfa = (z1[:, None, :] - z2[None, :, :]).abs()
    r = torch.sqrt((dfa * dfa).sum(-1))
    dr = (4 * U32 * (z1.abs()[:, None, :] + z2.abs()[None, :, :]) + U32 * dfa).sum(-1) + (D + 3) * U32 * r
    e, _ = coeffs(q, D)
    k = kernel_r(r, q, D)
    near = (r < 1.0 + dr).double()
    kv = k @ v.abs()
    per = (max_slope(q, D) * dr * near) @ v.abs() + (e + 12) * U32 * kv
    m = near.sum(1, keepdim=True)
    return 2.0 * S * (per + (m + 4) * U32 * kv) + 1e-30


def grads(x1, x2, ls, q: int, S: float, L, R):
    """d/dl (shape of ls) and d/dS of sum(L * (S K R)) by fp64 autograd through the dense kernel."""
    ls_t = torch.tensor(np.asarray(ls, dtype=np.float64).reshape(-1), requires_grad=True)
    S_t = torch.tensor(float(S), dtype=torch.float64, requires_grad=True)
    x1, x2 = x1.double().cpu(), x2.double().cpu()
    d = (x1[:, None, :] - x2[None, :, :]) / ls_t
    r2 = (d * d).sum(-1)
    r = torch.sqrt(torch.where(r2 > 0, r2, torch.ones_like(r2)))
    k = torch.where(r2 > 0, kernel_r(r, q, x1.size(1)), torch.ones_like(r2))
    F = (L.double().cpu() * (S_t * k @ R.double().cpu())).sum()
    gl, gs = torch.autograd.grad(F, (ls_t, S_t))
    return gl.numpy(), float(gs)


# ---- the schedule, as compact.cu forms it -----------------------------------------------------------------------------------
def key_bits(d: int) -> int:
    return min(20, 60 // d)


def morton_perm(X: np.ndarray) -> np.ndarray:
    """Sorted position -> row: a stable sort of the Morton keys of the raw fp32 inputs (pp_key_kernel)."""
    X = np.asarray(X, dtype=np.float32)
    n, d = X.shape
    bits = key_bits(d)
    cells = float(1 << bits)
    keys = np.zeros(n, dtype=np.uint64)
    for c in range(d):
        col = X[:, c]
        fin = np.isfinite(col)
        if fin.any():
            lo, hi = float(col[fin].min()), float(col[fin].max())
        else:
            lo, hi = math.inf, -math.inf
        cell = np.zeros(n, dtype=np.uint64)
        if hi > lo:
            t = ((col.astype(np.float64) - lo) / (hi - lo)) * cells
            ok = fin
            tt = np.where(ok, t, 0.0)
            cc = np.where(tt >= cells, (1 << bits) - 1, np.floor(tt)).astype(np.uint64)
            cell = np.where(ok, cc, 0).astype(np.uint64)
        for b in range(bits):
            keys |= ((cell >> np.uint64(b)) & np.uint64(1)) << np.uint64(b * d + c)
    return np.argsort(keys, kind="stable")


def boxes(X: np.ndarray, perm: np.ndarray, tile: int) -> np.ndarray:
    """[ntile, 2, d] raw fp32 lo / hi of every tile of sorted points (non-finite values ignored)."""
    Xs = np.asarray(X, dtype=np.float32)[perm]
    n, d = Xs.shape
    nt = -(-n // tile)
    out = np.empty((nt, 2, d), dtype=np.float32)
    with np.errstate(invalid="ignore"):
        for t in range(nt):
            blk = Xs[t * tile:(t + 1) * tile]
            blk_lo = np.where(np.isnan(blk), np.inf, blk)
            blk_hi = np.where(np.isnan(blk), -np.inf, blk)
            out[t, 0] = blk_lo.min(0)
            out[t, 1] = blk_hi.max(0)
    return out


def reach(b1: np.ndarray, b2: np.ndarray, ls) -> np.ndarray:
    """[nt1, nt2] whether a row tile and a column tile are listed (pp_reach: fp64, dimension order, fmax)."""
    d = b1.shape[2]
    ls = np.broadcast_to(np.asarray(ls, dtype=np.float32).astype(np.float64).reshape(-1), (d,))
    s = np.zeros((b1.shape[0], b2.shape[0]))
    with np.errstate(invalid="ignore"):
        for c in range(d):
            g1 = b2[None, :, 0, c].astype(np.float64) - b1[:, None, 1, c].astype(np.float64)
            g2 = b1[:, None, 0, c].astype(np.float64) - b2[None, :, 1, c].astype(np.float64)
            g = np.fmax(np.fmax(g1, g2), 0.0)
            u = g / ls[c]
            s = s + u * u
    return s < PP_REACH2


def schedule(X1: np.ndarray, X2: np.ndarray | None, ls):
    """(perm1, perm2, reach [nt1, nt2]) of a square (X2 None) or cross plan."""
    perm1 = morton_perm(X1)
    perm2 = perm1 if X2 is None else morton_perm(X2)
    b1 = boxes(X1, perm1, PP_TI)
    b2 = boxes(X1 if X2 is None else X2, perm2, PP_TJ)
    return perm1, perm2, reach(b1, b2, ls)


def uncovered_pairs(X1: np.ndarray, X2: np.ndarray | None, ls) -> int:
    """Pairs with fp64 r < 1 whose tile pair is not listed (must be 0)."""
    perm1, perm2, R = schedule(X1, X2, ls)
    X2_ = X1 if X2 is None else X2
    pos1 = np.empty(len(perm1), dtype=np.int64)
    pos1[perm1] = np.arange(len(perm1))
    pos2 = np.empty(len(perm2), dtype=np.int64)
    pos2[perm2] = np.arange(len(perm2))
    ls64 = np.asarray(ls, dtype=np.float32).astype(np.float64).reshape(-1)
    a = np.asarray(X1, dtype=np.float32).astype(np.float64) / ls64
    b = np.asarray(X2_, dtype=np.float32).astype(np.float64) / ls64
    r = np.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1))
    ii, jj = np.nonzero(r < 1.0)
    return int((~R[pos1[ii] // PP_TI, pos2[jj] // PP_TJ]).sum())


def count_pairs(X1: np.ndarray, X2: np.ndarray | None, ls, rows_per_chunk: int = 256) -> int:
    """The number of listed tile pairs, in row-tile chunks (no ntile_i x ntile_j array at large N)."""
    perm1 = morton_perm(X1)
    perm2 = perm1 if X2 is None else morton_perm(X2)
    b1 = boxes(X1, perm1, PP_TI)
    b2 = boxes(X1 if X2 is None else X2, perm2, PP_TJ)
    return int(sum(reach(b1[t:t + rows_per_chunk], b2, ls).sum() for t in range(0, b1.shape[0], rows_per_chunk)))
