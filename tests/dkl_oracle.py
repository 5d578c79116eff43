"""fp64 closed form of the SKI input gradient (gp_ski_input_grad) for the DKL tests.

F = sum_i L_i . (K_ski R)_i, K_ski = s W K_uu W^T.  Only W moves with x, row i with x_i alone:
  dF/dx_ik = sum_c [ L_ic (d_k W_i B_R)_c + R_ic (d_k W_i B_L)_c ],  B_R = s K_uu W^T R,  B_L = s K_uu W^T L,
d_k W_i = row i's tensor-product weights with the dimension-k factor replaced by its derivative.  The per-axis weights are the
Keys cubic kernel of oracle/ski.py; their derivative is written out here (sign(s) (4.5 u^2 - 5 u) for u < 1, sign(s) (-1.5 u^2 +
5 u - 4) for 1 <= u < 2, times 1 / step), and exactly 0 in the one-hot first / last cells.
"""
from functools import reduce
from operator import mul

import torch

from oracle import ski

NPT = 4


def cubic_dw(s):
    u = s.abs()
    v = torch.where(u < 1, (4.5 * u - 5.0) * u, (-1.5 * u + 5.0) * u - 4.0)
    return torch.sign(s) * v


def axis_weights(g, x):
    """(first node [n] int64, w [n, 4], dw [n, 4]) of coordinates x [n] on grid axis g (fp64), the cell choice of oracle/ski.py."""
    G = g.numel()
    h = (g[1] - g[0]).clamp_min(1e-10)
    t = (x - g[0]) / h
    cell = torch.floor(t)
    frac = t - cell
    first = cell - 1
    s = frac.unsqueeze(-1) + torch.tensor([1.0, 0.0, -1.0, -2.0], dtype=x.dtype)
    w = ski.cubic_interp_weights(s)
    dw = cubic_dw(s) / h
    for edge, base, nodes in ((first < 0, 0, g[:NPT]), (first > G - NPT, G - NPT, g[-NPT:])):
        if bool(edge.any()):
            near = (nodes.unsqueeze(0) - x[edge].unsqueeze(1)).abs().argmin(1)
            w[edge] = torch.nn.functional.one_hot(near, NPT).to(w)
            dw[edge] = 0.0
            first = torch.where(edge, torch.full_like(first, base), first)
    return first.long(), w, dw


def interp_with_derivatives(axes, x):
    """(idx [n, 4^d], val [n, 4^d], dval [d, n, 4^d]) in oracle/ski.interpolate's column order (dimension 0 most significant)."""
    n, d = x.shape
    sizes = [int(g.numel()) for g in axes]
    per = [axis_weights(g, x[:, i]) for i, g in enumerate(axes)]
    idx = torch.zeros(n, 1, dtype=torch.long)
    val = torch.ones(n, 1, dtype=x.dtype)
    dval = [torch.ones(n, 1, dtype=x.dtype) for _ in range(d)]
    for i, (f, w, dw) in enumerate(per):
        stride = reduce(mul, sizes[i + 1:], 1)
        idx = (idx.unsqueeze(-1) + ((f.unsqueeze(-1) + torch.arange(NPT)) * stride).unsqueeze(1)).reshape(n, -1)
        val = (val.unsqueeze(-1) * w.unsqueeze(1)).reshape(n, -1)
        dval = [(dv.unsqueeze(-1) * (dw if k == i else w).unsqueeze(1)).reshape(n, -1) for k, dv in enumerate(dval)]
    return idx, val, torch.stack(dval)


def ski_input_grad(kind, x, axes, lengthscale, outputscale, L, R):
    """dF/dx [n, d] in fp64, and the same formula with every factor replaced by its absolute value (the scale of the fp32 error)."""
    idx, val, dval = interp_with_derivatives(axes, x)
    M = reduce(mul, [int(g.numel()) for g in axes], 1)
    cols = ski.grid_toeplitz_columns(kind, axes, lengthscale)
    out, mag = [], []
    acols = [c.abs() for c in cols]
    BR = outputscale * ski.kron_toeplitz_matmul(cols, ski.left_t_interp(idx, val, R, M))
    BL = outputscale * ski.kron_toeplitz_matmul(cols, ski.left_t_interp(idx, val, L, M))
    aBR = outputscale * ski.kron_toeplitz_matmul(acols, ski.left_t_interp(idx, val.abs(), R.abs(), M))
    aBL = outputscale * ski.kron_toeplitz_matmul(acols, ski.left_t_interp(idx, val.abs(), L.abs(), M))
    for k in range(x.size(1)):
        out.append((L * ski.left_interp(idx, dval[k], BR)).sum(-1) + (R * ski.left_interp(idx, dval[k], BL)).sum(-1))
        mag.append((L.abs() * ski.left_interp(idx, dval[k].abs(), aBR)).sum(-1)
                   + (R.abs() * ski.left_interp(idx, dval[k].abs(), aBL)).sum(-1))
    return torch.stack(out, -1), torch.stack(mag, -1)


def dense_ski(kind, x, axes, lengthscale, outputscale):
    """s W K_uu W^T as a dense fp64 matrix, differentiable in x through oracle/ski.interpolate (autograd reference)."""
    idx, val = ski.interpolate(axes, x)
    M = reduce(mul, [int(g.numel()) for g in axes], 1)
    W = torch.zeros(x.size(0), M, dtype=x.dtype).scatter_add(1, idx, val)
    cols = ski.grid_toeplitz_columns(kind, axes, lengthscale)
    return outputscale * W @ ski.kron_toeplitz_matmul(cols, W.t().contiguous())
