"""The separable entry formula of the SKI operator that csrc/ski_rows.cuh evaluates (single rows and the diagonal of
K_ski = s W (T_0 x ... x T_{d-1}) W^T without a product with the operator), restated in fp64 from oracle/ski.py's interpolation
and Toeplitz columns, against the oracle's dense product ski_matmul(..., I):

    K_ski(i, j) = s prod_k a_k(i, j),   a_k(i, j) = sum_b w_jk[b] u_k[f_jk + b],   u_k = T_k[:, f_ik : f_ik + 4] w_ik

Both sides are fp64 restatements of the same operator that differ only in the order of the sums (the dense product runs through
a circulant FFT per mode), so they agree to a small multiple of 2^-53 relative to max |K|; 1e-12 leaves room for the FFTs.
"""
import pytest
import torch

from oracle import ski


def per_dim_interp(axes, x):
    """(first [n, d] int64, weights [n, d, 4]) from oracle.ski.interpolate run one dimension at a time (the 1-D indices are the
    node numbers, and the d-dimensional weights are their products)."""
    firsts, wts = [], []
    for k, g in enumerate(axes):
        idx, val = ski.interpolate([g], x[:, k:k + 1])
        firsts.append(idx[:, 0])
        wts.append(val)
    return torch.stack(firsts, 1), torch.stack(wts, 1)


def toeplitz_factors(kind, axes, lengthscale):
    """Dense T_k [G_k, G_k] from the oracle's first columns."""
    out = []
    for col in ski.grid_toeplitz_columns(kind, axes, lengthscale):
        g = col.numel()
        ar = torch.arange(g)
        out.append(col[(ar[:, None] - ar[None, :]).abs()])
    return out


def separable_rows(kind, x, axes, lengthscale, outputscale, rows):
    """K_ski[rows, :] by the row formula (u_k of each requested row, 4 products per dimension and entry)."""
    first, w = per_dim_interp(axes, x)
    T = toeplitz_factors(kind, axes, lengthscale)
    ar4 = torch.arange(4)
    out = torch.full((len(rows), x.size(0)), float(outputscale), dtype=torch.float64)
    for r, i in enumerate(rows):
        for k, Tk in enumerate(T):
            u = Tk[:, first[i, k] + ar4] @ w[i, k]
            out[r] *= (w[:, k] * u[first[:, k, None] + ar4]).sum(-1)
    return out


def separable_diag(kind, x, axes, lengthscale, outputscale):
    """diag K_ski: w_ik^T T_k[f_ik : f_ik + 4, f_ik : f_ik + 4] w_ik per dimension."""
    first, w = per_dim_interp(axes, x)
    T = toeplitz_factors(kind, axes, lengthscale)
    ar4 = torch.arange(4)
    out = torch.full((x.size(0),), float(outputscale), dtype=torch.float64)
    for k, Tk in enumerate(T):
        f = first[:, k, None] + ar4
        blk = Tk[f[:, :, None], f[:, None, :]]                      # [n, 4, 4]
        out *= torch.einsum("na,nab,nb->n", w[:, k], blk, w[:, k])
    return out


def special_points(axes, n, seed):
    """n points in the grid's interior, with some in the first / last cell (one-hot snapping) and some exactly on nodes."""
    g = torch.Generator().manual_seed(seed)
    d = len(axes)
    lo = torch.tensor([float(a[0]) for a in axes], dtype=torch.float64)
    hi = torch.tensor([float(a[-1]) for a in axes], dtype=torch.float64)
    step = torch.tensor([float(a[1] - a[0]) for a in axes], dtype=torch.float64)
    x = lo + step + torch.rand(n, d, generator=g, dtype=torch.float64) * (hi - lo - 2 * step)
    x[:5] = lo + torch.rand(5, d, generator=g, dtype=torch.float64) * step * 0.999
    x[5:10] = hi - torch.rand(5, d, generator=g, dtype=torch.float64) * step * 0.999
    x[10] = torch.stack([a[min(3, a.numel() - 1)] for a in axes])
    x[11] = torch.stack([a[a.numel() // 2] for a in axes])
    return x


CASES = [
    (1, [24], "rbf", [0.3]), (1, [4], "matern12", [0.5]), (2, [12, 9], "matern32", [0.25, 0.6]),
    (3, [8, 7, 6], "matern52", [0.4]), (4, [6, 5, 6, 5], "rbf", [0.3, 0.5, 0.4, 0.7]), (2, [30, 30], "matern12", [0.2]),
]


@pytest.mark.parametrize("d,sizes,kind,ls", CASES)
def test_separable_rows_and_diagonal_match_dense_ski(d, sizes, kind, ls):
    axes = ski.create_grid(sizes, [(0.0, 1.0)] * d, dtype=torch.float64)
    n = 120
    x = special_points(axes, n, seed=d * 7 + sizes[0])
    lsv = ls[0] if len(ls) == 1 else torch.tensor(ls, dtype=torch.float64)
    dense = ski.ski_matmul(kind, x, axes, lsv, 1.3, torch.eye(n, dtype=torch.float64))
    scale = float(dense.abs().max())
    rows = [0, 4, 6, 9, 10, 11, n - 1]
    got = separable_rows(kind, x, axes, lsv, 1.3, rows)
    assert float((got - dense[rows]).abs().max()) <= 1e-12 * scale
    dg = separable_diag(kind, x, axes, lsv, 1.3)
    assert float((dg - dense.diagonal()).abs().max()) <= 1e-12 * scale
    assert float((dg[rows] - got[:, rows].diagonal()).abs().max()) <= 1e-12 * scale   # the row formula at j = i is the diagonal


def test_ski_preconditioner_is_off_by_default():
    from gpytorch_b200 import settings

    assert settings.ski_preconditioner.off()
    with settings.ski_preconditioner(True):
        assert settings.ski_preconditioner.on()
    assert settings.ski_preconditioner.off()
    assert settings.ski_preconditioner in settings.snapshot()
