"""fp64 restatement of KISS-GP prediction on the grid (InterpolatedPredictionStrategy,
gpytorch/models/exact_prediction_strategies.py:481-827), built only from the pinned pieces of oracle/ski.py:
`interpolate` (checked against the reference's own interpolation code), `left_t_interp`, `left_interp` and
`kron_toeplitz_matmul`.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

    c   = s K_uu W^T alpha                 mean_cache (:578-606), alpha = K_hat^{-1} (y - mu)
    C   = s K_uu W^T R                     covar_cache (:490-503, :679-746), R R^T ~= K_hat^{-1}
    mean = W* c                            exact_predictive_mean (:780-786), without the prior mean
    U    = W* C,  covar = K**_test - U U^T exact_predictive_covar under fast_pred_var (:788-827)

`interp_dtype` (default: the inputs' dtype) is the precision of the interpolation step only: with torch.float32 the weights
are those the reference computes for fp32 data (the grid coordinate (x - u_0) / spacing rounded in fp32, as a fp32 engine
computes it), promoted to the inputs' dtype for everything after.
"""
from __future__ import annotations

from functools import reduce
from operator import mul

import torch

from . import ski


def _interp(grid_axes, x, interp_dtype=None):
    dt = interp_dtype or x.dtype
    idx, val = ski.interpolate([a.to(dt) for a in grid_axes], x.to(dt))
    return idx, val.to(x.dtype)


def _kuu_apply(kind, grid_axes, lengthscale, outputscale, u):
    cols = ski.grid_toeplitz_columns(kind, grid_axes, lengthscale)
    return outputscale * ski.kron_toeplitz_matmul(cols, u)


def grid_matmul(kind, x, grid_axes, lengthscale, outputscale, v, interp_dtype=None):
    """s K_uu W^T v for v [n, t] over the points x: [M, t] in the flat grid order (dimension 0 slowest)."""
    idx, val = _interp(grid_axes, x, interp_dtype)
    M = reduce(mul, [int(g.numel()) for g in grid_axes], 1)
    return _kuu_apply(kind, grid_axes, lengthscale, outputscale, ski.left_t_interp(idx, val, v, M))


def interp_matmul(grid_axes, x, c, interp_dtype=None):
    """W c for grid values c [M, t]: [n, t]."""
    idx, val = _interp(grid_axes, x, interp_dtype)
    return ski.left_interp(idx, val, c)


def dense_covariance(kind, x, grid_axes, lengthscale, outputscale, interp_dtype=None):
    """s W K_uu W^T over the points x, symmetrised."""
    n = x.size(0)
    K = interp_matmul(grid_axes, x, grid_matmul(kind, x, grid_axes, lengthscale, outputscale, torch.eye(n, dtype=x.dtype),
                                                interp_dtype), interp_dtype)
    return 0.5 * (K + K.T)


def interpolated_prediction(kind, x, xt, y, grid_axes, lengthscale, outputscale, noise, R, interp_dtype=None):
    """The grid caches and the predictive moments of a KISS-GP model, all in the dtype of the inputs (fp64 for parity).

    x [n, d] training points, xt [m, d] test points, y [n] the training residuals y - mu(x), noise a scalar or a per-row [n]
    vector, R [n, J] the LOVE root (R R^T ~= K_hat^{-1}; the caller supplies the model's own).  Returns a dict with alpha, c, C,
    mean (= W* c, prior mean not added), U (= W* C), Kss (the test-test SKI covariance, dense) and covar (= Kss - U U^T)."""
    n = x.size(0)
    eye = torch.eye(n, dtype=x.dtype)
    K = dense_covariance(kind, x, grid_axes, lengthscale, outputscale, interp_dtype)
    nz = torch.as_tensor(noise, dtype=x.dtype)
    Khat = K + (torch.diag(nz) if nz.dim() == 1 else nz * eye)
    alpha = torch.linalg.solve(Khat, y.reshape(n, 1))
    c = grid_matmul(kind, x, grid_axes, lengthscale, outputscale, alpha, interp_dtype)
    C = grid_matmul(kind, x, grid_axes, lengthscale, outputscale, R, interp_dtype)
    mean = interp_matmul(grid_axes, xt, c, interp_dtype)[:, 0]
    U = interp_matmul(grid_axes, xt, C, interp_dtype)
    Kss = dense_covariance(kind, xt, grid_axes, lengthscale, outputscale, interp_dtype)
    return {"alpha": alpha[:, 0], "c": c[:, 0], "C": C, "mean": mean, "U": U, "Kss": Kss, "covar": Kss - U @ U.T}
