"""fp64 dense reference of the Hadamard multitask GP (IndexKernel times a data kernel, per-task noise), as the reference builds it
in examples/03_Multitask_Exact_GPs/Hadamard_Multitask_GP_Regression.ipynb:

    K_hat[i, j] = s k(x_i, x_j) B[t_i, t_j] + sigma^2_{t_i} delta_ij,   B = F F^T + diag(v)   (kernels/index_kernel.py:91-117)

Everything is dense and differentiable (torch autograd), so it doubles as the gradient reference.
"""
import math

import torch

from oracle import kernels as ok


def index_covar(covar_factor: torch.Tensor, var: torch.Tensor) -> torch.Tensor:
    """IndexKernel.covar_matrix: F F^T + diag(v)."""
    return covar_factor @ covar_factor.transpose(-1, -2) + torch.diag_embed(var)


def hadamard_matrix(kind, x1, x2, t1, t2, lengthscale, outputscale, B, x1_eq_x2=None):
    """s K(x1, x2) o B[t1, t2]."""
    k = ok.kernel_matrix(kind, x1, x2, lengthscale, outputscale, x1_eq_x2)
    return k * B[t1.long()][:, t2.long()]


def khat(kind, x, t, lengthscale, outputscale, B, task_noise):
    n = x.size(0)
    K = hadamard_matrix(kind, x, x, t, t, lengthscale, outputscale, B, True)
    return K + torch.diag(task_noise[t.long()])


def mll(kind, x, t, y, lengthscale, outputscale, B, task_noise, mean=0.0):
    """ExactMarginalLogLikelihood / n of the Hadamard model (exact Cholesky, fp64)."""
    A = khat(kind, x, t, lengthscale, outputscale, B, task_noise)
    L = torch.linalg.cholesky(A)
    r = (y - mean).unsqueeze(-1)
    a = torch.cholesky_solve(r, L)
    n = y.numel()
    inv_quad = (r * a).sum()
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    return -0.5 * (inv_quad + logdet + n * math.log(2 * math.pi)) / n


def posterior(kind, x, t, y, xs, ts, lengthscale, outputscale, B, task_noise, mean=0.0):
    """Posterior mean and covariance of the latent f at (xs, ts)."""
    A = khat(kind, x, t, lengthscale, outputscale, B, task_noise)
    Ksx = hadamard_matrix(kind, xs, x, ts, t, lengthscale, outputscale, B, False)
    Kss = hadamard_matrix(kind, xs, xs, ts, ts, lengthscale, outputscale, B, True)
    L = torch.linalg.cholesky(A)
    alpha = torch.cholesky_solve((y - mean).unsqueeze(-1), L).squeeze(-1)
    W = torch.cholesky_solve(Ksx.transpose(0, 1), L)
    return mean + Ksx @ alpha, Kss - Ksx @ W
