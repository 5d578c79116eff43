"""fp64 dense reference of the Kronecker multitask GP (MultitaskKernel, MultitaskGaussianLikelihood with rank 0), as the reference
builds it in examples/03_Multitask_Exact_GPs/Multitask_GP_Regression.ipynb:

    K_hat[i T + a, j T + b] = s k(x_i, x_j) B[a, b] + (sigma^2 + sigma^2_a) delta_ij delta_ab,   B = F F^T + diag(v)

(KroneckerProductLinearOperator(covar_x, covar_i), interleaved rows).  Everything is dense and differentiable (torch autograd), so
it doubles as the gradient reference.
"""
import math

import torch

from oracle import kernels as ok


def index_covar(covar_factor: torch.Tensor, var: torch.Tensor) -> torch.Tensor:
    """IndexKernel.covar_matrix: F F^T + diag(v)."""
    return covar_factor @ covar_factor.transpose(-1, -2) + torch.diag_embed(var)


def kron_matrix(kind, x1, x2, lengthscale, outputscale, B, x1_eq_x2=None):
    """(s K(x1, x2)) (x) B, row i T + a."""
    k = ok.kernel_matrix(kind, x1, x2, lengthscale, outputscale, x1_eq_x2)
    return torch.kron(k, B)


def noise_diag(n, task_noises, noise):
    """sigma^2 + sigma^2_a at row i T + a."""
    return (task_noises + noise).repeat(n)


def khat(kind, x, lengthscale, outputscale, B, task_noises, noise):
    return kron_matrix(kind, x, x, lengthscale, outputscale, B, True) + torch.diag(noise_diag(x.size(0), task_noises, noise))


def mll(kind, x, y, lengthscale, outputscale, B, task_noises, noise, mean=0.0):
    """ExactMarginalLogLikelihood / (n T) of the Kronecker model; y and mean [n, T] (exact Cholesky, fp64)."""
    A = khat(kind, x, lengthscale, outputscale, B, task_noises, noise)
    L = torch.linalg.cholesky(A)
    r = (y - mean).reshape(-1, 1)
    a = torch.cholesky_solve(r, L)
    N = r.numel()
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    return -0.5 * ((r * a).sum() + logdet + N * math.log(2 * math.pi)) / N


def posterior(kind, x, y, xs, lengthscale, outputscale, B, task_noises, noise, mean=0.0, mean_s=0.0):
    """Posterior mean [m, T] and covariance [m T, m T] of the latent f at xs."""
    T = B.shape[-1]
    A = khat(kind, x, lengthscale, outputscale, B, task_noises, noise)
    Ksx = kron_matrix(kind, xs, x, lengthscale, outputscale, B, False)
    Kss = kron_matrix(kind, xs, xs, lengthscale, outputscale, B, True)
    L = torch.linalg.cholesky(A)
    alpha = torch.cholesky_solve((y - mean).reshape(-1, 1), L).squeeze(-1)
    W = torch.cholesky_solve(Ksx.transpose(0, 1), L)
    mu = (Ksx @ alpha).reshape(-1, T) + mean_s
    return mu, Kss - Ksx @ W


def pivoted_cholesky(A, rank):
    """Greedy pivoted Cholesky of a dense PSD matrix (first pivot = argmax of the diagonal, earliest on ties): (L^T [k, n], pivots)."""
    n = A.size(0)
    d = torch.diagonal(A).clone()
    Lt = torch.zeros(rank, n, dtype=A.dtype)
    piv = []
    for m in range(rank):
        i = int(torch.argmax(d))
        piv.append(i)
        row = A[i] - Lt[:m, i] @ Lt[:m]
        Lt[m] = row / math.sqrt(float(d[i]))
        d = d - Lt[m] ** 2
        d[piv] = -math.inf
    return Lt, piv
