"""Dense fp64 oracle of the Matern-5/2 value / gradient covariance (Matern52KernelGrad) over interleaved rows i (d+1) + a, written
from the block table: with D = x_i - x'_j, u_a = D_a / l_a^2, rho = sqrt(5) |D / l|, e = exp(-rho), A = (5/3) (1 + rho) e and
B = (25/3) e (times the outputscale s),
    [0, 0] = (1 + rho + rho^2 / 3) e,   [0, b] = A u_b,   [a, 0] = -A u_a,   [a, b] = A delta_ab / l_a^2 - B u_a u_b.
Every function takes torch tensors and works in float64; the lengthscale is a scalar or a [d] vector.  Differentiable in the
lengthscale and outputscale, also at coincident points: there rho is the constant 0 (torch.where on a safe argument), which is
the true derivative (every entry's derivative in the lengthscale carries a factor q_c = (D_c / l_c)^2 = 0 at D = 0)."""
import torch


def _ls(ls, d, device=None):
    ls = torch.as_tensor(ls, dtype=torch.float64, device=device).reshape(-1)
    return ls.expand(d) if ls.numel() == 1 else ls


def _rho(r2):
    """sqrt(5 r^2) with a finite gradient at r^2 = 0 (where the true one is 0 times a bounded factor in every entry)."""
    safe = torch.where(r2 > 0, r2, torch.ones_like(r2))
    return torch.where(r2 > 0, torch.sqrt(5.0 * safe), torch.zeros_like(r2))


def m52grad_dense(x1, x2, ls, os=1.0):
    """[n1 (d+1), n2 (d+1)] fp64."""
    x1 = torch.as_tensor(x1).double()
    x2 = torch.as_tensor(x2).double()
    n1, d = x1.shape
    n2 = x2.shape[0]
    l = _ls(ls, d, x1.device)
    D = x1[:, None, :] - x2[None, :, :]                          # [n1, n2, d]
    u = D / l ** 2
    rho = _rho(((D / l) ** 2).sum(-1))                           # [n1, n2]
    e = torch.exp(-rho)
    A = (5.0 / 3.0) * (1 + rho) * e
    B = (25.0 / 3.0) * e
    K = torch.empty(n1, d + 1, n2, d + 1, dtype=torch.float64, device=x1.device)
    K[:, 0, :, 0] = (1 + rho + rho ** 2 / 3) * e
    K[:, 0, :, 1:] = A[..., None] * u
    K[:, 1:, :, 0] = (-A[..., None] * u).permute(0, 2, 1)
    hess = A[..., None, None] * torch.diag_embed((1.0 / l ** 2).expand(n1, n2, d)) - \
        B[..., None, None] * u[..., :, None] * u[..., None, :]
    K[:, 1:, :, 1:] = hess.permute(0, 2, 1, 3)
    return torch.as_tensor(os, dtype=torch.float64, device=x1.device) * K.reshape(n1 * (d + 1), n2 * (d + 1))


def m52grad_diag(n, ls, d, os=1.0):
    """Interleaved diagonal of the square operator: s at value rows, (5/3) s / l_a^2 at derivative rows."""
    l = _ls(ls, d)
    one = torch.cat([torch.ones(1, dtype=torch.float64), (5.0 / 3.0) / l ** 2])
    return torch.as_tensor(os, dtype=torch.float64) * one.repeat(n)


def m52grad_majorant(x1, x2, ls, os=1.0):
    """|K| entrywise with |u_a| raised by 1 / l_a and the rho terms by 1:  |s| (k0, A' |u_b|', A' |u_a|', A' / l_a^2 + B |u_a|' |u_b|')
    with |u_a|' = |u_a| + 1 / l_a and A' = (5/3) (2 + rho) e.  The scale of every product's rounding error: u_a is formed from a
    rounded packed difference (absolute error a small multiple of 2^-24 |z| in units of 1 / l_a however small D_a is), and rho from
    sqrt.approx of a rounded |dz|^2 / 2, whose absolute error is at most ~2^-22 (|z| = O(1)) plus a relative 2^-22 (DESIGN 4.16):
    a perturbation of rho by delta changes A by at most (5/3) rho e delta <= A' delta."""
    x1 = torch.as_tensor(x1).double()
    x2 = torch.as_tensor(x2).double()
    n1, d = x1.shape
    n2 = x2.shape[0]
    l = _ls(ls, d, x1.device)
    D = x1[:, None, :] - x2[None, :, :]
    u = (D / l ** 2).abs() + 1.0 / l
    rho = torch.sqrt(5.0 * ((D / l) ** 2).sum(-1))
    e = torch.exp(-rho)
    A = (5.0 / 3.0) * (2 + rho) * e
    B = (25.0 / 3.0) * e
    K = torch.empty(n1, d + 1, n2, d + 1, dtype=torch.float64, device=x1.device)
    K[:, 0, :, 0] = (1 + rho + rho ** 2 / 3) * e
    K[:, 0, :, 1:] = A[..., None] * u
    K[:, 1:, :, 0] = (A[..., None] * u).permute(0, 2, 1)
    hess = A[..., None, None] * torch.diag_embed((1.0 / l ** 2).expand(n1, n2, d)) + \
        B[..., None, None] * u[..., :, None] * u[..., None, :]
    K[:, 1:, :, 1:] = hess.permute(0, 2, 1, 3)
    return abs(float(os)) * K.reshape(n1 * (d + 1), n2 * (d + 1))
