"""Dense fp64 oracle of the RBF value / gradient covariance (RBFKernelGrad) over interleaved rows i (d+1) + a, written from the
block table: with D = x_i - x'_j, u_a = D_a / l_a^2 and k = s exp(-|D / l|^2 / 2),
    [0, 0] = k,   [0, b] = k u_b,   [a, 0] = -k u_a,   [a, b] = k (delta_ab / l_a^2 - u_a u_b).
Every function takes torch tensors and works in float64; the lengthscale is a scalar or a [d] vector.  Differentiable in the
lengthscale and outputscale (the gradient tests autograd through it)."""
import torch


def _ls(ls, d, device=None):
    ls = torch.as_tensor(ls, dtype=torch.float64, device=device).reshape(-1)
    return ls.expand(d) if ls.numel() == 1 else ls


def deriv_dense(x1, x2, ls, os=1.0):
    """[n1 (d+1), n2 (d+1)] fp64."""
    x1 = torch.as_tensor(x1).double()
    x2 = torch.as_tensor(x2).double()
    n1, d = x1.shape
    n2 = x2.shape[0]
    l = _ls(ls, d, x1.device)
    D = x1[:, None, :] - x2[None, :, :]                          # [n1, n2, d]
    u = D / l ** 2
    k = torch.exp(-0.5 * ((D / l) ** 2).sum(-1))                 # [n1, n2]
    K = torch.empty(n1, d + 1, n2, d + 1, dtype=torch.float64, device=x1.device)
    K[:, 0, :, 0] = k
    K[:, 0, :, 1:] = (k[..., None] * u)
    K[:, 1:, :, 0] = (-k[..., None] * u).permute(0, 2, 1)
    hess = torch.diag_embed((1.0 / l ** 2).expand(n1, n2, d)) - u[..., :, None] * u[..., None, :]
    K[:, 1:, :, 1:] = (k[..., None, None] * hess).permute(0, 2, 1, 3)
    return torch.as_tensor(os, dtype=torch.float64, device=x1.device) * K.reshape(n1 * (d + 1), n2 * (d + 1))


def deriv_diag(n, ls, d, os=1.0):
    """Interleaved diagonal of the square operator: s at value rows, s / l_a^2 at derivative rows."""
    l = _ls(ls, d)
    one = torch.cat([torch.ones(1, dtype=torch.float64), 1.0 / l ** 2])
    return torch.as_tensor(os, dtype=torch.float64) * one.repeat(n)


def deriv_majorant(x1, x2, ls, os=1.0):
    """|K| entrywise with |u_a| raised by 1 / l_a: |s k| (1, |u_b|', |u_a|', 1 / l_a^2 + |u_a|' |u_b|'), |u_a|' = |u_a| + 1 / l_a.
    The scale of every product's rounding error: u_a is formed from a rounded packed difference, whose absolute error is a small
    multiple of 2^-24 |z| (|z| = O(1)) in units of 1 / l_a, however small D_a is."""
    x1 = torch.as_tensor(x1).double()
    x2 = torch.as_tensor(x2).double()
    n1, d = x1.shape
    n2 = x2.shape[0]
    l = _ls(ls, d, x1.device)
    D = x1[:, None, :] - x2[None, :, :]
    u = (D / l ** 2).abs() + 1.0 / l
    k = torch.exp(-0.5 * ((D / l) ** 2).sum(-1))
    K = torch.empty(n1, d + 1, n2, d + 1, dtype=torch.float64, device=x1.device)
    K[:, 0, :, 0] = k
    K[:, 0, :, 1:] = k[..., None] * u
    K[:, 1:, :, 0] = (k[..., None] * u).permute(0, 2, 1)
    hess = torch.diag_embed((1.0 / l ** 2).expand(n1, n2, d)) + u[..., :, None] * u[..., None, :]
    K[:, 1:, :, 1:] = (k[..., None, None] * hess).permute(0, 2, 1, 3)
    return abs(float(os)) * K.reshape(n1 * (d + 1), n2 * (d + 1))


def franke(x, y):
    """The Franke function and its partial derivatives (the 2-d notebook's data): returns f, df/dx, df/dy."""
    x = torch.as_tensor(x, dtype=torch.float64)
    y = torch.as_tensor(y, dtype=torch.float64)
    t1 = 0.75 * torch.exp(-((9 * x - 2) ** 2) / 4 - ((9 * y - 2) ** 2) / 4)
    t2 = 0.75 * torch.exp(-((9 * x + 1) ** 2) / 49 - (9 * y + 1) / 10)
    t3 = 0.5 * torch.exp(-((9 * x - 7) ** 2) / 4 - ((9 * y - 3) ** 2) / 4)
    t4 = 0.2 * torch.exp(-((9 * x - 4) ** 2) - (9 * y - 7) ** 2)
    f = t1 + t2 + t3 - t4
    dx = (-2 * (9 * x - 2) * 9 / 4) * t1 + (-2 * (9 * x + 1) * 9 / 49) * t2 + (-2 * (9 * x - 7) * 9 / 4) * t3 - (-2 * (9 * x - 4) * 9) * t4
    dy = (-2 * (9 * y - 2) * 9 / 4) * t1 + (-9 / 10) * t2 + (-2 * (9 * y - 3) * 9 / 4) * t3 - (-2 * (9 * y - 7) * 9) * t4
    return f, dx, dy
