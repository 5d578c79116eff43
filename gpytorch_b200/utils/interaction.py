"""gpytorch.utils.sum_interaction_terms for the accelerated path (the reference: utils/sum_interaction_terms.py)."""
from __future__ import annotations

import torch


def dense_interaction_terms(covars: torch.Tensor, max_degree: int) -> torch.Tensor:
    """sum_{m=1}^{M} e_m(K_1, .., K_D) entry by entry for covars [D, ...], by the positive recurrence e_m += K_i e_{m-1} (the same
    arithmetic as the engine's kernels; no alternating signs)."""
    D = covars.size(0)
    M = min(int(max_degree), D)
    e = [torch.ones_like(covars[0])] + [torch.zeros_like(covars[0]) for _ in range(M)]
    for i in range(D):
        for m in range(M, 0, -1):
            e[m] = e[m] + covars[i] * e[m - 1]
    out = e[1]
    for m in range(2, M + 1):
        out = out + e[m]
    return out


def sum_interaction_terms(covars, max_degree: int | None = None, dim: int = -3):
    """Sum of D covariances K_1 .. K_D (the batch dimension `dim`) and of all their interaction terms up to degree max_degree
    (None: D), i.e. sum_{m=1}^{M} e_m(K_1, .., K_D) with e_m the elementary symmetric polynomial of degree m taken entry by entry
    (Duvenaud et al., Additive Gaussian Processes).

    A BatchLinearOperator of D one-dimensional RBF / Matern kernel operators (`ScaleKernel(RBFKernel(batch_shape=[D],
    ard_num_dims=1))(X.mT.unsqueeze(-1))`) becomes ONE engine operator (operators.AdditiveKernelLinearOperator, dim -3 only); a
    dense tensor [..., D, N, N] is combined in torch by the same recurrence.  dim must be negative, as in the reference."""
    from ..operators import AdditiveKernelLinearOperator, BatchLinearOperator, _additive_components

    if dim >= 0:
        raise ValueError("Argument 'dim' must be a negative integer.")
    if max_degree is not None and int(max_degree) < 1:
        raise ValueError(f"max_degree must be >= 1 (got {max_degree})")
    if isinstance(covars, BatchLinearOperator):
        if dim != -3:
            raise NotImplementedError(f"sum_interaction_terms over dim={dim} of a BatchLinearOperator: only its batch dimension (-3) "
                                      "is available on the accelerated path")
        ops = _additive_components(covars.ops, "sum_interaction_terms")
        return AdditiveKernelLinearOperator(ops, len(ops) if max_degree is None else max_degree)
    if torch.is_tensor(covars):
        if covars.dim() < -dim:
            raise ValueError(f"sum_interaction_terms: covars of shape {tuple(covars.shape)} has no dimension {dim}")
        c = covars.movedim(dim, 0)
        return dense_interaction_terms(c, c.size(0) if max_degree is None else max_degree)
    raise NotImplementedError(f"sum_interaction_terms takes a BatchLinearOperator of kernel operators or a dense tensor, not "
                              f"{type(covars).__name__}")
