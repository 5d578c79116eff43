"""Function seam: the reference's functional entry points with their signatures.

linear_cg mirrors linear_operator.utils.linear_cg (call shape attested at
gpytorch/variational/ciq_variational_strategy.py:56-64; tests patch "linear_operator.utils.linear_cg",
test/lazy/test_lazy_evaluated_kernel_tensor.py:82-83), restricted to operators the engine owns:
`matmul_closure` must be (the bound matmul of) an AddedDiagLinearOperator / KernelLinearOperator.
"""
import torch

from . import settings
from .operators import AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator, RootLinearOperator
from .sampling import psd_safe_cholesky


def _as_operator(obj):
    if isinstance(obj, AddedDiagLinearOperator):
        return obj
    if isinstance(obj, KernelLinearOperator):
        return AddedDiagLinearOperator(obj, ConstantDiagLinearOperator(torch.zeros((), device=obj.device), obj.shape[0]))
    owner = getattr(obj, "__self__", None)
    if owner is not None:
        return _as_operator(owner)
    raise RuntimeError("linear_cg: matmul_closure must be an engine operator (KernelLinearOperator / AddedDiagLinearOperator)")


def linear_cg(matmul_closure, rhs, n_tridiag=0, tolerance=None, eps=1e-10, stop_updating_after=1e-10, max_iter=None,
              max_tridiag_iter=None, initial_guess=None, preconditioner=None):
    op = _as_operator(matmul_closure)
    if initial_guess is not None and bool(initial_guess.ne(0).any()):
        raise NotImplementedError("non-zero initial_guess")
    if tolerance is None:
        tolerance = settings.eval_cg_tolerance.value() if settings._use_eval_tolerance.on() else settings.cg_tolerance.value()
    max_iter = settings.max_cg_iterations.value() if max_iter is None else max_iter
    max_tridiag_iter = settings.max_lanczos_quadrature_iterations.value() if max_tridiag_iter is None else max_tridiag_iter
    vec = rhs.dim() == 1
    r2 = rhs.unsqueeze(-1) if vec else rhs
    w = preconditioner if torch.is_tensor(preconditioner) else None
    solves, tmat, info = op._plan().mbcg(r2.float(), n_tridiag, tolerance, max_iter, max_tridiag_iter, w)
    solves = solves.squeeze(-1) if vec else solves
    return (solves, tmat) if n_tridiag else solves


def pivoted_cholesky(mat, rank, error_tol=None, return_pivots=False):
    """gpytorch.pivoted_cholesky (gpytorch/__init__.py:146-173): returns L [n, m] (and pivots)."""
    op = mat.kernel_op if isinstance(mat, AddedDiagLinearOperator) else mat
    tol = settings.preconditioner_tolerance.value() if error_tol is None else error_tol
    lt, piv, _ = op.plan().pivoted_cholesky(rank, tol)
    return (lt.t(), piv) if return_pivots else lt.t()


def inv_quad_logdet(mat, inv_quad_rhs=None, logdet=False, reduce_inv_quad=True):
    """gpytorch.inv_quad_logdet (gpytorch/__init__.py:118-145)."""
    return mat.inv_quad_logdet(inv_quad_rhs=inv_quad_rhs, logdet=logdet, reduce_inv_quad=reduce_inv_quad)


def solve(mat, rhs, lhs=None):
    """gpytorch.solve (gpytorch/__init__.py:215-249)."""
    return mat.solve(rhs, lhs)


def root_decomposition(mat, method=None):
    """gpytorch.root_decomposition (gpytorch/__init__.py:176-188): R with R R^T ~= mat ("cholesky" or "lanczos"; None picks by
    size as sampling does).  A dense tensor gets the psd-safe Cholesky factor."""
    if torch.is_tensor(mat):
        return RootLinearOperator(psd_safe_cholesky(mat))
    return mat.root_decomposition(method=method)


def lanczos_tridiag(mat, max_iter, init_vecs=None, tol=1e-5):
    op = _as_operator(mat)
    init = init_vecs if init_vecs is not None else torch.randn(op.shape[0], device=op.device)
    if init.dim() == 2:
        init = init[:, 0]
    return op._plan().lanczos(init.float(), max_iter, tol)
