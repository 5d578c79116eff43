"""gpytorch.kernels.{Kernel, RBFKernel, MaternKernel, ScaleKernel, AdditiveKernel, GridInterpolationKernel} for the accelerated path.

Same constructor kwargs and call contract as the reference (kernels/kernel.py:163-171, :454-534;
rbf_kernel.py:68-85; matern_kernel.py:79-110; scale_kernel.py:64-118), but `forward` returns an
engine-backed KernelLinearOperator (the KeOps plug-in pattern, kernels/keops/rbf_kernel.py:44-55)
instead of a dense tensor: K is never materialised.
"""
from __future__ import annotations

import torch

from .constraints import Positive
from .module import Module
from .operators import KernelLinearOperator


class Kernel(Module):
    has_lengthscale = False
    kind = None

    def __init__(self, ard_num_dims=None, batch_shape=None, active_dims=None, lengthscale_prior=None,
                 lengthscale_constraint=None, eps=1e-6, **kwargs):
        super().__init__()
        self.batch_shape = torch.Size(batch_shape) if batch_shape is not None else torch.Size()
        if len(self.batch_shape) > 1:
            raise NotImplementedError("one leading batch dimension is supported (BASELINE config 4: batch = 16)")
        self.ard_num_dims = ard_num_dims
        self.active_dims = None if active_dims is None else torch.as_tensor(active_dims, dtype=torch.long)
        self.eps = eps
        if self.has_lengthscale:
            n = 1 if ard_num_dims is None else ard_num_dims
            # kernels/kernel.py:213-219: lengthscale has shape batch_shape x 1 x (ard_num_dims or 1)
            self.register_parameter("raw_lengthscale", torch.nn.Parameter(torch.zeros(*self.batch_shape, 1, n)))
            self.register_constraint("raw_lengthscale", lengthscale_constraint or Positive())

    @property
    def lengthscale(self):
        return self.raw_lengthscale_constraint.transform(self.raw_lengthscale) if self.has_lengthscale else None

    @lengthscale.setter
    def lengthscale(self, value):
        self._set_lengthscale(value)

    def _set_lengthscale(self, value):
        if not self.has_lengthscale:
            raise RuntimeError("Kernel has no lengthscale.")
        self._set_constrained("raw_lengthscale", value)

    def forward(self, x1, x2, diag=False, **params):
        raise NotImplementedError

    def __add__(self, other):
        # k1 + k2 -> AdditiveKernel with nested sums flattened (kernels/kernel.py:541-545)
        parts = []
        for k in (self, other):
            parts.extend(k.kernels if isinstance(k, AdditiveKernel) else (k,))
        return AdditiveKernel(*parts)

    def _batch_size(self):
        return self.batch_shape[0] if len(self.batch_shape) else None

    def __call__(self, x1, x2=None, diag=False, **params):
        # kernels/kernel.py:454-534: active dims, 1-D -> 2-D, x2=None -> x1, size check
        if self.active_dims is not None:
            idx = self.active_dims.to(x1.device)
            x1 = x1.index_select(-1, idx)
            if x2 is not None:
                x2 = x2.index_select(-1, idx)
        if x1.dim() == 1:
            x1 = x1.unsqueeze(1)
        if x2 is not None:
            if x2.dim() == 1:
                x2 = x2.unsqueeze(1)
            if x1.size(-1) != x2.size(-1):
                raise RuntimeError("x1_ and x2_ must have the same number of dimensions!")
        if self.ard_num_dims is not None and self.ard_num_dims != x1.size(-1):
            raise RuntimeError(f"Expected the input to have {self.ard_num_dims} dimensionality "
                               f"(based on the ard_num_dims argument). Got {x1.size(-1)}.")
        same = x2 is None
        nb = self._batch_size()
        if x1.dim() == 3 or nb is not None:
            # one leading batch dimension (kernels/kernel.py:119-121 broadcasts every op over it): B independent operators, each
            # with its own inputs and hyper-parameters; the solver runs them concurrently (operators.BatchLinearOperator)
            from .operators import BatchLinearOperator
            B = x1.size(0) if x1.dim() == 3 else nb
            if nb is not None and nb != B:
                raise RuntimeError(f"inputs have batch size {B} but the kernel has batch_shape {tuple(self.batch_shape)}")
            ops = []
            for b in range(B):
                xb1 = (x1[b] if x1.dim() == 3 else x1).contiguous()
                xb2 = xb1 if same else (x2[b] if x2.dim() == 3 else x2).contiguous()
                ops.append(self.forward(xb1, xb2, diag=diag, _same=same, _batch_index=(b if nb is not None else None), **params))
            return torch.stack(ops) if diag else BatchLinearOperator(ops)
        if x1.dim() != 2:
            raise NotImplementedError("inputs must be [n, d] or [batch, n, d]")
        res = self.forward(x1.contiguous(), x1.contiguous() if same else x2.contiguous(), diag=diag, _same=same, **params)
        return res


class _StationaryKernel(Kernel):
    has_lengthscale = True

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, **params):
        ls = self.lengthscale if _batch_index is None else self.lengthscale[_batch_index]
        ls = ls.reshape(-1)
        ls = ls[0] if ls.numel() == 1 else ls
        op = KernelLinearOperator(x1, None if _same else x2, self.kind, ls)
        if diag:
            return op.diagonal()
        return op


class RBFKernel(_StationaryKernel):
    """k = exp(-0.5 |x1 - x2|^2 / l^2)  (kernels/rbf_kernel.py)."""
    kind = "rbf"


class MaternKernel(_StationaryKernel):
    """Matern nu in {0.5, 1.5, 2.5}  (kernels/matern_kernel.py:79-110)."""

    def __init__(self, nu=2.5, **kwargs):
        if nu not in {0.5, 1.5, 2.5}:
            raise RuntimeError("nu expected to be 0.5, 1.5, or 2.5")
        super().__init__(**kwargs)
        self.nu = nu

    @property
    def kind(self):
        return {0.5: "matern12", 1.5: "matern32", 2.5: "matern52"}[self.nu]


class ScaleKernel(Kernel):
    """K <- outputscale * base(K)  (kernels/scale_kernel.py:64-118); the scale is folded into the fused kernel."""

    def __init__(self, base_kernel, outputscale_prior=None, outputscale_constraint=None, **kwargs):
        if base_kernel.active_dims is not None:
            kwargs["active_dims"] = base_kernel.active_dims
        super().__init__(**kwargs)
        self.base_kernel = base_kernel
        if len(self.batch_shape) == 0 and len(base_kernel.batch_shape):
            self.batch_shape = base_kernel.batch_shape
        self.register_parameter("raw_outputscale", torch.nn.Parameter(torch.zeros(self.batch_shape)))
        self.register_constraint("raw_outputscale", outputscale_constraint or Positive())

    @property
    def outputscale(self):
        return self.raw_outputscale_constraint.transform(self.raw_outputscale)

    @outputscale.setter
    def outputscale(self, value):
        self._set_outputscale(value)

    def _set_outputscale(self, value):
        self._set_constrained("raw_outputscale", value)

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, **params):
        bi = _batch_index if len(self.base_kernel.batch_shape) else None
        if isinstance(self.base_kernel, AdditiveKernel):
            # s (k_1 + ... + k_m): the scale is distributed over the terms' folded outputscales (autograd sees the products)
            from .operators import SumKernelLinearOperator
            if _batch_index is not None:
                raise NotImplementedError("batched ScaleKernel over an AdditiveKernel")
            inner = self.base_kernel(x1, None if _same else x2)
            terms = inner.ops if isinstance(inner, SumKernelLinearOperator) else [inner]
            scaled = [KernelLinearOperator(t.x1, t.x2, t.kind, t.lengthscale, self.outputscale * t.outputscale) for t in terms]
            op = scaled[0] if len(scaled) == 1 else SumKernelLinearOperator(scaled)
            return op.diagonal() if diag else op
        if isinstance(self.base_kernel, GridInterpolationKernel):
            base = self.base_kernel.forward(x1, x2, diag=False, _same=_same, **params)
        else:
            base = self.base_kernel.forward(x1, x2, diag=False, _same=_same, _batch_index=bi, **params)
        os_ = self.outputscale if (_batch_index is None or self.outputscale.dim() == 0) else self.outputscale[_batch_index]
        from .operators import SKIKernelLinearOperator
        if isinstance(base, SKIKernelLinearOperator):
            op = SKIKernelLinearOperator(base.x1, base.kind, base.lengthscale, os_, base.grid_sizes, base.grid_lo, base.grid_step)
            return op.diagonal() if diag else op
        op = KernelLinearOperator(base.x1, base.x2, base.kind, base.lengthscale, os_)
        return op.diagonal() if diag else op

    def __call__(self, x1, x2=None, diag=False, **params):
        self.active_dims = None  # selection happens once, here (base active_dims were lifted in __init__)
        if self.base_kernel.active_dims is not None:
            idx = self.base_kernel.active_dims.to(x1.device)
            x1 = x1.index_select(-1, idx)
            x2 = None if x2 is None else x2.index_select(-1, idx)
        return Kernel.__call__(self, x1, x2, diag=diag, **params)


class AdditiveKernel(Kernel):
    """k = k_1 + ... + k_m (kernels/kernel.py:592-621).  Every component is called on the full inputs (so its own active_dims
    apply, as in the reference) and must produce an engine kernel operator; the sum is ONE SumKernelLinearOperator whose
    products / solves run natively (gp_plan_set_sum), not a dense addition."""

    def __init__(self, *kernels):
        super().__init__()
        for k in kernels:
            if not isinstance(k, Kernel):
                raise RuntimeError("AdditiveKernel components must be kernels")
            if len(k.batch_shape):
                raise NotImplementedError("batched components of an AdditiveKernel")
        self.kernels = torch.nn.ModuleList(kernels)

    def forward(self, x1, x2, diag=False, **params):
        raise NotImplementedError("AdditiveKernel dispatches to its components in __call__")

    def __call__(self, x1, x2=None, diag=False, **params):
        from .operators import SKIKernelLinearOperator, SumKernelLinearOperator
        terms = [k(x1, x2, diag=diag, **params) for k in self.kernels]
        if diag:
            out = terms[0]
            for t in terms[1:]:
                out = out + t
            return out
        if any(isinstance(t, SKIKernelLinearOperator) or not isinstance(t, KernelLinearOperator) for t in terms):
            raise NotImplementedError("AdditiveKernel components must be RBF / Matern kernels (optionally scaled) on the accelerated path")
        return terms[0] if len(terms) == 1 else SumKernelLinearOperator(terms)


class IndexKernel(Module):
    """Task covariance B = F F^T + diag(v) over task indices (kernels/index_kernel.py:18-117): parameters `covar_factor` [T, rank]
    and `raw_var` [T] with the reference's names and initialisation.  Calling it on task ids returns a lazy IndexLinearOperator
    that a data kernel's operator multiplies in (`covar_x.mul(covar_i)`): the Hadamard multitask model.  Unbatched, no prior."""

    def __init__(self, num_tasks, rank=1, batch_shape=None, prior=None, var_constraint=None, **kwargs):
        if rank > num_tasks:
            raise RuntimeError("Cannot create a task covariance matrix larger than the number of tasks")
        super().__init__()
        self.batch_shape = torch.Size(batch_shape) if batch_shape is not None else torch.Size()
        if len(self.batch_shape):
            raise NotImplementedError("a batched IndexKernel is not available on the accelerated path")
        if prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        if num_tasks > 32:
            raise NotImplementedError("the accelerated path supports up to 32 tasks")
        self.num_tasks = num_tasks
        self.register_parameter("covar_factor", torch.nn.Parameter(torch.randn(*self.batch_shape, num_tasks, rank)))
        self.register_parameter("raw_var", torch.nn.Parameter(torch.randn(*self.batch_shape, num_tasks)))
        self.register_constraint("raw_var", var_constraint or Positive())

    @property
    def var(self):
        return self.raw_var_constraint.transform(self.raw_var)

    @var.setter
    def var(self, value):
        self._set_var(value)

    def _set_var(self, value):
        self._set_constrained("raw_var", value)

    def _eval_covar_matrix(self):
        cf = self.covar_factor
        return cf @ cf.transpose(-1, -2) + torch.diag_embed(self.var)

    @property
    def covar_matrix(self):
        """B as a dense [T, T] tensor (the reference returns it as PsdSumLinearOperator(RootLinearOperator(F), DiagLinearOperator(v)))."""
        return self._eval_covar_matrix()

    def __call__(self, i1, i2=None, **params):
        from .operators import IndexLinearOperator
        i1 = i1.long().reshape(-1)
        i2 = i1 if i2 is None else i2.long().reshape(-1)
        return IndexLinearOperator(i1, i2, self._eval_covar_matrix())

    forward = __call__


class MultitaskKernel(Kernel):
    """Kronecker multitask kernel (kernels/multitask_kernel.py:13-61): K = K_data(x1, x2) (x) B over interleaved rows i T + a, B from
    `task_covar_module` (an IndexKernel with the reference's covar_factor / raw_var).  `data_covar_module` is an RBFKernel /
    MaternKernel, optionally inside a ScaleKernel; forward returns one engine KroneckerKernelLinearOperator (gp_plan_set_kron).
    Unbatched, no prior."""

    def __init__(self, data_covar_module, num_tasks, rank=1, task_covar_prior=None, **kwargs):
        super().__init__(**kwargs)
        if len(self.batch_shape):
            raise NotImplementedError("a batched MultitaskKernel is not available on the accelerated path")
        if task_covar_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        self.task_covar_module = IndexKernel(num_tasks=num_tasks, batch_shape=self.batch_shape, rank=rank, prior=task_covar_prior)
        self.data_covar_module = data_covar_module
        self.num_tasks = num_tasks

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, last_dim_is_batch=False, **params):
        if last_dim_is_batch:
            raise RuntimeError("MultitaskKernel does not accept the last_dim_is_batch argument.")
        if _batch_index is not None:
            raise NotImplementedError("a batched MultitaskKernel is not available on the accelerated path")
        dm = self.data_covar_module
        base = dm.base_kernel if isinstance(dm, ScaleKernel) else dm
        if not isinstance(base, _StationaryKernel) or len(dm.batch_shape):
            raise NotImplementedError("the accelerated MultitaskKernel takes an RBFKernel / MaternKernel data kernel, optionally "
                                      "inside a ScaleKernel")
        covar_x = dm(x1, None if _same else x2)
        from .operators import KroneckerKernelLinearOperator
        op = KroneckerKernelLinearOperator(covar_x.x1, None if covar_x.same else covar_x.x2, covar_x.kind, covar_x.lengthscale,
                                           covar_x.outputscale, self.task_covar_module.covar_matrix)
        return op.diagonal() if diag else op

    def num_outputs_per_input(self, x1, x2):
        """An n x m data covariance becomes an (n T) x (m T) multitask covariance."""
        return self.num_tasks


class GridInterpolationKernel(Kernel):
    """SKI / KISS-GP (kernels/grid_interpolation_kernel.py:14-213): base_kernel(x, x') ~= w_x^T K_grid w_x' with cubic interpolation
    onto a regular grid; K_grid is a Kronecker product of per-dimension Toeplitz matrices (kernels/grid_kernel.py:107-177).
    `base_kernel` must be an RBFKernel / MaternKernel (optionally inside a ScaleKernel OUTSIDE this kernel, as in the reference's
    examples: ScaleKernel(GridInterpolationKernel(RBFKernel(), grid_size, num_dims))).  grid_bounds=None sizes the grid from the
    first inputs it sees (:154-190)."""

    def __init__(self, base_kernel, grid_size, num_dims=None, grid_bounds=None, active_dims=None):
        super().__init__(active_dims=active_dims)
        if not isinstance(base_kernel, _StationaryKernel):
            raise RuntimeError("GridInterpolationKernel needs an RBFKernel or MaternKernel base kernel on the accelerated path")
        if num_dims is None:
            raise RuntimeError("num_dims must be supplied")
        self.base_kernel = base_kernel
        self.num_dims = num_dims
        self.grid_sizes = [int(grid_size)] * num_dims if isinstance(grid_size, int) else [int(g) for g in grid_size]
        if len(self.grid_sizes) != num_dims:
            raise RuntimeError("The number of grid sizes provided through grid_size do not match num_dims.")
        self.grid_is_dynamic = grid_bounds is None
        self.grid_bounds = None if grid_bounds is None else tuple((float(a), float(b)) for a, b in grid_bounds)
        self.register_buffer("has_initialized_grid", torch.tensor(not self.grid_is_dynamic, dtype=torch.bool))

    def _grid(self):
        """(first node, spacing) per dimension: utils/grid.py:142-180 create_grid extends the bounds by one cell on both sides."""
        lo, step = [], []
        for gsz, (a, b) in zip(self.grid_sizes, self.grid_bounds):
            axis = torch.linspace(a - (b - a) / (gsz - 2), b + (b - a) / (gsz - 2), gsz)   # the reference's own float32 nodes
            lo.append(float(axis[0]))
            step.append(float(axis[1] - axis[0]))
        return lo, step

    def forward(self, x1, x2, diag=False, _same=False, **params):
        if not _same and not (x1.shape == x2.shape and torch.equal(x1, x2)):
            raise NotImplementedError("the SKI operator is built for the training covariance K(X, X)")
        if self.grid_is_dynamic and not bool(self.has_initialized_grid):
            # grid_interpolation_kernel.py:154-190: bounds from the data, 2.01 cells of slack
            mins, maxs = x1.min(0)[0].tolist(), x1.max(0)[0].tolist()
            sp = [(mx - mn) / (g - 4.02) for g, mn, mx in zip(self.grid_sizes, mins, maxs)]
            self.grid_bounds = tuple((mn - 2.01 * s_, mx + 2.01 * s_) for mn, mx, s_ in zip(mins, maxs, sp))
            self.has_initialized_grid.fill_(True)
        from .operators import SKIKernelLinearOperator
        lo, step = self._grid()
        ls = self.base_kernel.lengthscale.reshape(-1)
        ls = ls[0] if ls.numel() == 1 else ls
        op = SKIKernelLinearOperator(x1, self.base_kernel.kind, ls, None, self.grid_sizes, lo, step)
        return op.diagonal() if diag else op
