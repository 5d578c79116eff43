"""gpytorch.kernels.{Kernel, RBFKernel, RBFKernelGrad, MaternKernel, Matern52KernelGrad, RQKernel, PolynomialKernel,
PiecewisePolynomialKernel, SpectralMixtureKernel,
PeriodicKernel, ScaleKernel, AdditiveKernel, ProductKernel, IndexKernel, MultitaskKernel, LCMKernel, GridInterpolationKernel} for the
accelerated path.

Same constructor kwargs and call contract as the reference (kernels/kernel.py:163-171, :454-534;
rbf_kernel.py:68-85; matern_kernel.py:79-110; scale_kernel.py:64-118), but `forward` returns an
engine-backed KernelLinearOperator (the KeOps plug-in pattern, kernels/keops/rbf_kernel.py:44-55)
instead of a dense tensor: K is never materialised.
"""
from __future__ import annotations

import logging

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

    def __mul__(self, other):
        # k1 * k2 -> ProductKernel with nested products flattened (kernels/kernel.py:547-551)
        parts = []
        for k in (self, other):
            parts.extend(k.kernels if isinstance(k, ProductKernel) else (k,))
        return ProductKernel(*parts)

    def _batch_size(self):
        return self.batch_shape[0] if len(self.batch_shape) else None

    def _batchable(self):
        """Whether batched inputs or a batch_shape can run (one independent operator per batch entry)."""
        return True

    def _unbatched_name(self):
        """The kernel named when batched inputs or a batch_shape are refused (_batchable() is False)."""
        return "RBFKernelGrad"

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
        if (x1.dim() == 3 or nb is not None) and not self._batchable():
            raise NotImplementedError(f"a batched {self._unbatched_name()} (batched inputs or a batch_shape) is not available "
                                      "on the accelerated path")
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


class RBFKernelGrad(RBFKernel):
    """Covariance of values and partial derivatives of an RBF GP (kernels/rbf_kernel_grad.py): an n x m input pair gives an
    n (d+1) x m (d+1) operator over interleaved rows i (d+1) + a (a = 0: f(x_i), a = 1..d: df/dx_a at x_i), as the reference returns
    after its perfect shuffle.  forward returns one engine DerivKernelLinearOperator (gp_plan_set_deriv); d <= 16, unbatched.
    diag=True gives 1 at value rows and 1 / l_a^2 at derivative rows (times the outputscale inside a ScaleKernel)."""

    def _batchable(self):
        return False

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, **params):
        if _batch_index is not None or len(self.batch_shape) or x1.dim() != 2:
            raise NotImplementedError("a batched RBFKernelGrad is not available on the accelerated path")
        from .operators import DerivKernelLinearOperator
        if diag and not (_same or (x1.shape == x2.shape and torch.equal(x1, x2))):
            raise RuntimeError("diag=True only works when x1 == x2")
        ls = self.lengthscale.reshape(-1)
        ls = ls[0] if ls.numel() == 1 else ls
        op = DerivKernelLinearOperator(x1, None if _same else x2, ls)
        return op.diagonal() if diag else op

    def num_outputs_per_input(self, x1, x2):
        return x1.size(-1) + 1


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


class RQKernel(_StationaryKernel):
    """k = (1 + |x1 - x2|^2 / (2 alpha l^2))^-alpha (kernels/rq_kernel.py).  Parameters as in the reference: raw_lengthscale
    [*B, 1, ard_num_dims or 1] and raw_alpha [*B, 1], each with a Positive() constraint unless one is given.  forward returns one
    engine RQKernelLinearOperator (gp_plan_set_hypers_rq) on the tensor-core or CUDA-core K.V; inside a ScaleKernel the outputscale
    multiplies it, and scaled or not it may be a term of an AdditiveKernel.  One batch dimension at most, no priors.  Products, SKI,
    multitask, additive-component and derivative kernels do not take it."""
    kind = "rq"

    def __init__(self, alpha_constraint=None, lengthscale_prior=None, **kwargs):
        if lengthscale_prior is not None or kwargs.pop("alpha_prior", None) is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        super().__init__(**kwargs)
        self.register_parameter("raw_alpha", torch.nn.Parameter(torch.zeros(*self.batch_shape, 1)))
        self.register_constraint("raw_alpha", alpha_constraint or Positive())

    @property
    def alpha(self):
        return self.raw_alpha_constraint.transform(self.raw_alpha)

    @alpha.setter
    def alpha(self, value):
        self._set_alpha(value)

    def _set_alpha(self, value):
        self._set_constrained("raw_alpha", value)

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, outputscale=None, last_dim_is_batch=False, **params):
        from .operators import RQKernelLinearOperator
        if last_dim_is_batch:
            raise NotImplementedError("last_dim_is_batch is not available for an RQKernel on the accelerated path")
        if diag and not (_same or x1.size(0) == x2.size(0)):
            raise RuntimeError("diag=True needs x1 and x2 of equal sizes")
        ls, al = self.lengthscale, self.alpha
        if _batch_index is not None:
            ls, al = ls[_batch_index], al[_batch_index]
        ls = ls.reshape(-1)
        op = RQKernelLinearOperator(x1, None if _same else x2, ls[0] if ls.numel() == 1 else ls, al.reshape(-1)[0], outputscale)
        return op.diagonal() if diag else op


def _is_rq(k):
    """k is an RQKernel, or a ScaleKernel around one."""
    return isinstance(k, RQKernel) or isinstance(getattr(k, "base_kernel", None), RQKernel)


class PolynomialKernel(Kernel):
    """k = (x1 . x2 + c)^p over the raw inputs (kernels/polynomial_kernel.py).  Parameters as in the reference: the integer power
    (an int, an integral float or a one-element tensor, 1..8 on the accelerated path) and raw_offset [*B, 1] with a Positive()
    constraint unless one is given.  forward returns one engine PolynomialKernelLinearOperator (gp_plan_set_hypers_poly) on the
    tensor-core or CUDA-core K.V; inside a ScaleKernel the outputscale multiplies it, and scaled or not it may be a term of an
    AdditiveKernel.  One batch dimension at most, no priors.  The kernel is not stationary (no lengthscale, no centring), so it is
    not a _StationaryKernel: products, SKI, multitask, additive-component and derivative kernels do not take it."""
    kind = "poly"

    def __init__(self, power, offset_prior=None, offset_constraint=None, **kwargs):
        if offset_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        super().__init__(**kwargs)
        if torch.is_tensor(power):
            if power.numel() != 1:
                raise NotImplementedError("PolynomialKernel: power must be one integer")
            power = power.item()
        if isinstance(power, bool) or not isinstance(power, (int, float)) or float(power) != int(power):
            raise NotImplementedError(f"PolynomialKernel: power must be an integer (got {power!r})")
        power = int(power)
        if not 1 <= power <= 8:
            raise NotImplementedError(f"PolynomialKernel: power {power} is not available on the accelerated path (1 to 8)")
        self.power = power
        self.register_parameter("raw_offset", torch.nn.Parameter(torch.zeros(*self.batch_shape, 1)))
        self.register_constraint("raw_offset", offset_constraint or Positive())

    @property
    def offset(self):
        return self.raw_offset_constraint.transform(self.raw_offset)

    @offset.setter
    def offset(self, value):
        self._set_offset(value)

    def _set_offset(self, value):
        self._set_constrained("raw_offset", value)

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, outputscale=None, last_dim_is_batch=False, **params):
        from .operators import PolynomialKernelLinearOperator
        if last_dim_is_batch:
            raise NotImplementedError("last_dim_is_batch is not available for a PolynomialKernel on the accelerated path")
        if diag and not (_same or x1.size(0) == x2.size(0)):
            raise RuntimeError("diag=True needs x1 and x2 of equal sizes")
        off = self.offset if _batch_index is None else self.offset[_batch_index]
        op = PolynomialKernelLinearOperator(x1, None if _same else x2, self.power, off.reshape(-1)[0], outputscale)
        return op.diagonal() if diag else op


class PiecewisePolynomialKernel(Kernel):
    """k = (1 - r)_+^(j+q) poly_q(r), r = |x1 - x2| / l, j = floor(D / 2) + q + 1 with D the input columns after active_dims
    (kernels/piecewise_polynomial_kernel.py, with the module's own q = 2 coefficient (5 j + 3) / 3, DESIGN 4.24).  Parameters as in
    the reference: q in {0, 1, 2, 3} and raw_lengthscale [*B, 1, ard_num_dims or 1] with a Positive() constraint unless one is given.
    forward returns one engine PiecewisePolynomialKernelLinearOperator (gp_plan_set_hypers_pp) on the compact-support backend, whose
    products evaluate only the point pairs within one lengthscale; inside a ScaleKernel the outputscale multiplies it.  1 <= D <= 16,
    one batch dimension at most, no priors.  Not a _StationaryKernel on this path: sums, products, SKI, multitask and derivative
    kernels do not take it, and neither do inputs that require grad."""
    has_lengthscale = True
    kind = "ppoly"

    def __init__(self, q=2, lengthscale_prior=None, **kwargs):
        if lengthscale_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        super().__init__(**kwargs)
        if q not in {0, 1, 2, 3}:
            raise ValueError("q expected to be 0, 1, 2 or 3")
        self.q = q

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, outputscale=None, last_dim_is_batch=False, **params):
        from .operators import PiecewisePolynomialKernelLinearOperator
        if last_dim_is_batch:
            raise NotImplementedError("last_dim_is_batch is not available for a PiecewisePolynomialKernel on the accelerated path")
        if diag and not (_same or x1.size(0) == x2.size(0)):
            raise RuntimeError("diag=True needs x1 and x2 of equal sizes")
        ls = self.lengthscale if _batch_index is None else self.lengthscale[_batch_index]
        ls = ls.reshape(-1)
        op = PiecewisePolynomialKernelLinearOperator(x1, None if _same else x2, self.q, ls[0] if ls.numel() == 1 else ls, outputscale)
        return op.diagonal() if diag else op


def _is_pp(k):
    """k is a PiecewisePolynomialKernel, or a ScaleKernel around one."""
    return isinstance(k, PiecewisePolynomialKernel) or isinstance(getattr(k, "base_kernel", None), PiecewisePolynomialKernel)


class Matern52KernelGrad(MaternKernel):
    """Covariance of values and partial derivatives of a Matern-5/2 GP (kernels/matern52_kernel_grad.py): an n x m input pair gives
    an n (d+1) x m (d+1) operator over interleaved rows i (d+1) + a (a = 0: f(x_i), a = 1..d: df/dx_a at x_i), as the reference
    returns after its perfect shuffle.  `nu` is dropped and fixed to 2.5, as in the reference.  forward returns one engine
    DerivKernelLinearOperator of kind "matern52" (gp_plan_set_deriv_kind); d <= 16, unbatched.  diag=True gives 1 at value rows and
    (5/3) / l_a^2 at derivative rows (times the outputscale inside a ScaleKernel).  Sums, products, multitask and SKI kernels do not
    take it."""

    def __init__(self, **kwargs):
        kwargs.pop("nu", None)
        super().__init__(nu=2.5, **kwargs)

    def _batchable(self):
        return False

    def _unbatched_name(self):
        return "Matern52KernelGrad"

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, **params):
        if _batch_index is not None or len(self.batch_shape) or x1.dim() != 2:
            raise NotImplementedError("a batched Matern52KernelGrad is not available on the accelerated path")
        from .operators import DerivKernelLinearOperator
        if diag and not (_same or (x1.shape == x2.shape and torch.equal(x1, x2))):
            raise RuntimeError("diag=True only works when x1 == x2")
        ls = self.lengthscale.reshape(-1)
        ls = ls[0] if ls.numel() == 1 else ls
        op = DerivKernelLinearOperator(x1, None if _same else x2, ls, kind="matern52")
        return op.diagonal() if diag else op

    def num_outputs_per_input(self, x1, x2):
        return x1.size(-1) + 1


class SpectralMixtureKernel(Kernel):
    """k(x, x') = prod_d sum_q w_q exp(-2 pi^2 v_qd^2 tau_d^2) cos(2 pi mu_qd tau_d), tau = x - x' (Wilson & Adams 2013;
    kernels/spectral_mixture_kernel.py, whose forward sums the components of each dimension and multiplies over the dimensions).
    Parameters as in the reference: raw_mixture_weights [*B, Q], raw_mixture_means / raw_mixture_scales [*B, Q, 1, d], each with a
    Positive() constraint unless one is given.  forward returns one engine SpectralMixtureKernelLinearOperator (gp_plan_set_spectral);
    inside a ScaleKernel the outputscale S multiplies it.  1 <= num_mixtures <= 16, 1 <= d <= 8, num_mixtures * d <= 32, one batch
    dimension at most.  Sums, products, SKI, multitask and derivative kernels do not take it, and the inputs get no gradient."""

    is_stationary = True

    def __init__(self, num_mixtures=None, ard_num_dims=1, batch_shape=None, mixture_scales_prior=None, mixture_scales_constraint=None,
                 mixture_means_prior=None, mixture_means_constraint=None, mixture_weights_prior=None, mixture_weights_constraint=None,
                 **kwargs):
        if num_mixtures is None:
            raise RuntimeError("num_mixtures is a required argument")
        if mixture_means_prior is not None or mixture_scales_prior is not None or mixture_weights_prior is not None:
            logging.getLogger().warning("Priors not implemented for SpectralMixtureKernel")
        super().__init__(ard_num_dims=ard_num_dims, batch_shape=batch_shape, **kwargs)
        self.num_mixtures = int(num_mixtures)
        shape = torch.Size([*self.batch_shape, self.num_mixtures, 1, self.ard_num_dims])
        self.register_parameter("raw_mixture_weights", torch.nn.Parameter(torch.zeros(*self.batch_shape, self.num_mixtures)))
        self.register_parameter("raw_mixture_means", torch.nn.Parameter(torch.zeros(shape)))
        self.register_parameter("raw_mixture_scales", torch.nn.Parameter(torch.zeros(shape)))
        self.register_constraint("raw_mixture_scales", mixture_scales_constraint or Positive())
        self.register_constraint("raw_mixture_means", mixture_means_constraint or Positive())
        self.register_constraint("raw_mixture_weights", mixture_weights_constraint or Positive())

    @property
    def mixture_scales(self):
        return self.raw_mixture_scales_constraint.transform(self.raw_mixture_scales)

    @mixture_scales.setter
    def mixture_scales(self, value):
        self._set_mixture_scales(value)

    def _set_mixture_scales(self, value):
        self._set_constrained("raw_mixture_scales", value)

    @property
    def mixture_means(self):
        return self.raw_mixture_means_constraint.transform(self.raw_mixture_means)

    @mixture_means.setter
    def mixture_means(self, value):
        self._set_mixture_means(value)

    def _set_mixture_means(self, value):
        self._set_constrained("raw_mixture_means", value)

    @property
    def mixture_weights(self):
        return self.raw_mixture_weights_constraint.transform(self.raw_mixture_weights)

    @mixture_weights.setter
    def mixture_weights(self, value):
        self._set_mixture_weights(value)

    def _set_mixture_weights(self, value):
        self._set_constrained("raw_mixture_weights", value)

    def _training_inputs(self, train_x, train_y):
        if not torch.is_tensor(train_x) or not torch.is_tensor(train_y):
            raise RuntimeError("train_x and train_y should be tensors")
        if train_x.dim() == 1:
            train_x = train_x.unsqueeze(-1)
        if self.active_dims is not None:
            train_x = train_x[..., self.active_dims.to(train_x.device)]
        return train_x

    def initialize_from_data(self, train_x, train_y, **kwargs):
        """Scales from the data's extent, means from its finest spacing and weights from std(y) (the reference's statistics, with
        the same torch random draws: one randn_like of the scales, then one rand_like of the means).  For irregular samples."""
        with torch.no_grad():
            x = self._training_inputs(train_x, train_y)
            xs = x.sort(dim=-2)[0]
            span = xs[..., -1, :] - xs[..., 0, :]                                  # [*, d]
            gaps = xs[..., 1:, :] - xs[..., :-1, :]
            gaps = torch.where(gaps == 0, torch.full_like(gaps, 1.0e10), gaps)    # repeated points do not set the finest spacing
            finest = gaps.min(dim=-2)[0]                                           # [*, d]
            # one value per parameter slot: reduce the leading data dimensions the parameters do not carry
            extra = finest.dim() - 1 - len(self.batch_shape)
            for _ in range(max(extra, 0)):
                finest, span = finest.min(dim=0)[0], span.max(dim=0)[0]
            finest = finest.unsqueeze(-2).unsqueeze(-3)                            # [*B, 1, 1, d]
            span = span.unsqueeze(-2).unsqueeze(-3)
            # 1 / scale ~ |N(0, span^2)|;  mean ~ U(0, 0.5 / finest spacing);  weights std(y) / Q
            self.mixture_scales = torch.randn_like(self.raw_mixture_scales).mul_(span).abs_().reciprocal_()
            self.mixture_means = torch.rand_like(self.raw_mixture_means).mul_(0.5).div(finest)
            self.mixture_weights = train_y.std().div(self.num_mixtures)

    def initialize_from_data_empspect(self, train_x, train_y):
        """Means, scales and weights from a diagonal Gaussian mixture (scikit-learn, imported here) fitted to 1000 frequencies drawn
        from the empirical spectrum |FFT(y)|^2 / N of the outputs (numpy's global generator draws the uniforms).  Assumes evenly
        spaced inputs, as the reference does."""
        import numpy as np

        with torch.no_grad():
            self._training_inputs(train_x, train_y)
            y = train_y.detach().reshape(-1).cpu()
            N = y.numel()
            M = N // 2
            spect = (torch.fft.fft(y).abs() ** 2 / N)[: M + 1].double().numpy()
            freq = np.arange(M + 1, dtype=np.float64) / N
            # inverse-CDF sampling of the frequencies: the spectrum's trapezoidal CDF, linear between the grid frequencies
            cdf = np.concatenate([[0.0], np.cumsum(0.5 * (spect[1:] + spect[:-1]) * np.diff(freq))])
            cdf = cdf / cdf[-1]
            u = np.random.rand(1000, self.ard_num_dims)
            samples = np.interp(u, cdf, freq)
            from sklearn.mixture import GaussianMixture

            gmm = GaussianMixture(n_components=self.num_mixtures, covariance_type="diag").fit(samples)
            like = dict(dtype=self.raw_mixture_means.dtype, device=self.raw_mixture_means.device)
            self.mixture_means = torch.tensor(gmm.means_, **like).unsqueeze(-2)
            self.mixture_scales = torch.tensor(gmm.covariances_, **like).unsqueeze(-2)
            self.mixture_weights = torch.tensor(gmm.weights_, **like)

    def _check_dims(self, x1):
        d = len(self.active_dims) if self.active_dims is not None else (1 if x1.dim() == 1 else x1.size(-1))
        if d != self.ard_num_dims:
            raise RuntimeError(f"The SpectralMixtureKernel expected the input to have {self.ard_num_dims} dimensionality "
                               f"(based on the ard_num_dims argument). Got {d}.")

    def __call__(self, x1, x2=None, diag=False, **params):
        self._check_dims(x1)
        return Kernel.__call__(self, x1, x2, diag=diag, **params)

    def _parameters_of(self, batch_index):
        w, mu, v = self.mixture_weights, self.mixture_means, self.mixture_scales
        if batch_index is not None:
            w, mu, v = w[batch_index], mu[batch_index], v[batch_index]
        return w, mu, v

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, outputscale=None, **params):
        from .operators import SpectralMixtureKernelLinearOperator
        self._check_dims(x1)
        if diag and not (_same or x1.size(0) == x2.size(0)):
            raise RuntimeError("diag=True needs x1 and x2 of equal sizes")
        op = SpectralMixtureKernelLinearOperator(x1, None if _same else x2, *self._parameters_of(_batch_index), outputscale)
        return op.diagonal() if diag else op


class PeriodicKernel(Kernel):
    """k(x, x') = exp(-2 sum_d sin^2(pi (x_d - x'_d) / p_d) / l_d) (kernels/periodic_kernel.py; the lengthscale is not squared).
    Parameters as in the reference: raw_lengthscale and raw_period_length [*B, 1, ard_num_dims or 1], each with a Positive()
    constraint unless one is given.  forward returns one engine PeriodicKernelLinearOperator (gp_plan_set_periodic), which runs as
    an RBF kernel over the embedding (cos, sin)(2 pi x / p) on tensor cores; inside a ScaleKernel the outputscale multiplies it,
    and scaled or not it may be a term of an AdditiveKernel.  1 <= d <= 16, one batch dimension at most, no priors.  Products,
    SKI, multitask and derivative kernels do not take it, and the inputs get no gradient."""

    has_lengthscale = True

    def __init__(self, period_length_prior=None, period_length_constraint=None, lengthscale_prior=None, **kwargs):
        if period_length_prior is not None or lengthscale_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        super().__init__(**kwargs)
        n = self.ard_num_dims or 1
        self.register_parameter("raw_period_length", torch.nn.Parameter(torch.zeros(*self.batch_shape, 1, n)))
        self.register_constraint("raw_period_length", period_length_constraint or Positive())

    @property
    def period_length(self):
        return self.raw_period_length_constraint.transform(self.raw_period_length)

    @period_length.setter
    def period_length(self, value):
        self._set_period_length(value)

    def _set_period_length(self, value):
        self._set_constrained("raw_period_length", value)

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, outputscale=None, last_dim_is_batch=False, **params):
        from .operators import PeriodicKernelLinearOperator
        if last_dim_is_batch:
            raise NotImplementedError("last_dim_is_batch is not available for a PeriodicKernel on the accelerated path")
        if diag and not (_same or x1.size(0) == x2.size(0)):
            raise RuntimeError("diag=True needs x1 and x2 of equal sizes")
        ls, per = self.lengthscale, self.period_length
        if _batch_index is not None:
            ls, per = ls[_batch_index], per[_batch_index]
        ls, per = ls.reshape(-1), per.reshape(-1)
        op = PeriodicKernelLinearOperator(x1, None if _same else x2, ls[0] if ls.numel() == 1 else ls,
                                          per[0] if per.numel() == 1 else per, outputscale)
        return op.diagonal() if diag else op


def _is_periodic(k):
    """k is a PeriodicKernel, or a ScaleKernel around one."""
    return isinstance(k, PeriodicKernel) or isinstance(getattr(k, "base_kernel", None), PeriodicKernel)


def _is_m52_grad(k):
    """k is a Matern52KernelGrad, or a ScaleKernel around one."""
    return isinstance(k, Matern52KernelGrad) or isinstance(getattr(k, "base_kernel", None), Matern52KernelGrad)


class ScaleKernel(Kernel):
    """K <- outputscale * base(K)  (kernels/scale_kernel.py:64-118); the scale is folded into the fused kernel."""

    def __init__(self, base_kernel, outputscale_prior=None, outputscale_constraint=None, **kwargs):
        if isinstance(base_kernel, LCMKernel):
            raise NotImplementedError("ScaleKernel(LCMKernel(...)) is not available on the accelerated path: scale the base kernels")
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
            from .operators import with_outputscale
            inner = self.base_kernel(x1, None if _same else x2)
            terms = inner.ops if isinstance(inner, SumKernelLinearOperator) else [inner]
            scaled = [with_outputscale(t, self.outputscale * t.outputscale) for t in terms]   # periodic terms keep their period
            op = scaled[0] if len(scaled) == 1 else SumKernelLinearOperator(scaled)
            return op.diagonal() if diag else op
        if isinstance(self.base_kernel, ProductKernel):
            # s (k_1 ... k_m): the scale is folded into the first factor's outputscale (autograd sees the product)
            from .operators import ProductKernelLinearOperator
            if _batch_index is not None:
                raise NotImplementedError("batched ScaleKernel over a ProductKernel")
            f = self.base_kernel(x1, None if _same else x2).ops
            first = KernelLinearOperator(f[0].x1, f[0].x2, f[0].kind, f[0].lengthscale, self.outputscale * f[0].outputscale)
            op = ProductKernelLinearOperator([first, *f[1:]])
            return op.diagonal() if diag else op
        if isinstance(self.base_kernel, (SpectralMixtureKernel, PeriodicKernel, RQKernel, PolynomialKernel, PiecewisePolynomialKernel)):
            os_ = self.outputscale if (_batch_index is None or self.outputscale.dim() == 0) else self.outputscale[_batch_index]
            return self.base_kernel.forward(x1, x2, diag=diag, _same=_same, _batch_index=bi, outputscale=os_, **params)
        if isinstance(self.base_kernel, GridInterpolationKernel):
            base = self.base_kernel.forward(x1, x2, diag=False, _same=_same, **params)
        else:
            base = self.base_kernel.forward(x1, x2, diag=False, _same=_same, _batch_index=bi, **params)
        os_ = self.outputscale if (_batch_index is None or self.outputscale.dim() == 0) else self.outputscale[_batch_index]
        from .operators import DerivKernelLinearOperator, SKIKernelLinearOperator
        if isinstance(base, DerivKernelLinearOperator):   # s folded into the same value / gradient operator
            op = DerivKernelLinearOperator(base.x1, None if base.same else base.x2, base.lengthscale, os_, base.kind)
            return op.diagonal() if diag else op
        if isinstance(base, SKIKernelLinearOperator):
            op = SKIKernelLinearOperator(base.x1, base.kind, base.lengthscale, os_, base.grid_sizes, base.grid_lo, base.grid_step)
            return op.diagonal() if diag else op
        from .operators import (PeriodicKernelLinearOperator, PiecewisePolynomialKernelLinearOperator, PolynomialKernelLinearOperator,
                                RQKernelLinearOperator, SumKernelLinearOperator, with_outputscale)
        # operators with parameters beyond lengthscale and scale
        keep = (PeriodicKernelLinearOperator, RQKernelLinearOperator, PolynomialKernelLinearOperator, PiecewisePolynomialKernelLinearOperator)
        if isinstance(base, keep):   # a nested ScaleKernel: both scales folded in, the period / alpha kept
            op = with_outputscale(base, os_ * base.outputscale)
            return op.diagonal() if diag else op
        if isinstance(base, SumKernelLinearOperator) and any(isinstance(t, keep) for t in base.ops):
            # a ScaleKernel around a scaled sum with periodic or RQ terms: the scale folded into every term, periods and alphas kept
            op = SumKernelLinearOperator([with_outputscale(t, os_ * t.outputscale) for t in base.ops])
            return op.diagonal() if diag else op
        op = KernelLinearOperator(base.x1, base.x2, base.kind, base.lengthscale, os_)
        return op.diagonal() if diag else op

    def _batchable(self):
        return self.base_kernel._batchable()

    def _unbatched_name(self):
        return self.base_kernel._unbatched_name()

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
            if isinstance(k, ProductKernel) or isinstance(getattr(k, "base_kernel", None), ProductKernel):
                raise NotImplementedError("sums that contain a ProductKernel are not available on the accelerated path")
            if _is_m52_grad(k):
                raise NotImplementedError("sums that contain a Matern52KernelGrad are not available on the accelerated path")
            if _is_pp(k):
                raise NotImplementedError("sums that contain a PiecewisePolynomialKernel are not available on the accelerated path")
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


class ProductKernel(Kernel):
    """k = k_1 * ... * k_m (kernels/kernel.py:634-690).  Every factor is called on the full inputs (so its own active_dims apply, as
    in the reference) and must be an RBFKernel / MaternKernel, optionally inside a ScaleKernel; the product is ONE
    ProductKernelLinearOperator whose products / solves run natively (gp_plan_set_product), not a dense multiplication.  2 to 4
    unbatched factors."""

    def __init__(self, *kernels):
        super().__init__()
        if len(kernels) > 4:
            raise NotImplementedError(f"a ProductKernel takes up to 4 factors on the accelerated path (got {len(kernels)})")
        for k in kernels:
            if not isinstance(k, Kernel):
                raise RuntimeError("ProductKernel factors must be kernels")
            if _is_periodic(k):
                raise NotImplementedError("products with a PeriodicKernel factor are not available on the accelerated path")
            if _is_rq(k):
                raise NotImplementedError("products with an RQKernel factor are not available on the accelerated path")
            if _is_pp(k):
                raise NotImplementedError("products with a PiecewisePolynomialKernel factor are not available on the accelerated path")
            base = k.base_kernel if isinstance(k, ScaleKernel) else k
            if not isinstance(base, _StationaryKernel) or isinstance(base, (RBFKernelGrad, Matern52KernelGrad)):
                raise NotImplementedError("ProductKernel factors must be RBF / Matern kernels (optionally scaled) on the accelerated "
                                          "path: sums, SKI, multitask and derivative kernels inside a product are not available")
            if len(k.batch_shape):
                raise NotImplementedError("batched factors of a ProductKernel")
        self.kernels = torch.nn.ModuleList(kernels)

    def forward(self, x1, x2, diag=False, **params):
        raise NotImplementedError("ProductKernel dispatches to its factors in __call__")

    def __call__(self, x1, x2=None, diag=False, **params):
        from .operators import ProductKernelLinearOperator
        if x1.dim() == 3 or (x2 is not None and x2.dim() == 3):
            raise NotImplementedError("batched inputs of a ProductKernel")
        factors = [k(x1, x2, diag=diag, **params) for k in self.kernels]
        if diag:
            out = factors[0]
            for t in factors[1:]:
                out = out * t
            return out
        return factors[0] if len(factors) == 1 else ProductKernelLinearOperator(factors)


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
        if isinstance(base, PeriodicKernel):
            raise NotImplementedError("a PeriodicKernel data kernel of a MultitaskKernel is not available on the accelerated path")
        if isinstance(base, RQKernel):
            raise NotImplementedError("an RQKernel data kernel of a MultitaskKernel is not available on the accelerated path")
        if not isinstance(base, _StationaryKernel) or len(dm.batch_shape):
            raise NotImplementedError("the accelerated MultitaskKernel takes an RBFKernel / MaternKernel data kernel, optionally "
                                      "inside a ScaleKernel")
        if isinstance(base, Matern52KernelGrad):
            raise NotImplementedError("a Matern52KernelGrad data kernel of a MultitaskKernel is not available on the accelerated path")
        covar_x = dm(x1, None if _same else x2)
        from .operators import KroneckerKernelLinearOperator
        op = KroneckerKernelLinearOperator(covar_x.x1, None if covar_x.same else covar_x.x2, covar_x.kind, covar_x.lengthscale,
                                           covar_x.outputscale, self.task_covar_module.covar_matrix)
        return op.diagonal() if diag else op

    def num_outputs_per_input(self, x1, x2):
        """An n x m data covariance becomes an (n T) x (m T) multitask covariance."""
        return self.num_tasks


class LCMKernel(Kernel):
    """Linear model of coregionalisation (kernels/lcm_kernel.py): K = sum_q K_q(x1, x2) (x) B_q over interleaved rows i T + a, one
    MultitaskKernel per base kernel in `covar_module_list` (the reference's names, so state-dict keys match), each with its own
    IndexKernel B_q = F_q F_q^T + diag(v_q) of rank `rank` (an int, or one per base kernel).  Base kernels are what MultitaskKernel
    takes (RBFKernel / MaternKernel, optionally inside a ScaleKernel).  forward returns one engine operator: the term's
    KroneckerKernelLinearOperator for one base kernel, an LCMKernelLinearOperator (gp_plan_set_kron_terms) for 2 to 4.  Unbatched, no
    prior."""

    def __init__(self, base_kernels, num_tasks, rank=1, task_covar_prior=None):
        if len(base_kernels) < 1:
            raise ValueError("At least one base kernel must be provided.")
        for k in base_kernels:
            if not isinstance(k, Kernel):
                raise ValueError("base_kernels must only contain Kernel objects")
        if len(base_kernels) > 4:
            raise NotImplementedError(f"an LCMKernel takes up to 4 base kernels on the accelerated path (got {len(base_kernels)})")
        if task_covar_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        if not isinstance(rank, list):
            rank = [rank] * len(base_kernels)
        if len(rank) != len(base_kernels):
            raise ValueError(f"rank has {len(rank)} entries for {len(base_kernels)} base kernels")
        super().__init__()
        self.covar_module_list = torch.nn.ModuleList(
            [MultitaskKernel(k, num_tasks=num_tasks, rank=r, task_covar_prior=task_covar_prior) for k, r in zip(base_kernels, rank)])

    def forward(self, x1, x2, diag=False, _same=False, _batch_index=None, last_dim_is_batch=False, **params):
        if _batch_index is not None:
            raise NotImplementedError("a batched LCMKernel is not available on the accelerated path")
        terms = [m.forward(x1, x2, diag=diag, _same=_same, last_dim_is_batch=last_dim_is_batch, **params) for m in self.covar_module_list]
        if diag:
            out = terms[0]
            for t in terms[1:]:
                out = out + t
            return out
        if len(terms) == 1:
            return terms[0]
        from .operators import LCMKernelLinearOperator
        return LCMKernelLinearOperator(terms)

    def _batchable(self):
        return False

    def _unbatched_name(self):
        return "LCMKernel"

    def num_outputs_per_input(self, x1, x2):
        """An n x m data covariance becomes an (n T) x (m T) multitask covariance."""
        return self.covar_module_list[0].num_outputs_per_input(x1, x2)


class GridInterpolationKernel(Kernel):
    """SKI / KISS-GP (kernels/grid_interpolation_kernel.py:14-213): base_kernel(x, x') ~= w_x^T K_grid w_x' with cubic interpolation
    onto a regular grid; K_grid is a Kronecker product of per-dimension Toeplitz matrices (kernels/grid_kernel.py:107-177).
    `base_kernel` must be an RBFKernel / MaternKernel (optionally inside a ScaleKernel OUTSIDE this kernel, as in the reference's
    examples: ScaleKernel(GridInterpolationKernel(RBFKernel(), grid_size, num_dims))).  grid_bounds=None sizes the grid from the
    first inputs it sees (:154-190)."""

    def __init__(self, base_kernel, grid_size, num_dims=None, grid_bounds=None, active_dims=None):
        super().__init__(active_dims=active_dims)
        if isinstance(base_kernel, SpectralMixtureKernel):
            raise NotImplementedError("a SpectralMixtureKernel base kernel of a GridInterpolationKernel is not available on the "
                                      "accelerated path")
        if isinstance(base_kernel, PeriodicKernel):
            raise NotImplementedError("a PeriodicKernel base kernel of a GridInterpolationKernel is not available on the accelerated "
                                      "path")
        if isinstance(base_kernel, PiecewisePolynomialKernel):
            raise NotImplementedError("a PiecewisePolynomialKernel base kernel of a GridInterpolationKernel is not available on the "
                                      "accelerated path: it runs its own compact-support backend")
        if isinstance(base_kernel, RQKernel):
            raise NotImplementedError("an RQKernel base kernel of a GridInterpolationKernel is not available on the accelerated path: "
                                      "its heavy tails leave nothing for the band-limited grid products to skip")
        if not isinstance(base_kernel, _StationaryKernel):
            raise RuntimeError("GridInterpolationKernel needs an RBFKernel or MaternKernel base kernel on the accelerated path")
        if isinstance(base_kernel, Matern52KernelGrad):
            raise NotImplementedError("a Matern52KernelGrad base kernel of a GridInterpolationKernel is not available on the "
                                      "accelerated path")
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
