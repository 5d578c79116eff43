"""MultivariateNormal with a lazy covariance (gpytorch/distributions/multivariate_normal.py:44-64, :221-252, :254-337)."""
import math

import torch

from .sampling import psd_safe_cholesky


class MultivariateNormal:
    def __init__(self, mean, covariance_matrix):
        self.loc = mean
        self._covar = covariance_matrix
        if mean.shape[-1] != covariance_matrix.shape[-1]:
            raise RuntimeError("mean and covariance sizes do not match")

    @property
    def mean(self):
        return self.loc

    @property
    def lazy_covariance_matrix(self):
        return self._covar

    @property
    def covariance_matrix(self):
        c = self._covar
        return c if torch.is_tensor(c) else c.to_dense()

    @property
    def variance(self):
        c = self._covar
        return c.diagonal(dim1=-2, dim2=-1) if torch.is_tensor(c) else c.diagonal()

    @property
    def stddev(self):
        return self.variance.clamp_min(0).sqrt()

    def confidence_region(self):
        """(mean - 2 stddev, mean + 2 stddev) (multivariate_normal.py confidence_region)."""
        std2 = self.stddev.mul(2)
        mean = self.mean
        return mean.sub(std2), mean.add(std2)

    @property
    def event_shape(self):
        return self.loc.shape[-1:]

    def log_prob(self, value):
        """-0.5 (r^T K^-1 r + log det K + N log 2 pi), r = value - mean (multivariate_normal.py:221-252)."""
        mean, covar = self.loc, self._covar
        diff = value - mean
        if torch.is_tensor(covar):  # dense covariance: plain Cholesky
            chol = torch.linalg.cholesky(covar)
            sol = torch.cholesky_solve(diff.unsqueeze(-1), chol)
            inv_quad = (diff.unsqueeze(-1) * sol).sum((-2, -1))
            logdet = 2 * chol.diagonal(dim1=-2, dim2=-1).log().sum(-1)
        else:
            covar = covar.evaluate_kernel()
            inv_quad, logdet = covar.inv_quad_logdet(inv_quad_rhs=diff.unsqueeze(-1), logdet=True)
        return -0.5 * sum([inv_quad, logdet, diff.size(-1) * math.log(2 * math.pi)])

    def _root(self):
        """A root L with L L^T = covariance: the psd-safe Cholesky factor of a dense covariance (every posterior ExactGP returns),
        the operator's root_decomposition otherwise."""
        c = self._covar
        return psd_safe_cholesky(c) if torch.is_tensor(c) else c.root_decomposition().root

    def rsample(self, sample_shape=torch.Size(), base_samples=None):
        """sample_shape x batch_shape x N reparameterised samples mean + L eps (multivariate_normal.py:254-320).

        Gradients reach the mean always, and a dense covariance tensor through torch's Cholesky.  Samples of an engine operator
        (Cholesky / Lanczos root of the operator, or CIQ with settings.ciq_samples) are detached from its hyper-parameters."""
        sample_shape = torch.Size(sample_shape)
        covar = self._covar
        if base_samples is None:
            num_samples = sample_shape.numel() or 1
            if torch.is_tensor(covar):
                root = psd_safe_cholesky(covar)
                eps = torch.randn(*root.shape[:-1], num_samples, device=root.device, dtype=root.dtype)
                res = (root @ eps).permute(-1, *range(root.dim() - 2), root.dim() - 2)
            else:
                res = covar.zero_mean_mvn_samples(num_samples)
            res = res + self.loc.unsqueeze(0)
            return res.reshape(sample_shape + self.loc.shape)

        covar_root = self._root()
        if self.loc.shape != base_samples.shape[-self.loc.dim():] and covar_root.shape[-1] < base_samples.shape[-1]:
            raise RuntimeError(
                "The size of base_samples (minus sample shape dimensions) should agree with the size "
                "of self.loc. Expected ...{} but got {}".format(self.loc.shape, base_samples.shape))
        sample_shape = base_samples.shape[: base_samples.dim() - self.loc.dim()]
        base_samples = base_samples.reshape(-1, *self.loc.shape)
        base_samples = base_samples.permute(*range(1, self.loc.dim() + 1), 0)
        if covar_root.shape[-1] < base_samples.shape[-2]:          # a low-rank root uses the leading base samples
            base_samples = base_samples[..., : covar_root.shape[-1], :]
        res = covar_root.matmul(base_samples.to(covar_root.dtype)) + self.loc.unsqueeze(-1)
        res = res.permute(-1, *range(self.loc.dim())).contiguous()
        return res.reshape(sample_shape + self.loc.shape)

    def sample(self, sample_shape=torch.Size(), base_samples=None):
        """rsample without gradients (multivariate_normal.py:322-337)."""
        with torch.no_grad():
            return self.rsample(sample_shape=sample_shape, base_samples=base_samples)


class MultitaskMultivariateNormal(MultivariateNormal):
    """distributions/multitask_multivariate_normal.py:34-281 with interleaved=True: mean [n, T], covariance over the interleaved
    vector vec(mean) (row i T + a = point i, task a).  event_shape is (n, T), so ExactMarginalLogLikelihood divides by n T; log_prob,
    samples and the variance flatten / reshape row-major."""

    def __init__(self, mean, covariance_matrix, validate_args=False, interleaved=True):
        if not interleaved:
            raise NotImplementedError("a non-interleaved MultitaskMultivariateNormal is not available on the accelerated path")
        if not torch.is_tensor(mean) or mean.dim() != 2:
            raise RuntimeError("MultitaskMultivariateNormal takes a mean of shape [n, num_tasks] on the accelerated path")
        n, T = mean.shape
        if covariance_matrix.shape[-1] != n * T or covariance_matrix.shape[-2] != n * T:
            raise RuntimeError(f"mean shape {tuple(mean.shape)} is incompatible with covariance shape {tuple(covariance_matrix.shape)}")
        self._output_shape = mean.shape
        self._interleaved = True
        super().__init__(mean.reshape(-1), covariance_matrix)

    @property
    def num_tasks(self):
        return self._output_shape[-1]

    @property
    def mean(self):
        return self.loc.reshape(self._output_shape)

    @property
    def variance(self):
        return super().variance.reshape(self._output_shape)

    @property
    def event_shape(self):
        return self._output_shape

    def log_prob(self, value):
        return super().log_prob(value.reshape(-1))

    def rsample(self, sample_shape=torch.Size(), base_samples=None):
        if base_samples is not None:
            base_samples = base_samples.reshape(*base_samples.shape[:-2], -1)
        res = super().rsample(sample_shape=sample_shape, base_samples=base_samples)
        return res.reshape(*res.shape[:-1], *self._output_shape)
