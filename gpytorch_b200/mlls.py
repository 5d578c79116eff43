"""ExactMarginalLogLikelihood (gpytorch/mlls/exact_marginal_log_likelihood.py:54-89)."""
from . import settings
from .distributions import MultivariateNormal
from .likelihoods import _GaussianLikelihoodBase
from .module import Module
from .operators import MaskedLinearOperator


class ExactMarginalLogLikelihood(Module):
    def __init__(self, likelihood, model):
        if not isinstance(likelihood, _GaussianLikelihoodBase):
            raise RuntimeError("Likelihood must be Gaussian for exact inference")
        super().__init__()
        self.likelihood = likelihood
        self.model = model

    def forward(self, function_dist, target, *params, **kwargs):
        if not isinstance(function_dist, MultivariateNormal):
            raise RuntimeError("ExactMarginalLogLikelihood can only operate on Gaussian random variables")
        output = self.likelihood(function_dist, *params, **kwargs)
        policy = settings.observation_nan_policy.value()
        if policy == "mask":   # :70-79; a multitask target [n, T] is masked over the interleaved rows i T + a
            observed = settings.observation_nan_policy._get_observed(target, output.event_shape).reshape(-1)
            if not bool(observed.all()):
                output = MultivariateNormal(output.loc[..., observed],
                                            MaskedLinearOperator(output.lazy_covariance_matrix, observed, observed))
                target = target.reshape(*target.shape[: target.dim() - len(function_dist.event_shape)], -1)[..., observed]
        elif policy == "fill":
            raise ValueError("NaN observation policy 'fill' is not supported by ExactMarginalLogLikelihood!")
        res = output.log_prob(target)
        num_data = function_dist.event_shape.numel()
        return res.div_(num_data) if not res.requires_grad else res / num_data

    def __call__(self, *a, **k):
        return self.forward(*a, **k)
