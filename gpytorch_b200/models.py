"""ExactGP (gpytorch/models/exact_gp.py:265-333) with the default prediction strategy's mean / covariance
caches (models/exact_prediction_strategies.py:278-321, :371-478) on the engine's solve path."""
import torch

from . import settings
from .distributions import MultivariateNormal
from .likelihoods import _GaussianLikelihoodBase
from .module import Module
from .operators import LOWRANK_MAX_RANK, LowRankUpdatedKernelLinearOperator


def _posterior_covar_mode(k_ss) -> str:
    """Which posterior covariance an exact GP returns: 'skip' (zeros), 'lazy_love' (K** - U U^T as an engine operator: with
    settings.fast_pred_samples, which turns LOVE on by itself as in exact_prediction_strategies.py:787-826, when K** is a
    plan-backed non-SKI operator without batch dimension on an unsharded plan), 'love' (dense LOVE) or 'exact'."""
    if settings.skip_posterior_variances.on():
        return "skip"
    if settings.fast_pred_samples.on():
        return "lazy_love" if LowRankUpdatedKernelLinearOperator.supports(k_ss) else "love"
    return "love" if settings.fast_pred_var.on() else "exact"


class ExactGP(Module):
    def __init__(self, train_inputs, train_targets, likelihood):
        if train_inputs is not None and torch.is_tensor(train_inputs):
            train_inputs = (train_inputs,)
        if not isinstance(likelihood, _GaussianLikelihoodBase):
            raise RuntimeError("ExactGP can only handle Gaussian likelihoods")
        super().__init__()
        self.train_inputs = None if train_inputs is None else tuple(t.unsqueeze(-1) if t.dim() == 1 else t for t in train_inputs)
        self.train_targets = train_targets
        self.likelihood = likelihood
        self._mean_cache = None
        self._covar_cache = None

    def train(self, mode=True):
        if mode:
            self._mean_cache = self._covar_cache = None  # module.py:351-355: train() clears caches
        return super().train(mode)

    def __call__(self, *args, **kwargs):
        inputs = [a.unsqueeze(-1) if a.dim() == 1 else a for a in args]
        if self.training:  # exact_gp.py:265-282
            if self.train_inputs is None:
                raise RuntimeError("train_inputs, train_targets cannot be None in training mode. "
                                   "Call .eval() for prior predictions, or call .set_train_data() to add training data.")
            if not all(torch.equal(ti, inp) for ti, inp in zip(self.train_inputs, inputs)):
                raise RuntimeError("You must train on the training inputs!")
            return self.forward(*inputs, **kwargs)
        if self.train_inputs is None or self.train_targets is None:  # prior mode
            return self.forward(*inputs, **kwargs)
        # posterior mode (exact_gp.py:293-333, DefaultPredictionStrategy): the prior over the JOINT train + test inputs comes
        # from the user's forward() (exact_gp.py:315-322) -- so input transforms, active_dims and any mean module apply to
        # the test points exactly as they do in training -- and its blocks are taken by slicing the lazy covariance
        # (lazy_evaluated_kernel_tensor.py:136-243 re-indexes x1 / x2; nothing is materialised).
        train_x, test_x = self.train_inputs[0], inputs[0]
        n = train_x.size(-2)
        train_out = self.forward(train_x)
        full_out = self.forward(torch.cat([train_x, test_x], dim=-2))
        full_mean, full_covar = full_out.mean, full_out.lazy_covariance_matrix
        with settings._use_eval_tolerance(True):
            khat = self.likelihood(train_out).lazy_covariance_matrix
            if self._mean_cache is None:
                resid = (self.train_targets - train_out.mean).unsqueeze(-1)
                self._mean_cache = khat.solve(resid).squeeze(-1)  # exact_prediction_strategies.py:286
            k_star = full_covar[n:, :n]                           # K(test, train)
            k_ss = full_covar[n:, n:]
            test_mean = full_mean[..., n:] + k_star.matmul(self._mean_cache)  # :396
            m = test_x.size(-2)
            dense = lambda a: a if torch.is_tensor(a) else a.to_dense()  # noqa: E731
            mode = _posterior_covar_mode(k_ss)
            if mode == "skip":                               # exact_prediction_strategies.py:432-433
                covar = torch.zeros(m, m, device=test_x.device)
            elif mode in ("love", "lazy_love"):              # LOVE: :268-272 (cache), :464-478 (use)
                if self._covar_cache is None:
                    init = None
                    if settings.probe_seed.value() is not None:
                        g = torch.Generator(device="cpu").manual_seed(int(settings.probe_seed.value()))
                        init = torch.randn(n, generator=g).to(train_x.device)
                    self._covar_cache = khat.root_inv_decomposition(init).detach()   # [n, J], R R^T ~= K_hat^{-1}
                root = k_star.matmul(self._covar_cache)      # covar_inv_quad_form_root, [m, J]
                if mode == "lazy_love" and root.size(-1) <= LOWRANK_MAX_RANK:
                    covar = LowRankUpdatedKernelLinearOperator(k_ss, root.detach())
                else:
                    covar = dense(k_ss) - root @ root.transpose(-1, -2)
            else:
                rhs = dense(full_covar[:n, n:])          # K(train, test) [n, m]
                corr = k_star.matmul(khat.solve(rhs))    # exact predictive covariance, :435-462
                covar = dense(k_ss) - corr
        return MultivariateNormal(test_mean, covar)

    def set_train_data(self, inputs=None, targets=None, strict=True):
        if inputs is not None:
            if torch.is_tensor(inputs):
                inputs = (inputs,)
            self.train_inputs = tuple(t.unsqueeze(-1) if t.dim() == 1 else t for t in inputs)
        if targets is not None:
            self.train_targets = targets
        self._mean_cache = self._covar_cache = None
