"""ExactGP (gpytorch/models/exact_gp.py:265-333) with the default prediction strategy's mean / covariance
caches (models/exact_prediction_strategies.py:278-321, :371-478) on the engine's solve path, and the KISS-GP
grid caches of InterpolatedPredictionStrategy (:481-827) behind settings.ski_grid_prediction."""
import torch

from . import settings
from .distributions import MultitaskMultivariateNormal, MultivariateNormal
from .likelihoods import _GaussianLikelihoodBase
from .module import Module
from .operators import LOWRANK_MAX_RANK, LowRankUpdatedKernelLinearOperator, MaskedLinearOperator, SKIKernelLinearOperator

# Largest grid LOVE cache C = s K_uu W^T R (M x J fp32) the grid path builds; above it the covariance takes the joint path.  At
# the 100^3 grid of a 10^6-point KISS-GP model and J = 100 the cache is 400 MB; a 128^4 grid would need 100 GB.
SKI_GRID_LOVE_MAX_BYTES = 2 * 2**30


def _posterior_covar_mode(k_ss) -> str:
    """Which posterior covariance an exact GP returns: 'skip' (zeros), 'lazy_love' (K** - U U^T as an engine operator: with
    settings.fast_pred_samples, which turns LOVE on by itself as in exact_prediction_strategies.py:787-826, when K** is a
    plan-backed non-SKI operator without batch dimension on an unsharded plan), 'love' (dense LOVE) or 'exact'."""
    if settings.skip_posterior_variances.on():
        return "skip"
    if settings.fast_pred_samples.on():
        return "lazy_love" if LowRankUpdatedKernelLinearOperator.supports(k_ss) else "love"
    return "love" if settings.fast_pred_var.on() else "exact"


def _ski_grid_mode(train_op, test_op, J=None):
    """How a KISS-GP model predicts with settings.ski_grid_prediction on.  None: today's joint path, unchanged -- the flag is off,
    or the training covariance is not an unbatched, unsharded SKIKernelLinearOperator, or the test prior forward(test_x) is not a
    SKI operator on the same grid with the same kind, lengthscale and outputscale.  Otherwise the mean comes from the grid cache
    c = s K_uu W^T alpha and the covariance is
      'skip'        zeros (skip_posterior_variances wins, as on the joint path);
      'exact'       the joint path's exact covariance (neither LOVE flag: the reference's InterpolatedPredictionStrategy falls
                    back to the default strategy there, exact_prediction_strategies.py:788-789);
      'love'        a LOVE flag is on and the rank J of R is not known yet: ask again with J;
      'joint_love'  the grid cache C (M x J fp32) would exceed SKI_GRID_LOVE_MAX_BYTES: the joint path's dense LOVE;
      'lazy_love'   J <= 128: K**_test - U U^T, U = W* C, lazy on the test-only SKI plan;
      'dense_love'  J > 128: test_op.to_dense() - U U^T (products over the m test points only)."""
    if settings.ski_grid_prediction.off():
        return None
    if type(train_op) is not SKIKernelLinearOperator or not train_op.same_grid(test_op):
        return None
    for op in (train_op, test_op):
        if op._comm is not None or op._row_begin != 0 or op._row_count not in (0, op.shape[0]):
            return None
    if settings.skip_posterior_variances.on():
        return "skip"
    if settings.fast_pred_var.off() and settings.fast_pred_samples.off():
        return "exact"
    if J is None:
        return "love"
    M = 1
    for g in train_op.grid_sizes:
        M *= int(g)
    if M * int(J) * 4 > SKI_GRID_LOVE_MAX_BYTES:
        return "joint_love"
    return "lazy_love" if J <= LOWRANK_MAX_RANK else "dense_love"


def _dense(a):
    return a if torch.is_tensor(a) else a.to_dense()


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
        self._clear_caches()

    def _clear_caches(self):
        self._mean_cache = self._covar_cache = None
        self._cache_observed = None   # the observed-row mask the two caches were built for (None: every row)
        self._grid_mean_cache = self._grid_covar_cache = None   # c = s K_uu W^T alpha [M], C = s K_uu W^T R [M, J]

    def train(self, mode=True):
        if mode:
            self._clear_caches()  # module.py:351-355: train() clears caches
        return super().train(mode)

    def _love_root(self, khat, train_x):
        """R [n, J] with R R^T ~= K_hat^{-1} (exact_prediction_strategies.py:268-272), cached and detached."""
        if self._covar_cache is None:
            init = None
            if settings.probe_seed.value() is not None:
                g = torch.Generator(device="cpu").manual_seed(int(settings.probe_seed.value()))
                init = torch.randn(khat.shape[-1], generator=g).to(train_x.device)   # n (n T rows for a multitask model)
            self._covar_cache = khat.root_inv_decomposition(init).detach()
        return self._covar_cache

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
        multi = len(self.train_inputs) > 1
        if multi:
            # several inputs (e.g. x and the task index of a Hadamard multitask model): every input is concatenated, train then
            # test, for the joint forward, and the likelihood sees the train inputs (exact_prediction_strategies.py passes them)
            if len(inputs) != len(self.train_inputs):
                raise RuntimeError(f"the model was trained on {len(self.train_inputs)} inputs, got {len(inputs)}")
            train_out = self.forward(*self.train_inputs)
            full_out = self.forward(*[torch.cat([a, b], dim=-2) for a, b in zip(self.train_inputs, inputs)])
            lik_params = (self.train_inputs,)
        else:
            train_out = self.forward(train_x)
            if settings.ski_grid_prediction.on():
                test_out = self.forward(test_x)
                mode = _ski_grid_mode(train_out.lazy_covariance_matrix, test_out.lazy_covariance_matrix)
                if mode is not None:
                    return self._ski_grid_posterior(train_x, test_x, train_out, test_out, mode)
            full_out = self.forward(torch.cat([train_x, test_x], dim=-2))
            lik_params = ()
        full_mean, full_covar = full_out.mean, full_out.lazy_covariance_matrix
        # a Kronecker multitask model (MultitaskMultivariateNormal): every covariance block is over the interleaved rows i T + a,
        # so the joint operator is sliced at n T and the means are [n, T] (flattened row-major for the solves)
        multitask = isinstance(train_out, MultitaskMultivariateNormal)
        # settings.observation_nan_policy "mask" / "fill" (the same posterior here): condition on the observed rows only
        # (exact_prediction_strategies.py:278-321, :393-410); the rows of a multitask model are the interleaved i T + a
        observed = None
        if settings.observation_nan_policy.value() != "ignore":
            event = self.train_targets.shape[-2:] if multitask else self.train_targets.shape[-1:]
            obs = settings.observation_nan_policy._get_observed(self.train_targets, event).reshape(-1)
            observed = None if bool(obs.all()) else obs
        if (observed is None) != (self._cache_observed is None) or (observed is not None and not torch.equal(observed, self._cache_observed)):
            self._clear_caches()
            self._cache_observed = observed
        with settings._use_eval_tolerance(True):
            khat = self.likelihood(train_out, *lik_params).lazy_covariance_matrix
            if multitask:
                T = train_out.num_tasks
                n_rows = n * T
                resid = (self.train_targets - train_out.mean).reshape(-1, 1)
                k_star = full_covar[n_rows:, :n_rows]
                k_ss = full_covar[n_rows:, n_rows:]
                m = test_x.size(-2) * T
            else:
                n_rows = n
                resid = (self.train_targets - train_out.mean).unsqueeze(-1)
                k_star = full_covar[n:, :n]                           # K(test, train)
                k_ss = full_covar[n:, n:]
                m = test_x.size(-2)
            if observed is not None:   # K_hat over the observed rows, the observed columns of K(test, train)
                khat = MaskedLinearOperator(khat, observed, observed)
                k_star = MaskedLinearOperator(k_star, None, observed)
            if self._mean_cache is None:
                if observed is None:
                    self._mean_cache = khat.solve(resid).squeeze(-1)  # exact_prediction_strategies.py:286
                else:                                                 # NaN on the missing rows, as :298-307
                    cache = torch.full((n_rows,), float("nan"), device=resid.device, dtype=resid.dtype)
                    cache[observed] = khat.solve(resid[observed]).squeeze(-1)
                    self._mean_cache = cache
            cache = self._mean_cache if observed is None else self._mean_cache[observed]
            if multitask:
                test_mean = (full_mean[n:].reshape(-1) + k_star.matmul(cache)).reshape(-1, T)
            else:
                test_mean = full_mean[..., n:] + k_star.matmul(cache)  # :396
            mode = _posterior_covar_mode(k_ss)
            if mode == "skip":                               # exact_prediction_strategies.py:432-433
                covar = torch.zeros(m, m, device=test_x.device)
            elif mode in ("love", "lazy_love"):              # LOVE: :268-272 (cache), :464-478 (use)
                root = k_star.matmul(self._love_root(khat, train_x))   # covar_inv_quad_form_root, [m, J]
                if mode == "lazy_love" and root.size(-1) <= LOWRANK_MAX_RANK:
                    covar = LowRankUpdatedKernelLinearOperator(k_ss, root.detach())
                else:
                    covar = _dense(k_ss) - root @ root.transpose(-1, -2)
            else:
                rhs = _dense(full_covar[:n_rows, n_rows:])   # K(train, test) [n, m]
                if observed is not None:
                    rhs = rhs[observed]
                corr = k_star.matmul(khat.solve(rhs))        # exact predictive covariance, :435-462
                covar = _dense(k_ss) - corr
        if multitask:
            return MultitaskMultivariateNormal(test_mean, covar)
        return MultivariateNormal(test_mean, covar)

    def _ski_grid_posterior(self, train_x, test_x, train_out, test_out, mode):
        """InterpolatedPredictionStrategy (exact_prediction_strategies.py:481-827) on the engine: the caches live on the grid and
        every predict call interpolates them to the test points; see _ski_grid_mode for the covariance branches.  Deviations: R
        is the engine's Lanczos root of K_hat (started from probe_seed like the joint path, not from interpolated grid probes,
        :687-726); under fast_pred_samples the same lazy LOVE operator is sampled (the reference roots K_uu - C C^T, :733-739);
        all caches are detached (detach_test_caches)."""
        train_op, test_op = train_out.lazy_covariance_matrix, test_out.lazy_covariance_matrix
        m = test_x.size(-2)
        with settings._use_eval_tolerance(True):
            khat = self.likelihood(train_out).lazy_covariance_matrix
            if self._mean_cache is None:
                resid = (self.train_targets - train_out.mean).unsqueeze(-1)
                self._mean_cache = khat.solve(resid).squeeze(-1)
            if self._grid_mean_cache is None:
                self._grid_mean_cache = train_op.grid_matmul(self._mean_cache)            # mean_cache, :578-606
            test_mean = test_out.mean + test_op.interp_matmul(self._grid_mean_cache)   # exact_predictive_mean, :780-786
            if mode == "skip":
                return MultivariateNormal(test_mean, torch.zeros(m, m, device=test_x.device))
            if mode == "love":
                R = self._love_root(khat, train_x)
                mode = _ski_grid_mode(train_op, test_op, R.size(-1))
            if mode in ("exact", "joint_love"):
                n = train_x.size(-2)
                full_covar = self.forward(torch.cat([train_x, test_x], dim=-2)).lazy_covariance_matrix
                k_star, k_ss = full_covar[n:, :n], full_covar[n:, n:]
                if mode == "joint_love":
                    root = k_star.matmul(self._covar_cache)
                    covar = _dense(k_ss) - root @ root.transpose(-1, -2)
                else:
                    covar = _dense(k_ss) - k_star.matmul(khat.solve(_dense(full_covar[:n, n:])))
                return MultivariateNormal(test_mean, covar)
            if self._grid_covar_cache is None:
                self._grid_covar_cache = train_op.grid_matmul(self._covar_cache)      # covar_cache, :490-503, :679-746
            U = test_op.interp_matmul(self._grid_covar_cache)                        # [m, J]
            if mode == "lazy_love":
                covar = LowRankUpdatedKernelLinearOperator.on_ski(test_op, U)
            else:
                covar = test_op.to_dense() - U @ U.transpose(-1, -2)
        return MultivariateNormal(test_mean, covar)

    def set_train_data(self, inputs=None, targets=None, strict=True):
        if inputs is not None:
            if torch.is_tensor(inputs):
                inputs = (inputs,)
            self.train_inputs = tuple(t.unsqueeze(-1) if t.dim() == 1 else t for t in inputs)
        if targets is not None:
            self.train_targets = targets
        self._clear_caches()
