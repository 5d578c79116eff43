"""GaussianLikelihood / FixedNoiseGaussianLikelihood (gpytorch/likelihoods/gaussian_likelihood.py:117-121, :245-363;
noise_models.py:26-92, :150-190).  Module / parameter names follow the reference (`noise_covar.raw_noise`,
`second_noise_covar.raw_noise`) so that state dicts are interchangeable."""
import warnings

import torch

from .constraints import GreaterThan
from .distributions import MultitaskMultivariateNormal, MultivariateNormal
from .module import Module
from .operators import ConstantDiagLinearOperator, DiagLinearOperator


class HomoskedasticNoise(Module):
    """noise_models.py:26-92: one learned sigma^2 (per batch element), returned as a constant-diagonal operator."""

    def __init__(self, noise_prior=None, noise_constraint=None, batch_shape=torch.Size(), num_tasks=1):
        super().__init__()
        self.register_parameter("raw_noise", torch.nn.Parameter(torch.zeros(*batch_shape, num_tasks)))
        self.register_constraint("raw_noise", noise_constraint or GreaterThan(1e-4))  # noise_models.py:29-30

    @property
    def noise(self):
        return self.raw_noise_constraint.transform(self.raw_noise)

    @noise.setter
    def noise(self, value):
        self._set_noise(value)

    def _set_noise(self, value):
        self._set_constrained("raw_noise", value)

    def forward(self, *params, shape=None, **kwargs):
        if shape is None:
            p = params[0] if torch.is_tensor(params[0]) else params[0][0]
            shape = p.shape if p.dim() == 1 else p.shape[:-1]
        return ConstantDiagLinearOperator(self.noise, shape[-1])

    __call__ = forward


class FixedGaussianNoise(Module):
    """noise_models.py:150-190: known per-observation noise variances."""

    def __init__(self, noise):
        super().__init__()
        self.noise = noise

    def forward(self, *params, shape=None, noise=None, **kwargs):
        if shape is None:
            p = params[0] if torch.is_tensor(params[0]) else params[0][0]
            shape = p.shape if p.dim() == 1 else p.shape[:-1]
        if noise is not None:
            return DiagLinearOperator(noise)
        if shape[-1] == self.noise.shape[-1]:
            return DiagLinearOperator(self.noise)
        return None   # ZeroLinearOperator in the reference: sizes do not match and no noise was passed

    __call__ = forward

    def _apply(self, fn):
        self.noise = fn(self.noise)
        return super()._apply(fn)


class _GaussianLikelihoodBase(Module):
    def _shaped_noise_covar(self, base_shape, *params, **kwargs):
        return self.noise_covar(*params, shape=base_shape, **kwargs)

    def marginal(self, function_dist: MultivariateNormal, *params, **kwargs):
        """p(y) = N(mean, K + noise_covar): `covar + noise_covar` (gaussian_likelihood.py:117-121)."""
        mean, covar = function_dist.mean, function_dist.lazy_covariance_matrix
        noise_covar = self._shaped_noise_covar(mean.shape, *params, **kwargs)
        if noise_covar is None:
            return function_dist
        if torch.is_tensor(covar):
            full = covar + noise_covar.to_dense()
        else:
            full = covar + noise_covar
        return function_dist.__class__(mean, full)

    def __call__(self, input, *params, **kwargs):
        if isinstance(input, MultivariateNormal):
            return self.marginal(input, *params, **kwargs)
        raise RuntimeError("Likelihoods expects a MultivariateNormal input to make marginal predictions")


class GaussianLikelihood(_GaussianLikelihoodBase):
    def __init__(self, noise_prior=None, noise_constraint=None, batch_shape=torch.Size(), **kwargs):
        super().__init__()
        self.noise_covar = HomoskedasticNoise(noise_prior=noise_prior, noise_constraint=noise_constraint,
                                              batch_shape=torch.Size(batch_shape))
        self._register_load_state_dict_pre_hook(self._rename_flat_raw_noise)

    @staticmethod
    def _rename_flat_raw_noise(state_dict, prefix, *args):
        # state dicts written by round 1 of this package kept raw_noise at the top level
        if prefix + "raw_noise" in state_dict:
            state_dict[prefix + "noise_covar.raw_noise"] = state_dict.pop(prefix + "raw_noise")

    @property
    def noise(self):
        return self.noise_covar.noise

    @noise.setter
    def noise(self, value):
        self.noise_covar._set_noise(value)

    def _set_noise(self, value):
        self.noise_covar._set_noise(value)

    @property
    def raw_noise(self):
        return self.noise_covar.raw_noise

    @raw_noise.setter
    def raw_noise(self, value):
        self.noise_covar.initialize(raw_noise=value)


class MultitaskHomoskedasticNoise(HomoskedasticNoise):
    """noise_models.py:102-106: one learned sigma^2 per task, raw_noise [*batch_shape, num_tasks]."""

    def __init__(self, num_tasks, noise_prior=None, noise_constraint=None, batch_shape=torch.Size()):
        super().__init__(noise_prior=noise_prior, noise_constraint=noise_constraint, batch_shape=batch_shape, num_tasks=num_tasks)


class HadamardGaussianLikelihood(_GaussianLikelihoodBase):
    """Task-wise noise sigma^2_{t_i} for the Hadamard multitask model (likelihoods/hadamard_gaussian_likelihood.py): the noise
    covariance is the per-row diagonal noise[t] (gp_plan_set_noise_diag on the engine).  The task ids come as the first extra
    argument: a tensor of ids [n] / [n, 1], or the model's inputs (a tuple / list), where the integer-valued tensor is taken, or
    column `task_feature_index` of a single input that carries the task as a feature."""

    def __init__(self, num_tasks, noise_prior=None, noise_constraint=None, batch_shape=torch.Size(), task_feature_index=None,
                 **kwargs):
        super().__init__()
        if noise_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        if len(torch.Size(batch_shape)):
            raise NotImplementedError("a batched HadamardGaussianLikelihood is not available on the accelerated path")
        self.noise_covar = MultitaskHomoskedasticNoise(num_tasks=num_tasks, noise_constraint=noise_constraint,
                                                       batch_shape=torch.Size(batch_shape))
        self.num_tasks = num_tasks
        self.task_feature_index = task_feature_index

    @property
    def noise(self):
        return self.noise_covar.noise

    @noise.setter
    def noise(self, value):
        self.noise_covar._set_noise(value)

    @property
    def raw_noise(self):
        return self.noise_covar.raw_noise

    @raw_noise.setter
    def raw_noise(self, value):
        self.noise_covar.initialize(raw_noise=value)

    def _task_ids(self, params):
        if len(params) == 0 or params[0] is None or (not torch.is_tensor(params[0]) and len(params[0]) == 0):
            raise ValueError("Task indices must be provided.")
        p = params[0]
        if not torch.is_tensor(p):
            ints = [a for a in p if torch.is_tensor(a) and not a.is_floating_point()]
            p = ints[-1] if ints else p[0]
        if p.dim() > 1 and p.shape[-1] > 1:
            if self.task_feature_index is None:
                raise ValueError("Task indices must be a single dimension if task_feature_index is not provided.")
            p = p[..., self.task_feature_index]
        t = p.reshape(-1)
        if t.is_floating_point() and not torch.equal(t, t.round()):
            raise ValueError("Expected task indexes with integer values.")
        return t.long()

    def _shaped_noise_covar(self, base_shape, *params, **kwargs):
        t = self._task_ids(params)
        if t.numel() != base_shape[-1]:
            raise ValueError(f"Expected {base_shape[-1]} task indexes, got {t.numel()}.")
        return DiagLinearOperator(self.noise.reshape(-1)[t])


class FixedNoiseGaussianLikelihood(_GaussianLikelihoodBase):
    """Known heteroscedastic observation noise (+ optionally a learned homoskedastic term): gaussian_likelihood.py:245-363."""

    def __init__(self, noise, learn_additional_noise=False, batch_shape=torch.Size(), **kwargs):
        super().__init__()
        self.noise_covar = FixedGaussianNoise(noise=noise)
        self.second_noise_covar = None
        if learn_additional_noise:
            self.second_noise_covar = HomoskedasticNoise(noise_prior=kwargs.get("noise_prior"),
                                                         noise_constraint=kwargs.get("noise_constraint"),
                                                         batch_shape=torch.Size(batch_shape))

    @property
    def noise(self):
        return self.noise_covar.noise + self.second_noise

    @noise.setter
    def noise(self, value):
        self.noise_covar.noise = value

    @property
    def second_noise(self):
        return 0.0 if self.second_noise_covar is None else self.second_noise_covar.noise

    @second_noise.setter
    def second_noise(self, value):
        if self.second_noise_covar is None:
            raise RuntimeError("Attempting to set secondary learned noise for FixedNoiseGaussianLikelihood, "
                               "but learn_additional_noise must have been False!")
        self.second_noise_covar._set_noise(value)

    def _shaped_noise_covar(self, base_shape, *params, **kwargs):
        res = self.noise_covar(*params, shape=base_shape, **kwargs)
        if self.second_noise_covar is not None:
            second = self.second_noise_covar(*params, shape=base_shape, **kwargs)
            res = second if res is None else res + second
        elif res is None:
            warnings.warn("You have passed data through a FixedNoiseGaussianLikelihood that did not match the size "
                          "of the fixed noise, *and* you did not specify noise. This is treated as a no-op.")
        return res


class MultitaskGaussianLikelihood(_GaussianLikelihoodBase):
    """likelihoods/multitask_gaussian_likelihood.py:162-301 with rank = 0: noise sigma^2 + sigma^2_a on row i T + a of the interleaved
    covariance (:118-154), added through the per-row noise path (gp_plan_set_noise_diag).  `raw_task_noises` [T] and `raw_noise` [1]
    with GreaterThan(1e-4), the reference's names and initialisation."""

    def __init__(self, num_tasks, rank=0, batch_shape=torch.Size(), task_prior=None, noise_prior=None, noise_constraint=None,
                 has_global_noise=True, has_task_noise=True, **kwargs):
        super().__init__()
        if noise_constraint is None:
            noise_constraint = GreaterThan(1e-4)
        if not has_task_noise and not has_global_noise:
            raise ValueError("At least one of has_task_noise or has_global_noise must be specified. "
                             "Attempting to specify a likelihood that has no noise terms.")
        if rank != 0:
            raise NotImplementedError("a task noise covariance of rank > 0 is not available on the accelerated path")
        if noise_prior is not None or task_prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        if len(torch.Size(batch_shape)):
            raise NotImplementedError("a batched MultitaskGaussianLikelihood is not available on the accelerated path")
        if has_task_noise:
            self.register_parameter("raw_task_noises", torch.nn.Parameter(torch.zeros(num_tasks)))
            self.register_constraint("raw_task_noises", noise_constraint)
        if has_global_noise:
            self.register_parameter("raw_noise", torch.nn.Parameter(torch.zeros(1)))
            self.register_constraint("raw_noise", noise_constraint)
        self.num_tasks = num_tasks
        self.rank = rank
        self.has_global_noise = has_global_noise
        self.has_task_noise = has_task_noise

    @property
    def noise(self):
        return self.raw_noise_constraint.transform(self.raw_noise) if self.has_global_noise else None

    @noise.setter
    def noise(self, value):
        self._set_constrained("raw_noise", value)

    @property
    def task_noises(self):
        return self.raw_task_noises_constraint.transform(self.raw_task_noises) if self.has_task_noise else None

    @task_noises.setter
    def task_noises(self, value):
        self._set_constrained("raw_task_noises", value)

    def _task_noise_diag(self, n):
        """[n T]: sigma^2 + sigma^2_a at row i T + a."""
        per_task = None
        if self.has_task_noise:
            per_task = self.task_noises
        if self.has_global_noise:
            per_task = self.noise.expand(self.num_tasks) if per_task is None else per_task + self.noise
        return per_task.repeat(n)

    def _shaped_noise_covar(self, base_shape, *params, **kwargs):
        n, T = base_shape[-2], base_shape[-1]
        if T != self.num_tasks:
            raise RuntimeError(f"the likelihood has {self.num_tasks} tasks, the function has {T}")
        return DiagLinearOperator(self._task_noise_diag(n))

    def marginal(self, function_dist, *params, **kwargs):
        if not isinstance(function_dist, MultitaskMultivariateNormal):
            raise RuntimeError("MultitaskGaussianLikelihood needs a MultitaskMultivariateNormal")
        mean, covar = function_dist.mean, function_dist.lazy_covariance_matrix
        noise_covar = self._shaped_noise_covar(mean.shape, *params, **kwargs)
        full = covar + noise_covar.to_dense() if torch.is_tensor(covar) else covar + noise_covar
        return MultitaskMultivariateNormal(mean, full)
