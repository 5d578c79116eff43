"""Mean functions (gpytorch/means/constant_mean.py:33-113, zero_mean.py).  Parameter names and shapes follow the
reference (`raw_constant` of shape batch_shape) so that state dicts are interchangeable."""
from copy import deepcopy

import torch

from .module import Module


class ZeroMean(Module):
    def __init__(self, batch_shape=torch.Size(), **kwargs):
        super().__init__()
        self.batch_shape = torch.Size(batch_shape)

    def forward(self, x):
        shape = torch.broadcast_shapes(self.batch_shape, x.shape[:-2]) + x.shape[-2:-1]
        return torch.zeros(shape, dtype=x.dtype, device=x.device)

    __call__ = forward


class ConstantMean(Module):
    def __init__(self, constant_prior=None, constant_constraint=None, batch_shape=torch.Size(), **kwargs):
        super().__init__()
        self.batch_shape = torch.Size(batch_shape)
        self.register_parameter("raw_constant", torch.nn.Parameter(torch.zeros(self.batch_shape)))
        if constant_constraint is not None:
            self.register_constraint("raw_constant", constant_constraint)
        self._register_load_state_dict_pre_hook(self._rename_old_constant)

    @staticmethod
    def _rename_old_constant(state_dict, prefix, *args):
        # constant_mean.py:18-31: `constant` (batch_shape x 1) was renamed to `raw_constant` (batch_shape)
        if prefix + "constant" in state_dict:
            state_dict[prefix + "raw_constant"] = state_dict.pop(prefix + "constant").squeeze(-1)

    @property
    def constant(self):
        c = self.constraint_for("raw_constant")
        return self.raw_constant if c is None else c.transform(self.raw_constant)

    @constant.setter
    def constant(self, value):
        self._set_constant(value)

    def _set_constant(self, value):
        self._set_constrained("raw_constant", value)

    def forward(self, x):
        constant = self.constant.unsqueeze(-1)                  # constant_mean.py:111-113
        return constant.expand(torch.broadcast_shapes(constant.shape, x.shape[:-1]))

    def __call__(self, x):
        return self.forward(x)


class ConstantMeanGrad(Module):
    """means/constant_mean_grad.py: a constant mean for the value and zero for the d partial derivatives.  The parameter is named
    `constant` with shape [*batch_shape, 1], as in the reference, so state dicts interchange; forward returns [*batch, n, d + 1]."""

    def __init__(self, prior=None, batch_shape=torch.Size(), **kwargs):
        super().__init__()
        if prior is not None:
            raise NotImplementedError("priors are not available on the accelerated path")
        self.batch_shape = torch.Size(batch_shape)
        self.register_parameter("constant", torch.nn.Parameter(torch.zeros(*self.batch_shape, 1)))

    def forward(self, input):
        shape = torch.broadcast_shapes(self.batch_shape, input.shape[:-2]) + input.shape[-2:-1]
        value = self.constant.unsqueeze(-2).expand(*shape, 1)                        # [*batch, n, 1]
        return torch.cat([value, value.new_zeros(*shape, input.size(-1))], dim=-1)   # zero mean for the d derivatives

    def __call__(self, input):
        return self.forward(input)


class MultitaskMean(Module):
    """means/multitask_mean.py:20-45: one mean per task (a single mean is deep-copied T times); forward returns [n, T]."""

    def __init__(self, base_means, num_tasks):
        super().__init__()
        if isinstance(base_means, Module):
            base_means = [base_means]
        if not isinstance(base_means, list) or (len(base_means) != 1 and len(base_means) != num_tasks):
            raise RuntimeError("base_means should be a list of means of length either 1 or num_tasks")
        if len(base_means) == 1:
            base_means = base_means + [deepcopy(base_means[0]) for _ in range(num_tasks - 1)]
        self.base_means = torch.nn.ModuleList(base_means)
        self.num_tasks = num_tasks

    def forward(self, input):
        return torch.cat([sub_mean(input).unsqueeze(-1) for sub_mean in self.base_means], dim=-1)

    def __call__(self, input):
        return self.forward(input)
