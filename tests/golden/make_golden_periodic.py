"""Golden data for the periodic kernel: the reference's own PeriodicKernel (kernels/periodic_kernel.py) in fp64 -- full, diagonal,
cross and batched covariances for shared and ARD parameters at d in {1, 2, 3}, and the autograd gradients of sum(W * K) with
respect to the lengthscale and the period.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_periodic.py    # writes tests/golden/periodic_golden.npz

The reference module is loaded on its own.  Its package imports (constraints, priors, the Kernel base class, which needs
linear_operator) are replaced by minimal stand-ins: a base class that stores ard_num_dims / batch_shape, holds the lengthscale
parameter and computes covar_dist(last_dim_is_batch=True) as the per-dimension distance |x1_d - x2_d|, and an identity
constraint (so that the gradients with respect to the raw parameters are those with respect to the lengthscale and period).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get("GP_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "periodic_golden.npz")


class _Identity(torch.nn.Module):
    def transform(self, raw):
        return raw

    def inverse_transform(self, value):
        return value


class _Kernel(torch.nn.Module):
    def __init__(self, ard_num_dims=None, batch_shape=torch.Size([]), **kwargs):
        super().__init__()
        self.ard_num_dims = ard_num_dims
        self.batch_shape = torch.Size(batch_shape)
        self.raw_lengthscale = torch.nn.Parameter(torch.zeros(*self.batch_shape, 1, ard_num_dims or 1))

    @property
    def lengthscale(self):
        return self.raw_lengthscale

    def register_parameter(self, name, parameter):   # the reference calls it with keywords
        super().register_parameter(name, parameter)

    def register_constraint(self, name, constraint):
        self.add_module(name + "_constraint", constraint)

    def initialize(self, **kwargs):
        for name, val in kwargs.items():
            p = getattr(self, name)
            with torch.no_grad():
                p.copy_(torch.as_tensor(val, dtype=p.dtype).expand_as(p))
        return self

    def covar_dist(self, x1, x2, diag=False, last_dim_is_batch=False, **params):
        # kernels/kernel.py covar_dist with last_dim_is_batch: one distance matrix per input dimension, [..., d, n, m] ([..., d, n])
        a, b = x1.transpose(-1, -2).unsqueeze(-1), x2.transpose(-1, -2).unsqueeze(-1)
        if diag:
            return (a - b).abs().squeeze(-1)
        return (a - b.transpose(-1, -2)).abs()


def load_reference(ref=REF):
    pkg = types.ModuleType("refgp")
    pkg.__path__ = []
    cons = types.ModuleType("refgp.constraints")
    cons.Interval, cons.Positive = torch.nn.Module, _Identity
    pri = types.ModuleType("refgp.priors")
    pri.Prior = object
    kpkg = types.ModuleType("refgp.kernels")
    kpkg.__path__ = []
    kmod = types.ModuleType("refgp.kernels.kernel")
    kmod.Kernel = _Kernel
    for m in (pkg, cons, pri, kpkg, kmod):
        sys.modules[m.__name__] = m
    name = "refgp.kernels.periodic_kernel"
    mod = types.ModuleType(name)
    mod.__package__ = "refgp.kernels"
    path = os.path.join(ref, "gpytorch", "kernels", "periodic_kernel.py")
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod.PeriodicKernel


def main(ref=REF):
    PK = load_reference(ref)
    g = torch.Generator().manual_seed(20261017)
    out = {}
    # (d, ard, n1, n2, batch)
    cases = [(1, False, 7, 5, 0), (1, True, 6, 6, 0), (2, False, 5, 7, 0), (2, True, 6, 4, 0), (3, False, 5, 5, 0),
             (3, True, 7, 6, 0), (2, True, 5, 4, 3)]
    for ci, (d, ard, n1, n2, B) in enumerate(cases):
        bs = torch.Size([B]) if B else torch.Size([])
        kw = {"ard_num_dims": d} if ard else {}
        k = PK(batch_shape=bs, period_length_constraint=_Identity(), **kw).double()
        npar = d if ard else 1
        ls = 0.3 + 1.5 * torch.rand(*bs, 1, npar, generator=g, dtype=torch.float64)
        per = 0.5 + 2.0 * torch.rand(*bs, 1, npar, generator=g, dtype=torch.float64)
        k.raw_lengthscale.data.copy_(ls)
        k.raw_period_length.data.copy_(per)
        x1 = 4.0 * torch.randn(*bs, n1, d, generator=g, dtype=torch.float64)
        x2 = 4.0 * torch.randn(*bs, n2, d, generator=g, dtype=torch.float64)
        W = torch.randn(*bs, n1, n2, generator=g, dtype=torch.float64)
        K = k.forward(x1, x2)
        (K * W).sum().backward()
        out[f"c{ci}_meta"] = np.array([d, int(ard), n1, n2, B])
        out[f"c{ci}_ls"] = ls.numpy()
        out[f"c{ci}_per"] = per.numpy()
        out[f"c{ci}_x1"] = x1.numpy()
        out[f"c{ci}_x2"] = x2.numpy()
        out[f"c{ci}_W"] = W.numpy()
        out[f"c{ci}_K"] = K.detach().numpy()
        out[f"c{ci}_Kxx"] = k.forward(x1, x1).detach().numpy()
        out[f"c{ci}_diag"] = k.forward(x1, x1, diag=True).detach().numpy()
        out[f"c{ci}_gls"] = k.raw_lengthscale.grad.numpy()
        out[f"c{ci}_gper"] = k.raw_period_length.grad.numpy()
    out["ncases"] = np.array(len(cases))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    main()
