"""Golden data for the rational quadratic kernel: the reference's own RQKernel (kernels/rq_kernel.py) in fp64 -- full, diagonal,
cross and batched covariances for shared and ARD lengthscales at d in {1, 2, 3} and alpha in {0.05, 0.5, 2, 50, 1e4}, and the
autograd gradients of sum(W * K) with respect to the lengthscale and alpha.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_rq.py    # writes tests/golden/rq_golden.npz

The reference module is loaded on its own.  Its package imports (constraints, the Kernel base class, which needs linear_operator)
are replaced by minimal stand-ins: a base class that stores ard_num_dims / batch_shape, holds the lengthscale parameter and
computes covar_dist(square_dist=True) as the squared Euclidean distance, and an identity constraint (so that the gradients with
respect to the raw parameters are those with respect to the lengthscale and alpha).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rq_golden.npz")
ALPHAS = (0.05, 0.5, 2.0, 50.0, 1e4)


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

    def covar_dist(self, x1, x2, square_dist=False, diag=False, last_dim_is_batch=False, **params):
        if diag:
            d2 = ((x1 - x2) ** 2).sum(-1)
        else:
            d2 = ((x1.unsqueeze(-2) - x2.unsqueeze(-3)) ** 2).sum(-1)
        return d2 if square_dist else d2.sqrt()


def load_reference(ref):
    pkg = types.ModuleType("refgp")
    pkg.__path__ = []
    cons = types.ModuleType("refgp.constraints")
    cons.Interval, cons.Positive = torch.nn.Module, _Identity
    kpkg = types.ModuleType("refgp.kernels")
    kpkg.__path__ = []
    kmod = types.ModuleType("refgp.kernels.kernel")
    kmod.Kernel = _Kernel
    for m in (pkg, cons, kpkg, kmod):
        sys.modules[m.__name__] = m
    name = "refgp.kernels.rq_kernel"
    mod = types.ModuleType(name)
    mod.__package__ = "refgp.kernels"
    path = os.path.join(ref, "gpytorch", "kernels", "rq_kernel.py")
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod.RQKernel


def main(ref):
    RK = load_reference(ref)
    g = torch.Generator().manual_seed(20261018)
    out = {}
    # (d, ard, n1, n2, batch, alpha)
    cases = [(1, False, 7, 5, 0, 0.05), (1, True, 6, 6, 0, 0.5), (2, False, 5, 7, 0, 2.0), (2, True, 6, 4, 0, 50.0),
             (3, False, 5, 5, 0, 1e4), (3, True, 7, 6, 0, 1e4), (2, True, 5, 4, 3, 0.5)]
    for ci, (d, ard, n1, n2, B, alpha) in enumerate(cases):
        bs = torch.Size([B]) if B else torch.Size([])
        kw = {"ard_num_dims": d} if ard else {}
        k = RK(batch_shape=bs, alpha_constraint=_Identity(), **kw).double()
        npar = d if ard else 1
        ls = 0.3 + 1.5 * torch.rand(*bs, 1, npar, generator=g, dtype=torch.float64)
        al = alpha * (1.0 + 0.5 * torch.rand(*bs, 1, generator=g, dtype=torch.float64))
        k.raw_lengthscale.data.copy_(ls)
        k.raw_alpha.data.copy_(al)
        x1 = torch.randn(*bs, n1, d, generator=g, dtype=torch.float64)
        x2 = torch.randn(*bs, n2, d, generator=g, dtype=torch.float64)
        W = torch.randn(*bs, n1, n2, generator=g, dtype=torch.float64)
        K = k.forward(x1, x2)
        (K * W).sum().backward()
        out[f"c{ci}_meta"] = np.array([d, int(ard), n1, n2, B])
        out[f"c{ci}_ls"] = ls.numpy()
        out[f"c{ci}_alpha"] = al.numpy()
        out[f"c{ci}_x1"] = x1.numpy()
        out[f"c{ci}_x2"] = x2.numpy()
        out[f"c{ci}_W"] = W.numpy()
        out[f"c{ci}_K"] = K.detach().numpy()
        out[f"c{ci}_Kxx"] = k.forward(x1, x1).detach().numpy()
        out[f"c{ci}_diag"] = k.forward(x1, x1, diag=True).detach().numpy()
        out[f"c{ci}_gls"] = k.raw_lengthscale.grad.numpy()
        out[f"c{ci}_galpha"] = k.raw_alpha.grad.numpy()
    out["ncases"] = np.array(len(cases))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    ref = os.environ.get("GP_REFERENCE")
    if not ref:
        raise SystemExit("set GP_REFERENCE to a checkout of the reference")
    main(ref)
