"""Golden data for the spectral mixture kernel: the reference's own SpectralMixtureKernel (kernels/spectral_mixture_kernel.py) in
fp64 -- full, diagonal, cross and batched covariances for several (Q, d), the autograd gradients of sum(W * K) with respect to the
weights, means and scales, and initialize_from_data under fixed torch seeds.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_spectral.py    # writes tests/golden/spectral_golden.npz

The reference module is loaded on its own.  Its package imports (constraints, priors, the Kernel base class, which needs
linear_operator) are replaced by minimal stand-ins: a base class that stores ard_num_dims / batch_shape / active_dims and copies
values into raw parameters, the softplus Positive constraint, and an identity constraint for the gradient cases (so that the
gradients with respect to the raw parameters are those with respect to the weights, means and scales themselves).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get("GP_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "spectral_golden.npz")


class _Positive(torch.nn.Module):
    def transform(self, raw):
        return torch.nn.functional.softplus(raw)

    def inverse_transform(self, value):
        return value + torch.log(-torch.expm1(-value))


class _Identity(torch.nn.Module):
    def transform(self, raw):
        return raw

    def inverse_transform(self, value):
        return value


class _Kernel(torch.nn.Module):
    def __init__(self, ard_num_dims=None, batch_shape=torch.Size([]), active_dims=None, **kwargs):
        super().__init__()
        self.ard_num_dims = ard_num_dims
        self.batch_shape = torch.Size(batch_shape)
        self.active_dims = active_dims

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


def load_reference(ref=REF):
    pkg = types.ModuleType("refgp")
    pkg.__path__ = []
    cons = types.ModuleType("refgp.constraints")
    cons.Interval, cons.Positive = torch.nn.Module, _Positive
    pri = types.ModuleType("refgp.priors")
    pri.Prior = object
    kpkg = types.ModuleType("refgp.kernels")
    kpkg.__path__ = []
    kmod = types.ModuleType("refgp.kernels.kernel")
    kmod.Kernel = _Kernel
    for m in (pkg, cons, pri, kpkg, kmod):
        sys.modules[m.__name__] = m
    name = "refgp.kernels.spectral_mixture_kernel"
    mod = types.ModuleType(name)
    mod.__package__ = "refgp.kernels"
    path = os.path.join(ref, "gpytorch", "kernels", "spectral_mixture_kernel.py")
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod.SpectralMixtureKernel


def main(ref=REF):
    SM = load_reference(ref)
    g = torch.Generator().manual_seed(20261017)
    out = {}
    cases = [(1, 1, 6, 5), (4, 1, 7, 9), (3, 2, 5, 6), (2, 3, 6, 4), (4, 4, 5, 7), (4, 8, 4, 5)]
    for ci, (Q, d, n1, n2) in enumerate(cases):
        k = SM(num_mixtures=Q, ard_num_dims=d, mixture_scales_constraint=_Identity(), mixture_means_constraint=_Identity(),
               mixture_weights_constraint=_Identity()).double()
        w = torch.rand(Q, generator=g, dtype=torch.float64) * 1.5 + 0.2
        mu = torch.rand(Q, 1, d, generator=g, dtype=torch.float64) * 0.8 + 0.05
        v = torch.rand(Q, 1, d, generator=g, dtype=torch.float64) * 0.6 + 0.1
        with torch.no_grad():
            k.raw_mixture_weights.copy_(w)
            k.raw_mixture_means.copy_(mu)
            k.raw_mixture_scales.copy_(v)
        x1 = (torch.rand(n1, d, generator=g, dtype=torch.float64) * 6 - 3).float().double()   # fp32-representable inputs
        x2 = (torch.rand(n2, d, generator=g, dtype=torch.float64) * 6 - 3).float().double()
        W = torch.randn(n1, n2, generator=g, dtype=torch.float64)
        Kx = k.forward(x1, x2)
        (Kx * W).sum().backward()
        p = f"c{ci}_"
        out[p + "shape"] = np.array([Q, d])
        out[p + "x1"], out[p + "x2"], out[p + "w"], out[p + "mu"], out[p + "v"], out[p + "W"] = (
            t.numpy() for t in (x1, x2, w, mu, v, W))
        out[p + "K12"] = Kx.detach().numpy()
        out[p + "gw"] = k.raw_mixture_weights.grad.numpy()
        out[p + "gmu"] = k.raw_mixture_means.grad.numpy()
        out[p + "gv"] = k.raw_mixture_scales.grad.numpy()
        with torch.no_grad():
            out[p + "K11"] = k.forward(x1, x1).numpy()
            out[p + "diag"] = k.forward(x1, x1, diag=True).numpy()
            m = min(n1, n2)
            out[p + "diag12"] = k.forward(x1[:m], x2[:m], diag=True).numpy()
    # batched: batch_shape [2] over [2, n, d] inputs
    kb = SM(num_mixtures=3, ard_num_dims=2, batch_shape=torch.Size([2]), mixture_scales_constraint=_Identity(),
            mixture_means_constraint=_Identity(), mixture_weights_constraint=_Identity()).double()
    with torch.no_grad():
        kb.raw_mixture_weights.copy_(torch.rand(2, 3, generator=g, dtype=torch.float64) + 0.3)
        kb.raw_mixture_means.copy_(torch.rand(2, 3, 1, 2, generator=g, dtype=torch.float64) * 0.5 + 0.05)
        kb.raw_mixture_scales.copy_(torch.rand(2, 3, 1, 2, generator=g, dtype=torch.float64) * 0.5 + 0.1)
        xb = (torch.rand(2, 6, 2, generator=g, dtype=torch.float64) * 4 - 2).float().double()
        out["b_w"], out["b_mu"], out["b_v"], out["b_x"] = (t.numpy() for t in (kb.raw_mixture_weights, kb.raw_mixture_means,
                                                                              kb.raw_mixture_scales, xb))
        out["b_K"] = kb.forward(xb, xb).numpy()
    # initialize_from_data with the default Positive constraints, float32 parameters, fixed torch seeds
    for ii, (Q, d, n, bs) in enumerate([(4, 1, 15, []), (3, 2, 20, []), (2, 1, 12, [2])]):
        x = torch.rand(n, d, generator=g) * 5
        x[3] = x[1]                                              # a repeated point: zero gaps are skipped
        y = torch.randn(n, generator=g)
        ki = SM(num_mixtures=Q, ard_num_dims=d, batch_shape=torch.Size(bs))
        torch.manual_seed(100 + ii)
        ki.initialize_from_data(x, y)
        p = f"i{ii}_"
        out[p + "cfg"] = np.array([Q, d, n, len(bs) and bs[0]])
        out[p + "x"], out[p + "y"] = x.numpy(), y.numpy()
        out[p + "w"] = ki.mixture_weights.detach().numpy()
        out[p + "mu"] = ki.mixture_means.detach().numpy()
        out[p + "v"] = ki.mixture_scales.detach().numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays")


if __name__ == "__main__":
    main()
