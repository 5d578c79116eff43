"""Golden data for the polynomial kernel: the reference's own PolynomialKernel (kernels/polynomial_kernel.py) in fp64 -- full,
diagonal, cross and batched covariances for p in {1, 2, 3, 5, 8}, c in {0, 0.1, 10} and d in {1, 3, 8}, including inputs whose
dot products cancel the offset (x2 rows built so that x1 . x2 = -c), and the autograd gradients of sum(W * K) with respect to the
offset.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_poly.py    # writes tests/golden/poly_golden.npz

The reference module is loaded on its own.  Its package imports (constraints, priors, the Kernel base class, which needs
linear_operator) are replaced by minimal stand-ins: a base class that stores batch_shape and sets parameters through
initialize(), and an identity constraint (so that the gradient with respect to the raw offset is the one with respect to c).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "poly_golden.npz")


class _Identity(torch.nn.Module):
    def transform(self, raw):
        return raw

    def inverse_transform(self, value):
        return value


class _Kernel(torch.nn.Module):
    def __init__(self, batch_shape=torch.Size([]), **kwargs):
        super().__init__()
        self.batch_shape = torch.Size(batch_shape)

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


def load_reference(ref):
    pkg = types.ModuleType("refgp")
    pkg.__path__ = []
    cons = types.ModuleType("refgp.constraints")
    cons.Interval, cons.Positive = torch.nn.Module, _Identity
    pri = types.ModuleType("refgp.priors")
    pri.Prior = type("Prior", (), {})
    kpkg = types.ModuleType("refgp.kernels")
    kpkg.__path__ = []
    kmod = types.ModuleType("refgp.kernels.kernel")
    kmod.Kernel = _Kernel
    for m in (pkg, cons, pri, kpkg, kmod):
        sys.modules[m.__name__] = m
    name = "refgp.kernels.polynomial_kernel"
    mod = types.ModuleType(name)
    mod.__package__ = "refgp.kernels"
    path = os.path.join(ref, "gpytorch", "kernels", "polynomial_kernel.py")
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod.PolynomialKernel


def main(ref):
    PK = load_reference(ref)
    g = torch.Generator().manual_seed(20261018)
    out = {}
    # (power, offset, d, n1, n2, batch, cancel)
    cases = [(1, 0.0, 1, 7, 5, 0, False), (2, 0.1, 1, 6, 6, 0, True), (3, 10.0, 3, 5, 7, 0, False), (5, 0.1, 3, 6, 4, 0, True),
             (8, 0.0, 3, 5, 5, 0, False), (2, 10.0, 8, 7, 6, 0, True), (3, 0.1, 8, 5, 4, 3, False), (8, 10.0, 1, 6, 5, 0, True)]
    for ci, (p, c, d, n1, n2, B, cancel) in enumerate(cases):
        bs = torch.Size([B]) if B else torch.Size([])
        k = PK(power=p, batch_shape=bs, offset_constraint=_Identity()).double()
        off = c * (1.0 + 0.2 * torch.rand(*bs, 1, generator=g, dtype=torch.float64))
        k.raw_offset.data.copy_(off)
        x1 = torch.randn(*bs, n1, d, generator=g, dtype=torch.float64) / d ** 0.5
        x2 = torch.randn(*bs, n2, d, generator=g, dtype=torch.float64) / d ** 0.5
        if cancel:   # row 0 of x2 against row 0 of x1: x1_0 . x2_0 = -c, so the base cancels to (rounding of) 0
            x2[..., 0, :] = -off.reshape(*bs, 1) * x1[..., 0, :] / (x1[..., 0, :] ** 2).sum(-1, keepdim=True)
        W = torch.randn(*bs, n1, n2, generator=g, dtype=torch.float64)
        K = k.forward(x1, x2)
        (K * W).sum().backward()
        out[f"c{ci}_meta"] = np.array([p, d, n1, n2, B, int(cancel)])
        out[f"c{ci}_offset"] = off.numpy()
        out[f"c{ci}_x1"] = x1.numpy()
        out[f"c{ci}_x2"] = x2.numpy()
        out[f"c{ci}_W"] = W.numpy()
        out[f"c{ci}_K"] = K.detach().numpy()
        out[f"c{ci}_Kxx"] = k.forward(x1, x1).detach().numpy()
        out[f"c{ci}_diag"] = k.forward(x1, x1, diag=True).detach().numpy()
        out[f"c{ci}_goffset"] = k.raw_offset.grad.numpy()
    out["ncases"] = np.array(len(cases))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    ref = os.environ.get("GP_REFERENCE")
    if not ref:
        raise SystemExit("set GP_REFERENCE to a checkout of the reference")
    main(ref)
