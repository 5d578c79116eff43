"""Golden data for the piecewise polynomial kernel: the reference's own PiecewisePolynomialKernel
(kernels/piecewise_polynomial_kernel.py) in fp64 -- full, cross and diagonal covariances for q in {0, 1, 2, 3}, D in {1, 2, 3, 5},
shared and ARD lengthscales, and the autograd gradient of sum(W * K) with respect to the lengthscale.  The module's q = 2
coefficient differs from R&W's (DESIGN 4.24), so the data pins the module, not the textbook.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_ppoly.py    # writes tests/golden/ppoly_golden.npz

The reference module is loaded on its own, as make_golden_rq.py loads its module: the Kernel base class (which needs
linear_operator) is replaced by a stand-in that stores ard_num_dims / batch_shape, holds the lengthscale parameter and computes
covar_dist as the Euclidean distance of direct differences.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_rq import _Kernel  # noqa: E402  (the same stand-in base class)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ppoly_golden.npz")


def load_reference(ref):
    pkg = types.ModuleType("refgp")
    pkg.__path__ = []
    kpkg = types.ModuleType("refgp.kernels")
    kpkg.__path__ = []
    kmod = types.ModuleType("refgp.kernels.kernel")
    kmod.Kernel = _Kernel
    for m in (pkg, kpkg, kmod):
        sys.modules[m.__name__] = m
    name = "refgp.kernels.piecewise_polynomial_kernel"
    mod = types.ModuleType(name)
    mod.__package__ = "refgp.kernels"
    path = os.path.join(ref, "gpytorch", "kernels", "piecewise_polynomial_kernel.py")
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod.PiecewisePolynomialKernel


def main(ref):
    PK = load_reference(ref)
    g = torch.Generator().manual_seed(20261018)
    out = {}
    cases = [(q, D, ard) for q in (0, 1, 2, 3) for D in (1, 2, 3, 5) for ard in (False, True)]
    for ci, (q, D, ard) in enumerate(cases):
        n1, n2 = 7, 6
        kw = {"ard_num_dims": D} if ard else {}
        k = PK(q=q, **kw).double()
        npar = D if ard else 1
        ls = 1.0 + 1.5 * torch.rand(1, npar, generator=g, dtype=torch.float64)
        k.raw_lengthscale.data.copy_(ls)
        x1 = 0.5 * torch.randn(n1, D, generator=g, dtype=torch.float64)
        x2 = 0.5 * torch.randn(n2, D, generator=g, dtype=torch.float64)
        W = torch.randn(n1, n2, generator=g, dtype=torch.float64)
        K = k.forward(x1, x2)
        (K * W).sum().backward()
        out[f"c{ci}_meta"] = np.array([q, D, int(ard), n1, n2])
        out[f"c{ci}_ls"] = ls.numpy()
        out[f"c{ci}_x1"] = x1.numpy()
        out[f"c{ci}_x2"] = x2.numpy()
        out[f"c{ci}_W"] = W.numpy()
        out[f"c{ci}_K"] = K.detach().numpy()
        out[f"c{ci}_Kxx"] = k.forward(x1, x1).detach().numpy()
        out[f"c{ci}_diag"] = k.forward(x1, x1.clone(), diag=True).detach().numpy()
        out[f"c{ci}_gls"] = k.raw_lengthscale.grad.numpy()
    out["ncases"] = np.array(len(cases))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    ref = os.environ.get("GP_REFERENCE")
    if not ref:
        raise SystemExit("set GP_REFERENCE to a checkout of the reference")
    main(ref)
