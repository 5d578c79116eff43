#!/usr/bin/env python
"""Golden vectors for RBFKernelGrad, produced by EXECUTING the reference's own `RBFKernelGrad.forward` on the CPU in fp64.
`gpytorch/kernels/rbf_kernel_grad.py` imports KroneckerProductLinearOperator (linear_operator, absent) and `postprocess_rbf` /
`RBFKernel` from the kernel package, which pulls in the rest of gpytorch.  Its source is read where it lies, those two import
statements are dropped, and the class body is executed against stand-ins: a stub base with `lengthscale` and
`covar_dist(square_dist=True)`, `postprocess_rbf(d) = exp(-d / 2)` and a KroneckerProductLinearOperator whose to_dense() is
torch.kron.  Nothing is copied into the repo.
Output: tests/golden/deriv_golden.npz (committed).  Re-run:  python tests/golden/make_golden_deriv.py
"""
import os

import numpy as np
import torch

REF = os.environ.get("GP_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))


class _Kron:
    def __init__(self, a, b):
        self.a, self.b = a, b

    def to_dense(self):
        return torch.kron(self.a, self.b)


class _RBFStub:
    """The two members RBFKernelGrad.forward reads from its base: lengthscale [1, d or 1] and covar_dist; forward(diag=True) for
    the diagonal branch (the RBF diagonal of x1 == x2 is 1)."""

    def __init__(self, lengthscale):
        self.lengthscale = lengthscale

    def covar_dist(self, x1, x2, square_dist=True, **params):
        return ((x1[:, None, :] - x2[None, :, :]) ** 2).sum(-1)

    def forward(self, x1, x2, diag=False, **params):
        return torch.ones(x1.shape[:-1], dtype=x1.dtype)


def load_reference():
    src = open(f"{REF}/gpytorch/kernels/rbf_kernel_grad.py").read()
    keep = [ln for ln in src.splitlines() if not ln.startswith("from linear_operator") and not ln.startswith("from .rbf_kernel")]
    ns = {"KroneckerProductLinearOperator": _Kron, "postprocess_rbf": lambda d: d.div_(-2).exp_(), "RBFKernel": _RBFStub,
          "__name__": "ref_rbf_kernel_grad"}
    exec(compile("\n".join(keep), f"{REF}/gpytorch/kernels/rbf_kernel_grad.py", "exec"), ns)
    return ns["RBFKernelGrad"]


def main():
    RBFKernelGrad = load_reference()
    out = {}
    g = torch.Generator().manual_seed(2024)
    for d in (1, 2, 5):
        for ard in (False, True):
            ls = (0.4 + torch.rand(1, d, generator=g, dtype=torch.float64)) if ard else torch.tensor([[0.7]], dtype=torch.float64)
            k = RBFKernelGrad(ls)
            x1 = torch.rand(7, d, generator=g, dtype=torch.float64)
            x2 = torch.rand(5, d, generator=g, dtype=torch.float64)
            x2[0] = x1[3]                       # a coincident pair in the cross block
            tag = f"d{d}_{'ard' if ard else 'iso'}"
            out[f"{tag}_ls"] = ls.reshape(-1).numpy()
            out[f"{tag}_x1"] = x1.numpy()
            out[f"{tag}_x2"] = x2.numpy()
            out[f"{tag}_square"] = k.forward(x1, x1).numpy()
            out[f"{tag}_cross"] = k.forward(x1, x2).numpy()
            out[f"{tag}_diag"] = k.forward(x1, x1, diag=True).numpy()
    np.savez_compressed(os.path.join(HERE, "deriv_golden.npz"), **out)


if __name__ == "__main__":
    main()
