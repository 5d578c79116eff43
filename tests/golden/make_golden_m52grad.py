#!/usr/bin/env python
"""Golden vectors for Matern52KernelGrad, produced by EXECUTING the reference's own `Matern52KernelGrad.forward` on the CPU in fp64.
`gpytorch/kernels/matern52_kernel_grad.py` imports KroneckerProductLinearOperator (linear_operator, absent) and MaternKernel from
the kernel package, which pulls in the rest of gpytorch.  Its source is read where it lies, those two import statements are
dropped, and the class body is executed against stand-ins: a MaternKernel stub with `lengthscale`, `covar_dist` (the Euclidean
distance) and `forward(diag=True)` (the Matern diagonal of x1 == x2 is 1), and a KroneckerProductLinearOperator whose to_dense()
is torch.kron.  The known-answer test of `test/kernels/test_matern52_kernel_grad.py` (its inputs and expected matrix) is read
from that file as data.  Nothing is copied into the repo.
Output: tests/golden/m52grad_golden.npz (committed).  Re-run:  python tests/golden/make_golden_m52grad.py
"""
import ast
import math
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


class _MaternStub:
    """The members Matern52KernelGrad reads from its base: lengthscale [1, d or 1], covar_dist and forward(diag=True)."""

    def __init__(self, nu=2.5, lengthscale=None):
        self.nu = nu
        self.lengthscale = lengthscale

    def covar_dist(self, x1, x2, diag=False, **params):
        return ((x1[:, None, :] - x2[None, :, :]) ** 2).sum(-1).sqrt()

    def forward(self, x1, x2, diag=False, **params):
        return torch.ones(x1.shape[:-1], dtype=x1.dtype)


def load_reference():
    path = f"{REF}/gpytorch/kernels/matern52_kernel_grad.py"
    src = open(path).read()
    keep = [ln for ln in src.splitlines() if not ln.startswith("from linear_operator") and not ln.startswith("from gpytorch.kernels")]
    ns = {"KroneckerProductLinearOperator": _Kron, "MaternKernel": _MaternStub, "__name__": "ref_matern52_kernel_grad"}
    exec(compile("\n".join(keep), path, "exec"), ns)
    return ns["Matern52KernelGrad"]


def known_answer():
    """(a, b, expected) of the reference's test_kernel: the literals of its torch.tensor(...) calls, evaluated as data."""
    tree = ast.parse(open(f"{REF}/test/kernels/test_matern52_kernel_grad.py").read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "test_kernel")
    vals = {}
    for st in fn.body:
        if isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Name) and isinstance(st.value, ast.Call) and st.value.args:
            name = st.targets[0].id
            if name in ("a", "b", "actual"):
                vals[name] = np.array(ast.literal_eval(st.value.args[0]), dtype=np.float64)
    return vals["a"][0], vals["b"][0], vals["actual"]


def main():
    Matern52KernelGrad = load_reference()
    out = {}
    g = torch.Generator().manual_seed(2025)
    for d in (1, 2, 5):
        for ard in (False, True):
            ls = (0.4 + torch.rand(1, d, generator=g, dtype=torch.float64)) if ard else torch.tensor([[0.7]], dtype=torch.float64)
            k = Matern52KernelGrad(lengthscale=ls)
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
    a, b, actual = known_answer()
    out["ka_a"], out["ka_b"], out["ka_expected"] = a, b, actual
    out["ka_ls"] = np.array([math.log(2.0)])   # the reference's default lengthscale: softplus(0)
    out["ka_reference_fp64"] = Matern52KernelGrad(lengthscale=torch.tensor([[math.log(2.0)]], dtype=torch.float64)).forward(
        torch.tensor(a), torch.tensor(b)).numpy()
    np.savez_compressed(os.path.join(HERE, "m52grad_golden.npz"), **out)


if __name__ == "__main__":
    main()
