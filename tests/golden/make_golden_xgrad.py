#!/usr/bin/env python
"""Golden input gradients by EXECUTING the reference's own code (build container only).

The reference differentiates a kernel w.r.t. its inputs through the slow branch of RBFKernel.forward
(kernels/rbf_kernel.py:68-85): x / lengthscale -> covar_dist(square_dist=True) -> postprocess_rbf.  This script loads, as
make_golden.py does, the bodies of `sq_dist` / `dist` (kernels/kernel.py:26-60) and `postprocess_rbf` (kernels/rbf_kernel.py:10-11)
with `ast` and runs them under torch autograd in fp64:
    F = sum_ij W_ij s postprocess_rbf(sq_dist(x1 / l, x2 / l))      ->  dF/dx1, dF/dx2   (cross, one coinciding point pair)
    F = sum_ij W_ij s postprocess_rbf(sq_dist(x / l, x / l, x1_eq_x2=True))  ->  dF/dx   (square)
for scalar and ARD lengthscales.

The Matern slow branch (kernels/matern_kernel.py:94-107) is a method body that reads self.nu / self.lengthscale / self.covar_dist
of a Kernel module (whose module imports linear_operator, absent here), so it cannot be executed standalone; Matern input
gradients are pinned against fp64 autograd through oracle.kernels only.

Outputs: tests/golden/xgrad_golden.npz (committed).  Re-run:  python tests/golden/make_golden_xgrad.py
"""
import ast
import os
import sys

import numpy as np
import torch

REF = os.environ.get("GP_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))


def extract_functions(path, names):
    tree = ast.parse(open(path).read())
    ns = {"torch": torch}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def main():
    sq_dist, _dist = extract_functions(f"{REF}/gpytorch/kernels/kernel.py", ["sq_dist", "dist"])
    (postprocess_rbf,) = extract_functions(f"{REF}/gpytorch/kernels/rbf_kernel.py", ["postprocess_rbf"])
    out = {}
    cases = [("a", 7, 13, 3, False), ("b", 20, 31, 10, True), ("c", 16, 16, 5, False)]
    for tag, n1, n2, d, ard in cases:
        g = torch.Generator().manual_seed(4321 + n1 + d)
        x1 = torch.rand(n1, d, generator=g, dtype=torch.float64)
        x2 = torch.rand(n2, d, generator=g, dtype=torch.float64)
        x2[3] = x1[0]                                                    # one coinciding pair: contributes 0
        ls = torch.linspace(0.4, 1.2, d, dtype=torch.float64) if ard else torch.tensor(0.7, dtype=torch.float64)
        s = 1.7
        W = torch.randn(n1, n2, generator=g, dtype=torch.float64)
        Ws = torch.randn(n1, n1, generator=g, dtype=torch.float64)
        a1, a2 = x1.clone().requires_grad_(), x2.clone().requires_grad_()
        K = s * postprocess_rbf(sq_dist(a1 / ls, a2 / ls, x1_eq_x2=False))
        g1, g2 = torch.autograd.grad((W * K).sum(), (a1, a2))
        a = x1.clone().requires_grad_()
        Ksq = s * postprocess_rbf(sq_dist(a / ls, a / ls, x1_eq_x2=True))
        (gs,) = torch.autograd.grad((Ws * Ksq).sum(), (a,))
        for k, v in (("x1", x1), ("x2", x2), ("ls", ls), ("W", W), ("Wsq", Ws), ("dx1", g1), ("dx2", g2), ("dxsq", gs)):
            out[f"{tag}_{k}"] = v.detach().numpy()
        out[f"{tag}_os"] = np.float64(s)
    path = os.path.join(HERE, "xgrad_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;", len(out), "arrays")


if __name__ == "__main__":
    sys.exit(main())
