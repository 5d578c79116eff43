#!/usr/bin/env python
"""Golden kernel-product entries and lengthscale derivatives built from the outputs of the reference's own code.

The reference's ProductKernel (kernels/kernel.py:634-690) multiplies the dense matrices of its factors.  Its module imports
linear_operator, so it cannot be executed standalone; the two covariance functions its RBF / Matern factors call can
(gpytorch/functions/rbf_covariance.py, matern_covariance.py, loaded by file path as make_golden.py does, with the bodies of
sq_dist / dist from kernels/kernel.py:26-60).  For a few products this script stores
    K     = prod_f s_f k_f(x1[:, dims_f], x2[:, dims_f])                       (the factors' forward outputs multiplied)
    dK_f  = (prod_{g != f} s_g k_g) s_f dk_f/dl_f                               (each factor's backward with grad_output = 1)
in fp64.  Outputs: tests/golden/product_golden.npz (committed).  Re-run:  python tests/golden/make_golden_product.py
"""
import ast
import importlib.util
import os
import sys

import numpy as np
import torch

REF = os.environ.get("GP_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
NU = {"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]   # tests/ and the repository root
from product_oracle import GOLDEN_CASES as CASES  # noqa: E402


def load_by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def extract_functions(path, names):
    tree = ast.parse(open(path).read())
    ns = {"torch": torch}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def main():
    sq_dist, dist = extract_functions(f"{REF}/gpytorch/kernels/kernel.py", ["sq_dist", "dist"])
    RBF = load_by_path("ref_rbf_cov", f"{REF}/gpytorch/functions/rbf_covariance.py").RBFCovariance
    MAT = load_by_path("ref_mat_cov", f"{REF}/gpytorch/functions/matern_covariance.py").MaternCovariance
    out = {}
    for tag, (n1, n2, d, factors) in CASES.items():
        g = torch.Generator().manual_seed(977 + n1 + d)
        x1 = torch.rand(n1, d, generator=g, dtype=torch.float64)
        x2 = torch.rand(n2, d, generator=g, dtype=torch.float64) if n2 else None
        same = x2 is None
        ks, dks = [], []
        for kind, dims, ls, os_ in factors:
            a = x1[:, dims]
            b = a if same else x2[:, dims]
            l = torch.tensor([[ls]], dtype=torch.float64, requires_grad=True)
            if kind == "rbf":
                k = RBF.apply(a, b, l, lambda u, v: sq_dist(u, v, x1_eq_x2=same))
            else:
                k = MAT.apply(a, b, l, NU[kind], lambda u, v: dist(u, v, x1_eq_x2=same))
            # the functions' backward returns grad_output * dk/dl elementwise: grad_output = 1 reads dk/dl out
            dk = k.grad_fn.apply(torch.ones_like(k))[2]
            ks.append(os_ * k.detach())
            dks.append(os_ * dk.detach())
        K = torch.ones_like(ks[0])
        for k in ks:
            K = K * k
        out[f"{tag}_x1"] = x1.numpy()
        if not same:
            out[f"{tag}_x2"] = x2.numpy()
        out[f"{tag}_K"] = K.numpy()
        for f in range(len(factors)):
            dK = dks[f].clone()
            for h in range(len(factors)):
                if h != f:
                    dK = dK * ks[h]
            out[f"{tag}_dK{f}"] = dK.numpy()
    path = os.path.join(HERE, "product_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;", len(out), "arrays")


if __name__ == "__main__":
    sys.exit(main())
