"""Golden data for the additive operator: the reference's own sum_interaction_terms (utils/sum_interaction_terms.py, Newton-Girard)
on batches of univariate RBF / Matern matrices from the reference's covariance functions, in fp64.

    GP_REFERENCE=<reference checkout> python tests/golden/make_golden_additive.py    # writes tests/golden/additive_golden.npz

The reference module imports linear_operator only for `to_dense` and a type name; a stub module stands in for it.  The
covariances come from the reference's RBFCovariance / MaternCovariance functions, called directly in fp64 (no kernel modules).
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np
import torch


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


REF = os.environ.get("GP_REFERENCE", "/root/reference")


def main(ref=REF):
    stub = types.ModuleType("linear_operator")
    stub.LinearOperator = type("LinearOperator", (), {})
    stub.to_dense = lambda x: x
    sys.modules.setdefault("linear_operator", stub)
    sit = _load(os.path.join(ref, "gpytorch", "utils", "sum_interaction_terms.py"), "ref_sum_interaction_terms").sum_interaction_terms
    rbf = _load(os.path.join(ref, "gpytorch", "functions", "rbf_covariance.py"), "ref_rbf_covariance").RBFCovariance
    mat = _load(os.path.join(ref, "gpytorch", "functions", "matern_covariance.py"), "ref_matern_covariance").MaternCovariance

    def sq_dist(a, b):
        return (a.unsqueeze(-2) - b.unsqueeze(-3)).pow(2).sum(-1)

    def dist(a, b):
        return sq_dist(a, b).clamp_min(0).sqrt()

    g = torch.Generator().manual_seed(20261017)
    out = {}
    cases = [("rbf", 3, 5, 1), ("rbf", 4, 7, 2), ("matern12", 5, 6, 3), ("matern32", 3, 5, 2), ("matern52", 6, 4, 4),
             ("rbf", 7, 5, 7), ("matern52", 2, 9, 1)]
    for ci, (kind, D, n, M) in enumerate(cases):
        X1 = torch.rand(n, D, generator=g, dtype=torch.float64) * 4 - 2
        X2 = torch.rand(n + 2, D, generator=g, dtype=torch.float64) * 4 - 2
        ls = torch.rand(D, generator=g, dtype=torch.float64) * 1.5 + 0.3
        sc = torch.rand(D, generator=g, dtype=torch.float64) * 1.5 + 0.2
        covs = []
        for i in range(D):
            a = X1[:, i:i + 1]
            b = X2[:, i:i + 1]
            l = ls[i].reshape(1, 1)
            if kind == "rbf":
                k = rbf.apply(a, b, l, lambda x1, x2: sq_dist(x1, x2))
            else:
                nu = {"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}[kind]
                k = mat.apply(a, b, l, nu, lambda x1, x2: dist(x1, x2))
            covs.append(sc[i] * k)
        K = sit(torch.stack(covs), max_degree=M, dim=-3)
        for key, v in (("X1", X1), ("X2", X2), ("ls", ls), ("sc", sc), ("K", K)):
            out[f"c{ci}_{key}"] = v.detach().numpy()
        out[f"c{ci}_meta"] = np.array([["rbf", "matern12", "matern32", "matern52"].index(kind), D, M])
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "additive_golden.npz"), **out)


if __name__ == "__main__":
    main()
