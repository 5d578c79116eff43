#!/usr/bin/env python
"""ski_predict_bench.py -- KISS-GP prediction at C5: the grid path (settings.ski_grid_prediction) against the joint path, one JSON file.

    python tools/ski_predict_bench.py --out ski_predict_bench.json [--ms 10000,100000,1000000] [--joint-ms 10000] [--reps 3]

C5 training set: N = 10^6, d = 3, X ~ U[0,1]^{N x d}, ScaleKernel(GridInterpolationKernel(RBFKernel(), 100, grid_bounds [0, 1]^3)),
lengthscale 0.2, outputscale 1, GaussianLikelihood noise 0.1, LOVE rank J = 100 (max_root_decomposition_size).  alpha and R are
the model's own (one solve and one Lanczos run before any timing; they are shared by both paths).  Timed with CUDA events, best
of --reps (an L2 flush before each):
  * the grid mean cache c = s K_uu W^T alpha and the grid LOVE cache C = s K_uu W^T R (given alpha, R);
  * per test-set size m: the test plan (interpolation + tile sort of the test points), the mean W* c (gp_ski_interp_matmul,
    t = 1), U = W* C (t = J) with its achieved bytes/s against the M t cache read plus the m t output, the LOVE variance
    diag(K**) - |U_i|^2 and 16 CIQ samples of likelihood(posterior), then peak device memory;
  * end to end with warm caches, alternating in the same run: model(x*) + .variance with the flag on (fast_pred_var) and the
    joint path (flag off) at the sizes of --joint-ms.
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gpytorch_b200 as gp  # noqa: E402
from gpytorch_b200 import settings  # noqa: E402
from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator  # noqa: E402
from tools.sample_bench import _gpu_info, _timed  # noqa: E402

N, D, G, LS, NOISE, J = 1_000_000, 3, 100, 0.2, 0.1, 100


def _model(dev):
    gen = torch.Generator().manual_seed(0)
    x = torch.rand(N, D, generator=gen).to(dev)
    y = torch.sin(3 * x.sum(-1)) + 0.1 * torch.randn(N, generator=gen).to(dev)
    lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ZeroMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), grid_size=G, num_dims=D,
                                                                                       grid_bounds=[(0.0, 1.0)] * D))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    lik = lik.to(dev)
    model.covar_module.base_kernel.base_kernel.lengthscale = LS
    model.covar_module.outputscale = 1.0
    lik.noise = NOISE
    model.eval(); lik.eval()
    return model, lik


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="ski_predict_bench.json")
    ap.add_argument("--ms", default="10000,100000,1000000")
    ap.add_argument("--joint-ms", default="10000")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    result = {"gpu": _gpu_info(), "workload": "c5 prediction", "N": N, "grid": [G] * D, "J": J, "runs": [], "end_to_end": []}
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    model, lik = _model(dev)
    gen = torch.Generator().manual_seed(1)
    M = G ** D
    with torch.no_grad(), settings.probe_seed(0), settings.max_root_decomposition_size(J):
        # alpha, R and both grid caches, once (a prediction at a few points)
        with settings.ski_grid_prediction(True), settings.fast_pred_var(True):
            model(torch.rand(16, D, generator=gen).to(dev)).variance
        alpha, R = model._mean_cache, model._covar_cache
        result["J_actual"] = int(R.size(-1))
        train_op = model.forward(model.train_inputs[0]).lazy_covariance_matrix
        _, result["ms_grid_mean_cache"], _ = _timed(lambda: train_op.grid_matmul(alpha), flush, a.reps)
        _, result["ms_grid_love_cache"], _ = _timed(lambda: train_op.grid_matmul(R), flush, a.reps)
        c, Cg = model._grid_mean_cache, model._grid_covar_cache
        print(json.dumps({k: v for k, v in result.items() if k.startswith("ms_")}), flush=True)
        for m in (int(v) for v in a.ms.split(",")):
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            xt = torch.rand(m, D, generator=gen).to(dev)
            res = {"m": m}
            test_op = model.forward(xt).lazy_covariance_matrix

            def test_plan():
                test_op.x1.add_(0.0)          # a new version of the same points: the cached plan re-interpolates and re-sorts them
                test_op._plan = None
                return test_op.plan()

            _, res["ms_test_plan"], _ = _timed(test_plan, flush, a.reps)
            _, res["ms_mean"], _ = _timed(lambda: test_op.interp_matmul(c), flush, a.reps)
            U, ms_u, _ = _timed(lambda: test_op.interp_matmul(Cg), flush, a.reps)
            res["ms_U"] = ms_u
            t = Cg.size(-1)
            res["interp_U_bytes"] = 4.0 * (M * t + m * t)
            res["interp_U_GBps"] = res["interp_U_bytes"] / (ms_u * 1e-3) / 1e9
            res["interp_mean_GBps"] = 4.0 * (M + m) / (res["ms_mean"] * 1e-3) / 1e9
            post_cov = LowRankUpdatedKernelLinearOperator.on_ski(test_op, U)
            _, res["ms_variance"], _ = _timed(lambda: post_cov.diagonal(), flush, a.reps)
            post = gp.distributions.MultivariateNormal(torch.zeros(m, device=dev), post_cov)
            with settings.ciq_samples(True):
                torch.manual_seed(0)
                _, res["ms_ciq_16_samples"], _ = _timed(lambda: lik(post).rsample(torch.Size([16])), flush, 1)
            res["peak_mem_gb"] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
            result["runs"].append(res)
            print(json.dumps(res), flush=True)
            del U, post_cov, post, test_op
        # end to end, warm caches, the two paths alternated
        for m in (int(v) for v in a.joint_ms.split(",")):
            xt = torch.rand(m, D, generator=gen).to(dev)
            e2e = {"m": m, "ms_grid": [], "ms_joint": []}
            with settings.fast_pred_var(True):
                for _ in range(a.reps):
                    for key, on in (("ms_grid", True), ("ms_joint", False)):
                        with settings.ski_grid_prediction(on):
                            torch.cuda.reset_peak_memory_stats(dev)
                            out, ms, _ = _timed(lambda: (lambda p: (p.mean, p.variance))(model(xt)), flush, 1)
                            e2e[key].append(ms)
                            e2e[key.replace("ms_", "peak_mem_gb_")] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
                            e2e[key.replace("ms_", "mean_")] = out[0]
                            e2e[key.replace("ms_", "var_")] = out[1]
            e2e["mean_rel_diff"] = float((e2e.pop("mean_grid") - e2e["mean_joint"]).norm() / e2e.pop("mean_joint").norm())
            e2e["var_max_abs_diff"] = float((e2e.pop("var_grid") - e2e.pop("var_joint")).abs().max())
            result["end_to_end"].append(e2e)
            print(json.dumps(e2e), flush=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
