#!/usr/bin/env python
"""ski_solve_bench.py -- the solve side of the SKI preconditioner (settings.ski_preconditioner) at C5, one JSON file.

    python tools/ski_solve_bench.py --out ski_solve_bench.json [--ranks 0,15,100] [--reps 2]

C5: N = 10^6, d = 3, X ~ U[0,1]^{N x d}, RBF lengthscale 0.2, outputscale 1, noise 0.1, SKI grid of 100^3 nodes over [0, 1]^3.
For each preconditioner rank k (0: none), timed with CUDA events:
  * pivoted Cholesky + gp_precond_build (k > 0);
  * the prediction mean-cache solve K_hat^-1 y (one column, eval_cg_tolerance 0.01 and 1e-4): CG iterations and ms;
  * one MLL evaluation through the public API (inv_quad_logdet with the log-det, 10 probes, cg_tolerance 1): ms and CG iterations;
  * peak device memory of the run.
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

from gpytorch_b200 import operators, settings  # noqa: E402
from tools.sample_bench import WORKLOADS, _gpu_info, _operator, _timed  # noqa: E402


def run(k, reps, dev):
    cfg = WORKLOADS["c5"]
    gen = torch.Generator().manual_seed(0)
    op = _operator(cfg, dev, gen)
    y = torch.sin(3 * op.kernel_op.x1.sum(-1))[:, None].contiguous()
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    torch.cuda.reset_peak_memory_stats(dev)
    res = {"k": k}
    with settings.ski_preconditioner(k > 0), settings.max_preconditioner_size(k):
        if k > 0:
            plan = op._plan()

            def build():
                lt, _, _ = plan.pivoted_cholesky(k, settings.preconditioner_tolerance.value())
                return lt, plan.precond_build(lt)

            build()
            (lt, _), res["ms_pivchol_plus_precond_build"], _ = _timed(build, flush, reps)
            res["precond_rank"] = int(lt.size(0))
        w = op._preconditioner()[0]
        for tol in (0.01, 1e-4):
            with settings._use_eval_tolerance(True), settings.eval_cg_tolerance(tol):
                (_, _, it), ms, _ = _timed(lambda: operators._run_cg(op, y, 0, w), flush, reps)
            res[f"mean_cache_tol{tol:g}"] = {"cg_iters": it, "ms": ms}
        with settings.probe_seed(0), torch.no_grad():
            _, ms, _ = _timed(lambda: op.inv_quad_logdet(y, logdet=True), flush, reps)
        res["mll_api"] = {"ms": ms, "cg_iters": op.last_cg_iters}
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="ski_solve_bench.json")
    ap.add_argument("--ranks", default="0,15,100")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    result = {"gpu": _gpu_info(), "workload": "c5", "runs": []}
    for k in (int(v) for v in a.ranks.split(",")):
        r = run(k, a.reps, dev)
        result["runs"].append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
