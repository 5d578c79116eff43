#!/usr/bin/env python
"""sample_bench.py -- CIQ sampling (gp_ciq_sqrt_matmul, csrc/minres.cu) at three workloads, one JSON file.

    python tools/sample_bench.py --out sample_bench.json [--reps 3] [--skip c3,c5] [--precond-rank 0,100]

Workloads (Q = 15 quadrature points, msMINRES tolerance 1e-4, 16 samples, X ~ U[0,1]^{N x d}, outputscale 1, noise 0.1):
  c2  N = 50 000,  d = 10, RBF,        lengthscale 1
  c3  N = 200 000, d = 20, Matern-5/2, lengthscale 2  (the C3 shape on one GPU)
  c5  N = 10^6,    d = 3,  RBF on a SKI grid of 100^3 nodes, lengthscale 0.2
For each: ms for 16 samples (CUDA events; the L2 is evicted by a 192 MiB memset before every timed call, as bench.py does,
outside the timed region), msMINRES iterations, the quadrature interval (m, M), ms per iteration from the slope between
fixed 10- and 30-iteration runs next to the fused K.V launch alone (gp_time_kmv_kernel), and kernel launches per iteration from
the same two runs.  At c2 it also times dense fp32 Cholesky sampling of the same xi and reports the largest difference.
--precond-rank takes a comma-separated list of ranks k (default 0: the unpreconditioned run only).  For k > 0 the run uses the
split preconditioner of settings.ciq_preconditioner (gp_ciq_sqrt_matmul_precond) and also reports k, the build time (pivoted
Cholesky + gp_ciq_precond_build, CUDA events) and the trace interval [m, M]; c5 (SKI) runs with settings.ski_preconditioner on.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpytorch_b200 import settings  # noqa: E402
from gpytorch_b200.operators import (AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator,  # noqa: E402
                                     SKIKernelLinearOperator)
from gpytorch_b200.sampling import contour_quadrature  # noqa: E402

WORKLOADS = {
    "c2": dict(n=50_000, d=10, kind="rbf", ls=1.0),
    "c3": dict(n=200_000, d=20, kind="matern52", ls=2.0),
    "c5": dict(n=1_000_000, d=3, kind="rbf", ls=0.2, grid=100),
}


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1])}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "note": f"nvidia-smi: {e}"}


def _operator(cfg, dev, gen):
    n, d = cfg["n"], cfg["d"]
    x = torch.rand(n, d, generator=gen).to(dev)
    ls = torch.tensor(cfg["ls"], device=dev)
    os_ = torch.tensor(1.0, device=dev)
    if "grid" in cfg:
        g = cfg["grid"]
        lo, step = -1.0 / (g - 2), (1.0 + 2.0 / (g - 2)) / (g - 1)   # bounds [0, 1] extended by one cell, as create_grid does
        k = SKIKernelLinearOperator(x, cfg["kind"], ls, os_, [g] * d, [lo] * d, [step] * d)
    else:
        k = KernelLinearOperator(x, None, cfg["kind"], ls, os_)
    return AddedDiagLinearOperator(k, ConstantDiagLinearOperator(torch.tensor(0.1, device=dev), n))


def _timed(fn, flush, reps):
    ms = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return out, min(ms), ms


def run(name, cfg, reps, dev, rank=0):
    with settings.ski_preconditioner("grid" in cfg and rank > 0):
        return _run(name, cfg, reps, dev, rank)


def _run(name, cfg, reps, dev, rank):
    gen = torch.Generator().manual_seed(0)
    op = _operator(cfg, dev, gen)
    n, s, Q, tol = cfg["n"], 16, 15, 1e-4
    xi = torch.randn(n, s, generator=gen).to(dev)
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    plan = op._sampling_plan()
    u, extra = None, {}
    if rank == 0:
        m, M = op._ciq_bounds(plan, xi[:, 0])
    else:
        with settings.max_preconditioner_size(rank):
            pre = op._ciq_precond()
            if pre is None:
                raise RuntimeError(f"{name}: no preconditioner at rank {rank}")
            u, m, M = pre

            def build():
                lt, _, _ = plan.pivoted_cholesky(rank, settings.preconditioner_tolerance.value())
                return plan.ciq_precond_build(lt)

            build()                                                         # warm-up
            _, build_ms, _ = _timed(build, flush, reps)
        extra = {"precond_rank": int(u.size(1)), "build_ms_pivchol_plus_factor": build_ms}
    tau, w = contour_quadrature(m, M, Q)
    plan.ciq_sqrt_matmul(xi, tau, w, tol, 1000, precond_u=u)               # warm-up
    (out, info), best, all_ms = _timed(lambda: plan.ciq_sqrt_matmul(xi, tau, w, tol, 1000, precond_u=u), flush, reps)
    # the full public call, same xi: the interval estimate included (k = 0), the cached factor reused (k > 0)
    with settings.ciq_samples(True), settings.ciq_preconditioner(rank > 0), settings.max_preconditioner_size(max(rank, 1)):
        _, api_ms, _ = _timed(lambda: op._ciq_samples(xi), flush, reps)
    # per-iteration cost and launches: slope between fixed-length runs (tol = 0 never stops early)
    per = {}
    for k in (10, 30):
        l0 = plan.launches()
        _, t_k, _ = _timed(lambda: plan.ciq_sqrt_matmul(xi, tau, w, 0.0, k, warn=False, precond_u=u), flush, reps)
        per[k] = (t_k, plan.launches() - l0)
    ms_it = (per[30][0] - per[10][0]) / 20
    launches_it = (per[30][1] - per[10][1]) / (20 * reps)
    kmv_ms = plan.time_kmv_kernel(xi, warmup=2, reps=5)
    res = {"n": n, "d": cfg["d"], "kind": cfg["kind"], "samples": s, "Q": Q, "tol": tol, "ms_16_samples": best, "ms_all_reps": all_ms,
           "ms_16_samples_api_incl_bounds": api_ms, "iters": info.iters, "m": m, "M": M, "ms_per_iter": ms_it,
           "ms_kmv_launch": kmv_ms, "launches_per_iter": launches_it,
           "max_resid": max(max(r) for r in info.residual_norms), **extra}
    if "grid" in cfg:
        res["grid"] = [cfg["grid"]] * cfg["d"]
    if name == "c2" and rank == 0:
        dense = op.to_dense()
        torch.cuda.synchronize()

        def chol():
            return torch.linalg.cholesky(dense) @ xi

        ref, chol_ms, _ = _timed(chol, flush, reps)
        res["cholesky_ms_16_samples"] = chol_ms
        # L xi and K_hat^{1/2} xi are draws from the same distribution through different roots, so they are compared by their
        # norms (E |R xi|^2 = tr K_hat for every root R), not entry by entry
        res["cholesky_vs_ciq_sum_sq_rel"] = float((ref.double().pow(2).sum() - out.double().pow(2).sum()) / ref.double().pow(2).sum())
        res["max_abs_diff_vs_cholesky"] = float((out - ref).abs().max())
        res["note"] = "max_abs_diff_vs_cholesky compares two different square roots of K_hat applied to the same xi: not an error"
        del dense, ref
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="sample_bench.json")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip", default="")
    ap.add_argument("--precond-rank", default="0", help="comma-separated preconditioner ranks k (0: unpreconditioned)")
    a = ap.parse_args()
    ranks = [int(r) for r in a.precond_rank.split(",")]
    dev = torch.device("cuda:0")
    result = {"gpu": _gpu_info(), "l2_policy": "192 MiB memset before every timed call, outside the timed region", "workloads": {}}
    for name, cfg in WORKLOADS.items():
        if name in a.skip.split(","):
            continue
        for rank in ranks:
            key = name if rank == 0 else f"{name}_k{rank}"
            result["workloads"][key] = run(name, cfg, a.reps, dev, rank)
            print(key, json.dumps(result["workloads"][key]), flush=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
