#!/usr/bin/env python
"""posterior_sample_bench.py -- sampling an exact-GP posterior at large test sets through the lazy LOVE covariance
(settings.fast_pred_samples, operators.LowRankUpdatedKernelLinearOperator), one JSON file.

    python tools/posterior_sample_bench.py --out posterior_bench.json [--reps 3] [--sizes 10000,50000,200000] [--dense 10000,50000]

Training set: the C2 shape, N = 50 000, d = 10, RBF, lengthscale 1, outputscale 1, noise 0.1, X ~ U[0,1]^{N x d}.  Test sets
X* ~ U[0,1]^{m x d}.  For each m (CUDA events, best of --reps, the L2 evicted by a 192 MiB memset before every timed call):
  * love_cache_ms: the LOVE cache, R from 100 Lanczos steps on K_hat (root_inv_decomposition) plus U = K*x R (the product on the
    cross-covariance plan), as ExactGP.__call__ builds it;
  * variance_ms: diag(K**) - sum_j U_ij^2 (gp_kdiag on the low-rank plan);
  * ciq_ms_16: 16 samples of the observed posterior K** - U U^T + sigma^2 I by CIQ (Q = 15, msMINRES tolerance 1e-4), the
    quadrature interval included; its iterations, ms per iteration and kernel launches per iteration (slope between fixed 10- and
    30-iteration runs), next to one K.V launch on the test plan (gp_time_kmv_kernel) and to the low-rank correction's share
    (the same slope with U cleared);
  * peak_mib: torch's peak allocation plus the engine's own device buffers (free-memory delta) during the lazy run;
  * for the m in --dense: today's dense path (fast_pred_var): the m x m covariance K** - U U^T, its variance, and 16 samples by
    a psd-safe Cholesky of covariance + sigma^2 I.
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
                                     LowRankUpdatedKernelLinearOperator)
from gpytorch_b200.sampling import contour_quadrature, psd_safe_cholesky  # noqa: E402

N, D, LS, NOISE = 50_000, 10, 1.0, 0.1


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1]), "max_sm_clock_mhz": float(q[2])}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "note": f"nvidia-smi: {e}"}


def _timed(fn, flush, reps):
    ms, out = [], None
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return out, min(ms), ms


def run(m, dense, reps, dev, flush, khat, x, gen):
    ls, os_ = torch.tensor(LS, device=dev), torch.tensor(1.0, device=dev)
    xs = torch.rand(m, D, generator=gen).to(dev)
    k_star = KernelLinearOperator(xs, x, "rbf", ls, os_)
    init = torch.randn(N, generator=gen).to(dev)

    def cache():
        return k_star.matmul(khat.root_inv_decomposition(init))

    cache()                                                                   # warm-up
    U, cache_ms, _ = _timed(cache, flush, reps)
    k_ss = KernelLinearOperator(xs, xs, "rbf", ls, os_)
    res = {"m": m, "J": int(U.size(1)), "love_cache_ms": cache_ms}
    torch.cuda.synchronize()
    free0, reserved0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    lazy = LowRankUpdatedKernelLinearOperator(k_ss, U)
    obs = lazy + ConstantDiagLinearOperator(torch.tensor(NOISE, device=dev), m)
    _, res["variance_ms"], _ = _timed(lazy.diagonal, flush, reps)
    xi = torch.randn(m, 16, generator=gen).to(dev)
    with settings.ciq_samples(True):
        obs._ciq_samples(xi)                                                  # warm-up
        (_, infos), res["ciq_ms_16"], res["ciq_ms_all_reps"] = _timed(lambda: obs._ciq_samples(xi), flush, reps)
    mm, MM, _ = obs.last_ciq
    res.update({"ciq_iters": infos[0].iters, "ciq_interval": [mm, MM],
                "ciq_max_resid": max(max(r) for r in infos[0].residual_norms)})
    torch.cuda.synchronize()
    res["peak_mib"] = ((torch.cuda.max_memory_allocated() - base)
                       + max(0, free0 - torch.cuda.mem_get_info()[0] - (torch.cuda.memory_reserved() - reserved0))) / 2**20
    plan = obs._sampling_plan()
    tau, w = contour_quadrature(mm, MM, 15)

    def slope():
        per = {}
        for k in (10, 30):
            l0 = plan.launches()
            _, t_k, _ = _timed(lambda: plan.ciq_sqrt_matmul(xi, tau, w, 0.0, k, warn=False), flush, reps)
            per[k] = (t_k, plan.launches() - l0)
        return (per[30][0] - per[10][0]) / 20, (per[30][1] - per[10][1]) / (20 * reps)

    res["ms_per_iter"], res["launches_per_iter"] = slope()
    res["ms_kmv_launch_test_plan"] = plan.time_kmv_kernel(xi, warmup=2, reps=5)
    plan.set_lowrank(None)                                                    # the same loop on K** + sigma^2 I alone
    res["ms_per_iter_without_correction"], res["launches_per_iter_without_correction"] = slope()
    del lazy, obs
    if m in dense:
        k_ss_d = KernelLinearOperator(xs, xs, "rbf", ls, os_)

        def dense_path():
            covar = k_ss_d.to_dense() - U @ U.T                               # ExactGP's fast_pred_var branch
            var = covar.diagonal().clone()
            covar.diagonal().add_(NOISE)
            L = psd_safe_cholesky(covar)
            del covar
            return var, L @ xi

        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        dense_path()
        _, res["dense_ms_covar_variance_16_samples"], _ = _timed(dense_path, flush, reps)
        res["dense_peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2**20
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="posterior_bench.json")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="10000,50000,200000")
    ap.add_argument("--dense", default="10000,50000")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(0)
    x = torch.rand(N, D, generator=gen).to(dev)
    khat = AddedDiagLinearOperator(KernelLinearOperator(x, None, "rbf", torch.tensor(LS, device=dev), torch.tensor(1.0, device=dev)),
                                   ConstantDiagLinearOperator(torch.tensor(NOISE, device=dev), N))
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    dense = [int(v) for v in a.dense.split(",") if v]
    result = {"gpu": _gpu_info(), "train": {"n": N, "d": D, "kind": "rbf", "lengthscale": LS, "noise": NOISE},
              "l2_policy": "192 MiB memset before every timed call, outside the timed region", "sizes": {}}
    for m in [int(v) for v in a.sizes.split(",")]:
        result["sizes"][str(m)] = run(m, dense, a.reps, dev, flush, khat, x, gen)
        print(m, json.dumps(result["sizes"][str(m)]), flush=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
