#!/usr/bin/env python
"""input_grad_bench.py -- test-input gradients of an exact-GP posterior (gp_kmv_input_grad / gp_kdense_input_grad, csrc/xgrad.cu),
one JSON file.

    python tools/input_grad_bench.py --out input_grad_bench.json [--reps 3] [--sizes 1,64,1024,16384]

Training set: the C2 shape, N = 50 000, d = 10, RBF, lengthscale 1, outputscale 1, noise 0.1, X ~ U[0,1]^{N x d}.  The mean and
LOVE caches (J = 100 Lanczos steps) are built once, then for each m (X* ~ U[0,1]^{m x d}; CUDA events, best of --reps, the L2
evicted by a 192 MiB memset before every timed call):
  * fwd_ms / bwd_ms: mean + variance under settings.fast_pred_var, forward and the backward of mean.sum() + variance.sum() to X*;
  * prim_ms_t{1,100}: one gp_kmv_input_grad call for DX* of sum(G * (K*x V)) with t = 1 and t = 100 (packing, kernel and split
    reduction), and kernel_ms_t{1,100} the xgrad_kernel time alone from torch.profiler; fma_tflops counts 2 (t_chunk + 3 DP) flops
    per pair and chunk over the kernel time (t_chunk = 8 or 32 padded columns, DP = 12), next to the data-sheet 67 TFLOP/s;
  * torch_fwd_ms / torch_bwd_ms: the same mean + variance written as dense fp32 torch ops (K*x materialised) with torch autograd,
    where it fits in memory.
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

import gpytorch_b200 as gp  # noqa: E402
from gpytorch_b200 import settings  # noqa: E402
from gpytorch_b200.engine import Plan  # noqa: E402

N, D, LS, NOISE, J = 50_000, 10, 1.0, 0.1, 100


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
    return out, min(ms)


def _kernel_ms(fn, reps):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = sum(e.device_time_total for e in prof.key_averages() if "xgrad_kernel" in e.key)
    return tot / 1000.0 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="input_grad_bench.json")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1,64,1024,16384")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("input_grad_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    x = torch.rand(N, D, generator=g).to(dev)
    y = (torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(N, generator=g).to(dev)).contiguous()
    lik = gp.likelihoods.GaussianLikelihood().to(dev)

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    model.covar_module.base_kernel.lengthscale = LS
    model.covar_module.outputscale = 1.0
    lik.noise = NOISE
    model.eval(); lik.eval()
    flush = torch.empty(192 * 2**20 // 4, device=dev)
    with settings.fast_pred_var(), settings.probe_seed(0), torch.no_grad():
        model(torch.rand(1, D, device=dev))                                  # mean and LOVE caches
    alpha, R = model._mean_cache, model._covar_cache
    res = {"gpu": _gpu_info(), "N": N, "d": D, "J": int(R.size(1)), "sizes": []}
    for m in [int(v) for v in a.sizes.split(",")]:
        xs = torch.rand(m, D, generator=g).to(dev)
        row = {"m": m}

        def fwd():
            xg = xs.clone().requires_grad_(True)
            with settings.fast_pred_var():
                post = model(xg)
                return xg, post.mean.sum() + post.variance.sum()

        fwd()
        _, row["fwd_ms"] = _timed(fwd, flush, a.reps)
        bms = []
        for _ in range(a.reps):
            xg, f = fwd()
            torch.cuda.synchronize()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f.backward()
            e1.record()
            e1.synchronize()
            bms.append(e0.elapsed_time(e1))
        row["bwd_ms"] = min(bms)
        p = Plan(xs, x).set_hypers("rbf", LS, 1.0, 0.0)
        for t in (1, 100):
            G = torch.randn(m, t, device=dev)
            V = torch.randn(N, t, device=dev)

            def prim():
                return p.kmv_input_grad(G, V, True, False)

            prim()
            _, row[f"prim_ms_t{t}"] = _timed(prim, flush, a.reps)
            kms = _kernel_ms(prim, a.reps)
            tw = 8 if t <= 8 else 32
            chunks = -(-t // tw)
            flops = 2.0 * m * N * chunks * (tw + 3 * 12)
            row[f"kernel_ms_t{t}"] = kms
            row[f"fma_tflops_t{t}"] = flops / (kms * 1e-3) / 1e12 if kms > 0 else None
        p.close()
        # dense fp32 torch autograd baseline of the same mean + variance
        try:
            def tfwd():
                xg = xs.clone().requires_grad_(True)
                K = torch.exp(-0.5 * torch.cdist(xg, x).square() / LS**2)
                return xg, (K @ alpha).sum() + (1.0 - (K @ R).square().sum(-1)).sum()

            tfwd()
            _, row["torch_fwd_ms"] = _timed(tfwd, flush, a.reps)
            tb = []
            for _ in range(a.reps):
                xg, f = tfwd()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f.backward()
                e1.record()
                e1.synchronize()
                tb.append(e0.elapsed_time(e1))
            row["torch_bwd_ms"] = min(tb)
        except torch.cuda.OutOfMemoryError:
            row["torch_fwd_ms"] = row["torch_bwd_ms"] = None
        torch.cuda.empty_cache()
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)
    res["peak_fp32_tflops_datasheet"] = 67.0
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
