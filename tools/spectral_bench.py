"""Timing of the spectral mixture operator's K.V (csrc/spectral.cu) against the plain RBF kernels, and one MLL step.

    python tools/spectral_bench.py [--n 50000] [--t 16] [--reps 10] [--rounds 5] [--out FILE]

One K.V launch at N points with t columns, timed with CUDA events over `reps` launches (gp_time_kmv_kernel); every case runs once
per round, rounds alternate the cases, and the median over the rounds is reported.  Cases: Q in {1, 4, 8, 16} x d in {1, 4} (Q d
<= 32), and the plain RBF kernel at d = 1 on the tensor cores and on the CUDA cores.  Pairs/s is N^2 per launch time; MUFU/s
counts the 2 Q d special-function operations (ex2, cos) of every pair, the floor being 132 SMs x 16 per clock x the SM clock.
Then one MLL forward + backward at Q = 4, d = 1 through the public API with a rank-100 preconditioner.  The card's name, power
limit and maximum SM clock are read in the same process and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    except Exception as e:   # noqa: BLE001 -- reported, not fatal
        power, clock = f"unknown ({e})", "unknown"
    return name, power, clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--t", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectral_bench needs a GPU")
    from gpytorch_b200.engine import Plan

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    n, t = a.n, a.t
    X = torch.rand(n, 4, device=dev, generator=g) * 100
    V = torch.randn(n, t, device=dev, generator=g)
    cases = {}
    for Q in (1, 4, 8, 16):
        for d in (1, 4):
            if Q * d > 32:
                continue
            w = [1.0 / Q] * Q
            mu = [[0.05 + 0.4 * q / Q] * d for q in range(Q)]
            v = [[0.02] * d for _ in range(Q)]
            p = Plan(X[:, :d].contiguous()).set_hypers("rbf", 1.0, 1.0, 0.0).set_spectral(w, mu, v)
            cases[f"spectral Q={Q} d={d}"] = (p, 2 * Q * d)
    cases["plain RBF d=1 (tensor cores)"] = (Plan(X[:, :1].contiguous()).set_hypers("rbf", [8.0], 1.0, 0.0), 0)
    cases["plain RBF d=1 (CUDA cores)"] = (Plan(X[:, :1].contiguous(), backend="simt").set_hypers("rbf", [8.0], 1.0, 0.0), 0)
    times = {k: [] for k in cases}
    for k, (p, _) in cases.items():
        p.time_kmv_kernel(V, warmup=2, reps=2)
    for _ in range(a.rounds):
        for k, (p, _) in cases.items():
            times[k].append(p.time_kmv_kernel(V, warmup=1, reps=a.reps))
    name, power, clock = card()
    res = {"card": name, "power_limit": power, "max_sm_clock": clock, "n": n, "t": t, "reps": a.reps, "rounds": a.rounds, "kmv": {}}
    try:
        mhz = float(clock.split()[0])
    except ValueError:
        mhz = float("nan")
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    mufu_peak = n_sm * 16 * mhz * 1e6
    for k, (p, m) in cases.items():
        ms = statistics.median(times[k])
        pairs = n * n / (ms * 1e-3)
        res["kmv"][k] = {"ms": ms, "spread_ms": [min(times[k]), max(times[k])], "pairs_per_s": pairs, "backend": p.info()["backend"]}
        if m:
            res["kmv"][k]["mufu_per_s"] = pairs * m
            res["kmv"][k]["mufu_floor_ms"] = n * n * m / mufu_peak * 1e3
    res["mufu_peak_per_s"] = mufu_peak

    # one MLL forward + backward at Q = 4, d = 1 through the public API (CG path, rank-100 preconditioner)
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, likelihoods, means, models, settings

    xs = (torch.arange(n, device=dev, dtype=torch.float32) * 0.05).contiguous()
    y = (torch.sin(2 * math.pi * 0.13 * xs) + 0.5 * torch.sin(2 * math.pi * 0.031 * xs)).contiguous()

    class SMGP(models.ExactGP):
        def __init__(self):
            super().__init__(xs, y, likelihoods.GaussianLikelihood())
            self.mean_module = means.ConstantMean()
            k = kernels.SpectralMixtureKernel(num_mixtures=4)
            k.initialize_from_data(xs[:2000].cpu(), y[:2000].cpu())
            self.covar_module = kernels.ScaleKernel(k)

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    model = SMGP().to(dev)
    model.train()
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    step_times = []
    with settings.max_cholesky_size(0), settings.max_preconditioner_size(100):
        for it in range(4):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss = -mll(model(xs), y)
            loss.backward()
            torch.cuda.synchronize()
            if it > 0:
                step_times.append(time.perf_counter() - t0)
            model.zero_grad()
    res["mll"] = {"Q=4 d=1": {"s_per_step": statistics.median(step_times), "steps": step_times, "loss": loss.item()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
