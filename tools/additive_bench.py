"""Timing of the additive operator's K.V (csrc/additive.cu) against the plain fused kernel and the 4-term kernel sum.

    python tools/additive_bench.py [--n 50000] [--t 11] [--reps 20] [--rounds 5] [--out FILE]

One K.V launch at N points with t columns, timed with CUDA events over `reps` launches (gp_time_kmv_kernel); every case runs once
per round, rounds alternate the cases, and the median over the rounds is reported.  Cases: D in {4, 10, 32} x M in {1, 2, 3}
(RBF components), the plain tensor-core RBF kernel at d = 10, and the 4-term kernel sum of one-dimensional RBF terms at D = 4 on
the same data (one launch per term).  Then one MLL forward + backward at D = 10 for M = 1 and M = 2 through the public API.
Pairs/s is N^2 per launch time; ex2/s counts the D exponentials of every pair.  The card's name and power limit are read in the
same process and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001 -- reported, not fatal
        power = f"unknown ({e})"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--t", type=int, default=11)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("additive_bench needs a GPU")
    from gpytorch_b200.engine import Plan
    from gpytorch_b200.operators import KernelLinearOperator, SumKernelLinearOperator

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    n, t = a.n, a.t
    X = torch.rand(n, 32, device=dev, generator=g)
    V = torch.randn(n, t, device=dev, generator=g)
    cases = {}
    for D in (4, 10, 32):
        for M in (1, 2, 3):
            p = Plan(X[:, :D].contiguous()).set_additive(M, [1.0] * D).set_hypers("rbf", [0.3] * D, 1.0, 0.0)
            cases[f"additive D={D} M={M}"] = (p, D)
    cases["plain RBF d=10 (tensor cores)"] = (Plan(X[:, :10].contiguous()).set_hypers("rbf", [0.3] * 10, 1.0, 0.0), 0)
    cols = [X[:, i:i + 1].contiguous() for i in range(4)]
    terms = [KernelLinearOperator(c, None, "rbf", torch.tensor(0.3, device=dev), torch.tensor(1.0, device=dev)) for c in cols]
    cases["4-term kernel sum D=4"] = (SumKernelLinearOperator(terms).plan(0.0), 4)
    times = {k: [] for k in cases}
    for k, (p, _) in cases.items():
        p.time_kmv_kernel(V, warmup=3, reps=3)
    for _ in range(a.rounds):
        for k, (p, _) in cases.items():
            times[k].append(cases[k][0].time_kmv_kernel(V, warmup=2, reps=a.reps))
    name, power = card()
    res = {"card": name, "power_limit": power, "n": n, "t": t, "reps": a.reps, "rounds": a.rounds, "kmv": {}}
    for k, (p, D) in cases.items():
        ms = statistics.median(times[k])
        pairs = n * n / (ms * 1e-3)
        res["kmv"][k] = {"ms": ms, "spread_ms": [min(times[k]), max(times[k])], "pairs_per_s": pairs,
                         "ex2_per_s": pairs * D if D else None, "backend": p.info()["backend"]}
    add4, sum4 = res["kmv"]["additive D=4 M=1"]["ms"], res["kmv"]["4-term kernel sum D=4"]["ms"]
    res["additive_D4_M1_over_sum4"] = add4 / sum4

    # one MLL forward + backward at D = 10 through the public API
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, likelihoods, means, models, settings
    from gpytorch_b200.utils import sum_interaction_terms

    D = 10
    Xt = X[:, :D].contiguous()
    y = (torch.sin(6 * Xt[:, 0]) + Xt[:, 1] * Xt[:, 2]).contiguous()
    res["mll"] = {}
    for M in (1, 2):
        class AGP(models.ExactGP):
            def __init__(self):
                super().__init__(Xt, y, likelihoods.GaussianLikelihood())
                self.mean_module = means.ConstantMean()
                self.covar_module = kernels.ScaleKernel(kernels.RBFKernel(batch_shape=torch.Size([D]), ard_num_dims=1))

            def forward(self, x):
                b = self.covar_module(x.mT.unsqueeze(-1))
                return gp.distributions.MultivariateNormal(self.mean_module(x), b.sum(dim=-3) if M == 1 else
                                                           sum_interaction_terms(b, max_degree=M))

        model = AGP().to(dev)
        model.train()
        mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
        step_times = []
        with settings.max_cholesky_size(0):
            for it in range(4):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                loss = -mll(model(Xt), y)
                loss.backward()
                torch.cuda.synchronize()
                if it > 0:
                    step_times.append(time.perf_counter() - t0)
                model.zero_grad()
        res["mll"][f"D={D} M={M}"] = {"s_per_step": statistics.median(step_times), "steps": step_times, "loss": loss.item()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
