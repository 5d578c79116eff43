"""Polynomial kernel timings on one GPU: one K.V launch of a polynomial plan (powers 1, 2, 4) against an RBF launch of the same
width (the same tensor-core pipeline; the polynomial epilogue is FMA-pipe only, RBF's one ex2 per entry), the gradient call (two
tensor-core passes: k and dk/dc), and one MLL forward + backward of ScaleKernel(PolynomialKernel(2)) + ScaleKernel(RBFKernel())
through the API.

    python tools/poly_bench.py [--n 50000] [--t 16] [--dims 1 4 10] [--powers 1 2 4] [--rounds 5]

Every K.V time is the median over alternating rounds of gp_time_kmv_kernel (CUDA events around the kernel alone).  The card's
name, power limit and maximum SM clock are printed in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception:   # nvidia-smi missing: the name from torch, the rest unknown
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--t", type=int, default=16)
    ap.add_argument("--dims", type=int, nargs="+", default=[1, 4, 10])
    ap.add_argument("--powers", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("poly_bench needs a GPU")
    from gpytorch_b200 import kernels
    from gpytorch_b200.engine import Plan

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    res = {"card": card(), "n": a.n, "t": a.t, "kmv_ms": {}, "grad_ms": {}}
    V = torch.randn(a.n, a.t, generator=g).to(dev)
    for d in a.dims:
        x = ((torch.rand(a.n, d, generator=g) * 2 - 1) / d ** 0.5).to(dev)
        polys = {p: Plan(x).set_hypers_poly(p, 0.5, 1.0, 0.1) for p in a.powers}
        rb = Plan(x).set_hypers("rbf", [0.8], 1.0, 0.1)
        info = polys[a.powers[0]].info()
        assert info["backend"] == "tcgen05", info
        times = {f"poly{p}": [] for p in a.powers}
        times["rbf"] = []
        for _ in range(a.rounds):   # alternate the plans within every round
            for p, pl in polys.items():
                times[f"poly{p}"].append(pl.time_kmv_kernel(V, 3, a.reps))
            times["rbf"].append(rb.time_kmv_kernel(V, 3, a.reps))
        res["kmv_ms"][d] = {k: statistics.median(v) for k, v in times.items()}
        res["kmv_ms"][d]["kpad"] = info["kpad"]
        L = torch.randn(a.n, a.t, generator=g).to(dev)
        pg = polys[a.powers[min(1, len(a.powers) - 1)]]
        pg.bilinear_grad(L, V)
        torch.cuda.synchronize()
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            pg.bilinear_grad(L, V)   # ends in a device synchronise (the gradients are read back)
            ts.append((time.perf_counter() - t0) * 1e3)
        res["grad_ms"][d] = statistics.median(ts)
        for pl in (*polys.values(), rb):
            pl.close()
    # one MLL forward + backward through the API: a polynomial trend plus a smooth residual, exact GP on the CG path, d = 1
    import gpytorch_b200 as gp
    from gpytorch_b200 import likelihoods, means, models, settings

    x = torch.linspace(-1, 1, a.n, device=dev)
    y = 0.5 * x ** 2 + 0.2 * torch.sin(20.0 * x) + 0.1 * torch.randn(a.n, device=dev)

    class M(models.ExactGP):
        def __init__(self):
            super().__init__(x, y, likelihoods.GaussianLikelihood())
            self.mean_module = means.ConstantMean()
            self.covar_module = kernels.ScaleKernel(kernels.PolynomialKernel(2)) + kernels.ScaleKernel(kernels.RBFKernel())

        def forward(self, z):
            return gp.distributions.MultivariateNormal(self.mean_module(z), self.covar_module(z))

    model = M().to(dev)
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    model.train()
    ts = []
    with settings.max_cholesky_size(0):
        for i in range(4):
            model.zero_grad()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss = -mll(model(x), y)
            loss.backward()
            torch.cuda.synchronize()
            if i:
                ts.append((time.perf_counter() - t0) * 1e3)
    res["mll_fwd_bwd_ms"] = statistics.median(ts)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
