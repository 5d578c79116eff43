#!/usr/bin/env python
"""Time one deep-kernel-learning training step: network forward, MLL forward, the backward without the input gradient (the
features detached: hyper-parameters only) and the extra cost of the input backward (full backward minus that), plus the peak
device memory over 50 full training steps.  Prints the card name and power limit with the numbers (one JSON line per config).

    python tools/dkl_bench.py [--steps 50] [--reps 5] [--configs exact2,exact10,ski2,ski3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpytorch_b200 as gp  # noqa: E402
from gpytorch_b200.utils.grid import ScaleToBounds  # noqa: E402

CONFIGS = {   # name: (N, feature d, grid size or None)
    "exact2": (50_000, 2, None), "exact10": (50_000, 10, None), "ski2": (1_000_000, 2, 100), "ski3": (1_000_000, 3, 100)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def build(N, d, G, dev):
    g = torch.Generator().manual_seed(0)
    x = torch.rand(N, 8, generator=g)
    y = torch.sin(4 * x[:, 0]) * x[:, 1] + 0.05 * torch.randn(N, generator=g)
    x, y = x.to(dev), y.to(dev)
    lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.net = torch.nn.Sequential(torch.nn.Linear(8, 64), torch.nn.ReLU(), torch.nn.Linear(64, d))
            self.mean_module = gp.means.ConstantMean()
            if G is None:
                self.scale = torch.nn.Identity()
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())
            else:
                self.scale = ScaleToBounds(-1.0, 1.0)
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(
                    gp.kernels.RBFKernel(ard_num_dims=d), grid_size=G, num_dims=d, grid_bounds=[(-1.0, 1.0)] * d))

        detach_features = False

        def forward(self, xx):
            z = self.scale(self.net(xx))
            if self.detach_features:
                z = z.detach()
            return gp.distributions.MultivariateNormal(self.mean_module(z), self.covar_module(z))

    model = M().to(dev)
    return model, lik.to(dev), x, y


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0)


def run(name, steps, reps, dev):
    N, d, G = CONFIGS[name]
    model, lik, x, y = build(N, d, G, dev)
    model.train(); lik.train()
    mll = gp.ExactMarginalLogLikelihood(lik, model)
    rows = {"net_fwd": [], "mll_fwd": [], "hyper_bwd": [], "full_bwd": []}
    for r in range(reps + 1):
        for detach in (True, False):
            model.zero_grad()
            model.detach_features = detach
            z, t_net = timed(lambda: model.net(x))
            loss, t_mll = timed(lambda: -mll(model(x), y))
            _, t_bwd = timed(lambda: loss.backward())
            if r == 0:
                continue                      # warm-up: plans, workspaces, module loads
            if detach:
                rows["hyper_bwd"].append(t_bwd)
            else:
                rows["full_bwd"].append(t_bwd)
                rows["net_fwd"].append(t_net)
                rows["mll_fwd"].append(t_mll)
    med = {k: sorted(v)[len(v) // 2] for k, v in rows.items()}
    model.detach_features = False
    opt = torch.optim.Adam(list(model.parameters()) + list(lik.parameters()), lr=0.01)
    torch.cuda.reset_peak_memory_stats(dev)
    for _ in range(steps):
        opt.zero_grad()
        loss = -mll(model(x), y)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    return {"config": name, "N": N, "feature_d": d, "grid": None if G is None else f"{G}^{d}", "net_fwd_ms": med["net_fwd"],
            "mll_fwd_ms": med["mll_fwd"], "hyper_bwd_ms": med["hyper_bwd"], "input_bwd_ms": med["full_bwd"] - med["hyper_bwd"],
            "full_bwd_ms": med["full_bwd"], "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 1e9, "steps": steps,
            "plans_cached": len(gp.operators._PLAN_CACHE)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dkl_bench needs a GPU")
    dev = torch.device("cuda:0")
    info = card()
    for name in a.configs.split(","):
        res = run(name, a.steps, a.reps, dev)
        res["card"] = info
        print(json.dumps(res), flush=True)
        gp.operators.clear_plan_cache()


if __name__ == "__main__":
    main()
