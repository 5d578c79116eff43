#!/usr/bin/env python
"""kmv_bench.py -- the fused K.V kernel (csrc/kmv_tc.cu) alone, for every kernel kind at the C2 and C3 shapes.

    python tools/kmv_bench.py [--reps 20] [--shapes c2,c3] [--json out.json]

Shapes (X ~ U[0,1]^{N x d}, 11 right-hand sides = 10 probes + y, as bench.py):
  c2  N = 50 000,  d = 10, lengthscale 1
  c3  N = 200 000, d = 20, lengthscale 2  (the whole C3 matrix on one GPU)
Per kind and shape: ms per launch (gp_time_kmv_kernel: CUDA events around back-to-back launches), pairs / s, and two lower
bounds at the card's maximum SM clock:
  tensor  96 + 2 KP tf32 flop per pair (GEMM1 m64n64k8 x KP/8: 2 KP; GEMM2 8 x (m64n32k8 + m64n16k8): 96), i.e. 176 at
          KP = 40 (c2) and 224 at KP = 64 (c3), at 2048 dense tf32 flop / clk / SM
  mufu    one ex2 per pair (RBF) or ex2 + sqrt (Matern) at 16 MUFU ops / clk / SM
The card name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.
The gradient kinds (GP_DERIV + kind) are timed through gp_bilinear_grad with a scalar lengthscale (CUDA events around
the whole call): one launch of the forward kind, one of the derivative kind, two small dot-product kernels and a host
read-back.  "grad_ms" is that call; grad_ms - ms_per_launch approximates the derivative-kind launch.
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

SHAPES = {"c2": dict(n=50000, d=10, lengthscale=1.0), "c3": dict(n=200000, d=20, lengthscale=2.0)}
KINDS = ["rbf", "matern12", "matern32", "matern52"]
T_COLS = 11


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def time_bilinear_grad(plan, v, reps):
    left = torch.randn_like(v)
    for _ in range(2):
        plan.bilinear_grad(left, v)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = max(1, reps // 4)
    e0.record()
    for _ in range(n):
        plan.bilinear_grad(left, v)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from gpytorch_b200.engine import Plan

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    hz = gpu["max_sm_clock_mhz"] * 1e6
    rows = []
    for shape in args.shapes.split(","):
        w = SHAPES[shape]
        g = torch.Generator().manual_seed(0)
        x = torch.rand(w["n"], w["d"], generator=g, dtype=torch.float64).float().to(dev)
        v = torch.randn(w["n"], T_COLS, generator=g).to(dev)
        for kind in KINDS:
            plan = Plan(x, backend="tcgen05")
            plan.set_hypers(kind, w["lengthscale"], 1.0, 0.1)
            info = plan.info()
            ms = plan.time_kmv_kernel(v, warmup=3, reps=args.reps)
            pairs = float(w["n"]) * w["n"]
            flop_pair = 96.0 + 2.0 * info["kpad"]
            tensor_ms = pairs * flop_pair / (2048.0 * n_sm * hz) * 1e3
            mufu_ms = pairs * (1 if kind == "rbf" else 2) / (16.0 * n_sm * hz) * 1e3
            grad_ms = time_bilinear_grad(plan, v, args.reps)
            row = {"shape": shape, "kind": kind, "n": w["n"], "d": w["d"], "kpad": info["kpad"], "nsplit": info["nsplit"],
                   "ms_per_launch": ms, "pairs_per_s": pairs / (ms * 1e-3), "tensor_bound_ms": tensor_ms, "mufu_bound_ms": mufu_ms,
                   "grad_ms": grad_ms}
            rows.append(row)
            print(f"{shape} {kind:9s} KP={info['kpad']:3d} nsplit={info['nsplit']}  {ms:8.3f} ms  {row['pairs_per_s']:.3e} pairs/s  "
                  f"bounds: tensor {tensor_ms:.3f} ms, mufu {mufu_ms:.3f} ms  grad {grad_ms:8.3f} ms", flush=True)
            del plan
    out = {"gpu": gpu, "n_sm": n_sm, "results": rows}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
