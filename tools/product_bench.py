#!/usr/bin/env python
"""Device time of one fused K.V product of a kernel product against the plain fused kernel (CUDA events, gp_time_kmv_kernel).

    python tools/product_bench.py [--n 50000] [--t 11] [--reps 20] [--rounds 5]

Prints the card name and its power limit, then, at N x N with t right-hand sides, the median over `rounds` alternating rounds (one
process, after warm-up) of the time of ONE launch of
    plain      kmv_tc_kernel, RBF d = 10
    A tc/simt  RBF(d = 8) x Matern-5/2(d = 2)   on product_tc_kernel / product_simt_kernel
    B tc/simt  Matern-5/2(d = 8) x Matern-1/2(d = 2)
and every product's ratio to the plain kernel.  Needs a CUDA device: there is nothing to time without one."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--t", type=int, default=11)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("product_bench needs a CUDA device (H100): a time taken anywhere else says nothing about the kernels")
    from gpytorch_b200.engine import Plan

    dev = torch.device("cuda:0")
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(f"card: {card}; power limit: {power}")
    g = torch.Generator().manual_seed(0)
    x = torch.rand(a.n, 10, generator=g).to(dev)
    v = torch.randn(a.n, a.t, generator=g).to(dev)
    xa, xb = x[:, :8].contiguous(), x[:, 8:].contiguous()
    plans = {"plain": Plan(x, backend="tcgen05").set_hypers("rbf", 1.0, 1.0, 0.0)}
    keep = []
    for tag, ka, kb in (("A", "rbf", "matern52"), ("B", "matern52", "matern12")):
        for be in ("tcgen05", "simt"):
            fa = Plan(xa, backend=be).set_hypers(ka, 0.9, 1.0, 0.0)
            fb = Plan(xb, backend=be).set_hypers(kb, 0.4, 1.0, 0.0)
            keep += [fa, fb]
            p = Plan(x).set_product([fa, fb]).set_hypers("rbf", [1.0], 1.0, 0.0)
            assert p.info()["backend"] == "product"
            plans[f"{tag} {ka} x {kb} {'tc' if be == 'tcgen05' else 'simt'}"] = p
    times = {k: [] for k in plans}
    for k, p in plans.items():   # warm-up: module load, workspaces
        p.time_kmv_kernel(v, warmup=2, reps=2)
    for _ in range(a.rounds):     # alternate the kernels inside one process
        for k, p in plans.items():
            times[k].append(p.time_kmv_kernel(v, warmup=1, reps=a.reps))
    med = {k: statistics.median(ts) for k, ts in times.items()}
    for k, m in med.items():
        print(f"{k:34s} {m:9.3f} ms  (min {min(times[k]):.3f}, max {max(times[k]):.3f})  x{m / med['plain']:.2f} of plain")
    print(json.dumps({"card": card, "power_limit": power, "n": a.n, "t": a.t, "ms": med,
                      "ratio_to_plain": {k: m / med["plain"] for k, m in med.items()}}))


if __name__ == "__main__":
    main()
