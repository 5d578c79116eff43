"""Piecewise polynomial kernel timings on one GPU: one K.V launch of a compact-support plan (q = 2) against the dense fused RBF
kernel at the same N, the evaluated tile-pair fraction, the evaluated pairs per second, and one MLL evaluation (pivoted-Cholesky
preconditioner, mBCG, SLQ) with its CG iteration count.

    python tools/ppoly_bench.py [--ns 50000 200000 1000000] [--dims 2 3] [--neighbours 1000] [--rounds 5]

Uniform points on the unit cube with the lengthscale that gives about --neighbours points within r < 1 of each point.  Every K.V
time is the median over alternating rounds of gp_time_kmv_kernel (CUDA events around the launch alone, 16 columns).  The dense RBF
kernel runs up to --dense-max points; above that its time is extrapolated as (N / N_max)^2 times its time at N_max and labelled
"extrapolated".  The card's name, power limit and maximum SM clock are printed first, from the same run.  Prints JSON lines.
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


def ball_volume(d):
    return math.pi ** (d / 2) / math.gamma(d / 2 + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", type=int, nargs="+", default=[50000, 200000, 1000000])
    ap.add_argument("--dims", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--neighbours", type=float, default=1000.0)
    ap.add_argument("--dense-max", type=int, default=200000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ppoly_bench needs a GPU")
    from gpytorch_b200.engine import Plan
    from oracle import mll as om

    print(json.dumps({"card": card()}), flush=True)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    dense_ref = {}
    for d in a.dims:
        for n in sorted(a.ns):
            ls = (a.neighbours / (n * ball_volume(d))) ** (1.0 / d)   # n vol(ball of radius l) = neighbours
            x = torch.rand(n, d, generator=g).to(dev)
            V = torch.randn(n, 16, generator=g).to(dev)
            pp = Plan(x).set_hypers_pp(2, [ls], 1.0, 0.1)
            info = pp.info()
            row = {"d": d, "n": n, "lengthscale": ls, "tile_pairs": info["tile_pairs"], "tile_pairs_total": info["tile_pairs_total"],
                   "tile_pair_fraction": info["tile_pairs"] / info["tile_pairs_total"], "slots": info["nsplit"]}
            dense = Plan(x).set_hypers("rbf", [0.3], 1.0, 0.1) if n <= a.dense_max else None
            tp, td = [], []
            for _ in range(a.rounds):   # alternate the two kernels within every round
                tp.append(pp.time_kmv_kernel(V, 2, a.reps))
                if dense is not None:
                    td.append(dense.time_kmv_kernel(V, 2, a.reps))
            row["compact_kmv_ms"] = statistics.median(tp)
            pairs = info["tile_pairs"] * 128 * 64
            row["compact_pairs_per_s"] = pairs / (row["compact_kmv_ms"] * 1e-3)
            if dense is not None:
                row["dense_rbf_kmv_ms"] = statistics.median(td)
                row["dense_rbf_pairs_per_s"] = float(n) * n / (row["dense_rbf_kmv_ms"] * 1e-3)
                dense_ref[d] = (n, row["dense_rbf_kmv_ms"])
                dense.close()
            else:
                n0, t0 = dense_ref[d]
                row["dense_rbf_kmv_ms_extrapolated"] = t0 * (n / n0) ** 2
            # one MLL evaluation: preconditioner, mBCG with 10 probes, SLQ
            y = (torch.sin(8 * x[:, 0]) + 0.1 * torch.randn(n, device=dev)).contiguous()
            pn = om.make_probe_noise(n, 15, 10, 1)
            pn = tuple(t.to(dev) for t in pn)
            pp.mll(y, *pn, 10, 15, 2000)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res, _ = pp.mll(y, *pn, 10, 15, 2000)   # ends in a device synchronise (the results are read back)
            row["mll_ms"] = (time.perf_counter() - t0) * 1e3
            row["mll_cg_iters"] = res.cg_iters
            pp.close()
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
