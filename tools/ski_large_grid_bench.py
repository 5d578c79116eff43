"""KISS-GP on grids over 128 nodes per dimension: time of one SKI product (Plan.kmv, 16 columns), of an MLL evaluation with its
hyper-parameter gradient (gp_mll + bilinear_grad), and of grid prediction (gp_ski_grid_matmul of one column + gp_ski_interp_matmul
to 10^5 test points), at N = 10^6 on 1-D grids of 1024, 8192 and 131072 nodes and on a 1000^2 grid, for a short and a long
lengthscale.  The mode-product kernels alone are timed with torch.profiler and their 3xTF32 rate is reported against the band-limited flop
count sum_i (M / G_i) 16 nnz(T_i) 6 (nnz(T_i) = the entries with |a - b| < band_i; 3 MMAs of 2 flops per term).

    python tools/ski_large_grid_bench.py [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import shutil
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import ski_large_grid_oracle as lo  # noqa: E402
import ski_scale_oracle as so  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    smi = shutil.which("nvidia-smi")
    q = subprocess.run([smi, "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True) if smi else None
    return f"{name}, power limit {(q.stdout.strip() if q else '') or 'unknown'}"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def band_flops(sizes, kind, ls, step):
    M = math.prod(sizes)
    f = 0
    for G, s in zip(sizes, step):
        b = lo.band_end(lo.column_fp32(kind, G, s, ls)) if G > lo.DENSE_G else G
        nnz = G + 2 * sum(G - k for k in range(1, b))
        f += (M // G) * 16 * nnz * 6
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()
    from gpytorch_b200.engine import Plan

    dev = torch.device("cuda:0")
    print(f"# {card()}")
    n = args.n
    g = torch.Generator().manual_seed(0)
    xt = torch.rand(100_000, 2, generator=g)
    rows = []
    for sizes in ([1024], [8192], [131072], [1000, 1000]):
        d = len(sizes)
        axes, lo_, step = so.bench_grid(sizes)
        x = torch.rand(n, d, generator=g).to(dev)
        y = torch.sin(6 * x.sum(-1))
        for ls in (0.02, 0.2):
            p = Plan(x).set_ski(sizes, lo_, step).set_hypers("rbf", ls, 1.0, 0.1)
            V = torch.randn(n, 16, device=dev)
            kmv_ms = timed(lambda: p.kmv(V), args.reps)
            grid_ms = timed(lambda: p.ski_grid_matmul(V), args.reps)
            eps1 = torch.randn(n, 10, device=dev)
            eps2 = torch.randn(15, 10, device=dev)
            rad = (torch.randint(0, 2, (n, 10), device=dev) * 2 - 1).float()

            def mll_step():
                p.mll(y, eps1, eps2, rad, 10, 15, 10 ** 9, cg_tol=1.0, max_cg_iter=20, warn=False)
                p.bilinear_grad(V[:, :2], V[:, 2:4])

            mll_ms = timed(mll_step, max(1, args.reps // 5))
            c = p.ski_grid_matmul(y[:, None].contiguous())
            pt = Plan(xt[:, :d].contiguous().to(dev) * 0.98 + 0.01).set_ski(sizes, lo_, step).set_hypers("rbf", ls, 1.0, 0.1)
            pred_ms = timed(lambda: (p.ski_grid_matmul(y[:, None].contiguous()), pt.ski_interp_matmul(c)), args.reps)
            # mode-product kernel time (ski_mode_kernel / ski_mode_banded_kernel) of one product, from the profiler
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    p.kmv(V)
                torch.cuda.synchronize()
            mode_us = sum(e.device_time_total for e in prof.key_averages() if "ski_mode" in e.key) / 3
            fl = band_flops(sizes, "rbf", ls, step)
            band = [lo.band_end(lo.column_fp32("rbf", G, s, ls)) for G, s in zip(sizes, step)]
            row = dict(grid=sizes, n=n, ls=ls, band=band, kmv_ms=round(kmv_ms, 3), grid_matmul_ms=round(grid_ms, 3),
                       mll_step_ms=round(mll_ms, 2), predict_ms=round(pred_ms, 3), mode_us=round(mode_us, 1),
                       mode_tflops=round(fl / (mode_us * 1e-6) / 1e12, 2) if mode_us else None, band_gflop=round(fl / 1e9, 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
            pt.close()
            p.close()
    return rows


if __name__ == "__main__":
    main()
