"""Hadamard multitask K.V against the plain K.V on the same inputs (BASELINE C2 sizes: N = 50 000, d = 10, RBF), T in {1, 2, 4, 8}
tasks assigned at random, plus one MLL evaluation and the gradient passes of its backward on the multitask plan.

    python tools/hadamard_bench.py [--n 50000] [--d 10] [--reps 20]

Prints one JSON line per T with the card name and power limit.  The two products alternate launch by launch in one run, so clock
drift hits both alike; times are CUDA-event medians of whole gp_kmv calls (the multitask one includes the V gather, the V tiles,
one fused launch per column task and the combine pass).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpytorch_b200.engine import Plan  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=10).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--d", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tasks", default="1,2,4,8")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n, d = a.n, a.d
    x = torch.rand(n, d, device=dev, generator=g)
    y = torch.randn(n, device=dev, generator=g)
    V = torch.randn(n, 16, device=dev, generator=g)
    name, pl = _card()
    plain = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.1)
    for T in [int(v) for v in a.tasks.split(",")]:
        t = torch.randint(0, T, (n,), device=dev, generator=g)
        F = torch.randn(T, 2, device=dev, generator=g)
        B = F @ F.t() + torch.diag(0.5 + torch.rand(T, device=dev, generator=g))
        mt = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
        mt.set_tasks(t, None, T).set_task_covar(B)
        mt.set_noise_diag((0.05 + 0.1 * torch.rand(T, device=dev, generator=g))[t])
        for _ in range(3):
            plain.kmv(V)
            mt.kmv(V)
        tp, tm = [], []
        for _ in range(a.reps):
            tp.append(_time(lambda: plain.kmv(V)))
            tm.append(_time(lambda: mt.kmv(V)))
        tp_med, tm_med = statistics.median(tp), statistics.median(tm)
        # one MLL evaluation (preconditioner rank 100, 10 probes: BASELINE C2 settings), then its backward's gradient passes:
        # lengthscale / outputscale and dB of sum(L * (K o B) R) with L, R = [solves | probes] (11 columns)
        tpn = 10
        eps1 = torch.randn(100, tpn, device=dev, generator=g)
        eps2 = torch.randn(n, tpn, device=dev, generator=g)
        rad = torch.randint(0, 2, (n, tpn), device=dev, generator=g).float() * 2 - 1
        run_mll = lambda: mt.mll(y, eps1, eps2, rad, num_probes=tpn, precond_rank=100, warn=False)
        run_mll()
        t_mll = statistics.median([_time(run_mll) for _ in range(3)])
        Lf = torch.randn(n, tpn + 1, device=dev, generator=g)
        Rf = torch.randn(n, tpn + 1, device=dev, generator=g)
        mt.bilinear_grad(Lf, Rf)
        mt.task_covar_grad(Lf, Rf)
        t_hyp = statistics.median([_time(lambda: mt.bilinear_grad(Lf, Rf)) for _ in range(3)])
        t_dB = statistics.median([_time(lambda: mt.task_covar_grad(Lf, Rf)) for _ in range(3)])
        print(json.dumps({"T": T, "n": n, "d": d, "kmv_plain_ms": round(tp_med, 4), "kmv_hadamard_ms": round(tm_med, 4),
                          "ratio": round(tm_med / tp_med, 3), "mll_ms": round(t_mll, 3), "grad_ls_os_ms": round(t_hyp, 3),
                          "grad_B_ms": round(t_dB, 3), "card": name, "power_limit": pl}), flush=True)
        mt.close()


if __name__ == "__main__":
    main()
