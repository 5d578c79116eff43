"""Kronecker multitask K.V against the plain K.V and against the same operator in Hadamard form (N = 20 000, d = 10, RBF, 11
columns, T in {1, 2, 4, 8}, a random B of rank 2), plus one MLL evaluation and the gradient passes of its backward on the Kronecker
plan.

    python tools/kron_bench.py [--n 20000] [--d 10] [--reps 20] [--tasks 1,2,4,8]

Prints one JSON line per T with the card name and power limit.  The three products alternate call by call in one run, so clock
drift hits them alike; times are CUDA-event medians of whole gp_kmv calls:
  (a) plain     the data plan alone, [N, 11];
  (b) kron      the Kronecker plan, [N T, 11]: B mix, ceil(11 T / 16) launches of the data kernel, scatter;
  (c) hadamard  the Hadamard plan over the N T repeated inputs with task ids r mod T (the same operator), [N T, 11].
`launch_equiv` = ceil(11 T / 16); `kron_over_launch_equiv` = kron / (launch_equiv x plain).
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpytorch_b200.engine import KronPlan, Plan  # noqa: E402


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
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--d", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tasks", default="1,2,4,8")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n, d, t = a.n, a.d, 11
    x = torch.rand(n, d, device=dev, generator=g)
    name, pl = _card()
    data = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    V1 = torch.randn(n, t, device=dev, generator=g)
    for T in [int(v) for v in a.tasks.split(",")]:
        F = torch.randn(T, 2, device=dev, generator=g)
        B = F @ F.t() + torch.diag(0.5 + torch.rand(T, device=dev, generator=g))
        kp = KronPlan(data, T).set_noise(0.0)
        kp.set_task_covar(B)
        kp.set_noise_diag((0.05 + 0.1 * torch.rand(T, device=dev, generator=g)).repeat(n))
        hp = Plan(x.repeat_interleave(T, 0)).set_hypers("rbf", 0.5, 1.0, 0.0)
        hp.set_tasks(torch.arange(n * T, device=dev) % T, None, T).set_task_covar(B)
        VT = torch.randn(n * T, t, device=dev, generator=g)
        for _ in range(3):
            data.kmv(V1), kp.kmv(VT), hp.kmv(VT)
        ta, tb, tc = [], [], []
        for _ in range(a.reps):
            ta.append(_time(lambda: data.kmv(V1)))
            tb.append(_time(lambda: kp.kmv(VT)))
            tc.append(_time(lambda: hp.kmv(VT)))
        ma, mb, mc = statistics.median(ta), statistics.median(tb), statistics.median(tc)
        le = math.ceil(t * T / 16)
        # one MLL evaluation (preconditioner rank 100, 10 probes, per-task noise), then its backward's gradient passes: lengthscale /
        # outputscale and dB of sum(L * ((s K) (x) B) R) with L, R = [solves | probes] (11 columns)
        tpn = 10
        y = torch.randn(n * T, device=dev, generator=g)
        eps1 = torch.randn(100, tpn, device=dev, generator=g)
        eps2 = torch.randn(n * T, tpn, device=dev, generator=g)
        rad = torch.randint(0, 2, (n * T, tpn), device=dev, generator=g).float() * 2 - 1
        run_mll = lambda: kp.mll(y, eps1, eps2, rad, num_probes=tpn, precond_rank=100, warn=False)  # noqa: E731
        res, _ = run_mll()
        t_mll = statistics.median([_time(run_mll) for _ in range(3)])
        Lf = torch.randn(n * T, tpn + 1, device=dev, generator=g)
        Rf = torch.randn(n * T, tpn + 1, device=dev, generator=g)
        kp.bilinear_grad(Lf, Rf)
        kp.task_covar_grad(Lf, Rf)
        t_hyp = statistics.median([_time(lambda: kp.bilinear_grad(Lf, Rf)) for _ in range(3)])
        t_dB = statistics.median([_time(lambda: kp.task_covar_grad(Lf, Rf)) for _ in range(3)])
        print(json.dumps({"T": T, "n": n, "d": d, "t": t, "kmv_plain_ms": round(ma, 4), "kmv_kron_ms": round(mb, 4),
                          "kmv_hadamard_ms": round(mc, 4), "hadamard_over_kron": round(mc / mb, 3), "launch_equiv": le,
                          "kron_over_launch_equiv": round(mb / (le * ma), 3), "mll_ms": round(t_mll, 3), "mll_cg_iters": res.cg_iters,
                          "grad_ls_os_ms": round(t_hyp, 3), "grad_B_ms": round(t_dB, 3), "card": name, "power_limit": pl}), flush=True)
        kp.close()
        hp.close()


if __name__ == "__main__":
    main()
