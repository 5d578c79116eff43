"""LCM K.V (gp_plan_set_kron_terms) against the Kronecker products of its individual terms (N = 20 000, d = 10, 11 columns, T in
{2, 4, 8}, Q in {1, 2, 3} terms: RBF, Matern-5/2 and Matern-1/2 data kernels on the tensor cores, each with its own lengthscale and
a random rank-2 B_q), plus one MLL evaluation and one gp_kron_terms_grad call on the LCM plan.

    python tools/lcm_bench.py [--n 20000] [--d 10] [--reps 20] [--tasks 2,4,8] [--terms 1,2,3]

Prints one JSON line per (T, Q) with the card name and power limit.  The LCM product and its terms' Kronecker products alternate
call by call in one run, so clock drift hits them alike; times are CUDA-event medians of whole gp_kmv calls.
`lcm_over_sum_of_terms` = lcm / sum_q kron_q (the projection is 1: the LCM product is its terms' launches plus one scatter).
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

from gpytorch_b200.engine import KronPlan, LcmPlan, Plan  # noqa: E402

KINDS = ["rbf", "matern52", "matern12"]


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


def _B(T, g, dev):
    F = torch.randn(T, 2, device=dev, generator=g)
    return F @ F.t() + torch.diag(0.1 + torch.rand(T, device=dev, generator=g))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--d", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tasks", default="2,4,8")
    ap.add_argument("--terms", default="1,2,3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lcm_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n, d, t = a.n, a.d, 11
    x = torch.rand(n, d, device=dev, generator=g)
    name, pl = _card()
    datas = [Plan(x, backend="tcgen05").set_hypers(KINDS[q], 0.3 + 0.4 * q, 0.8 + 0.3 * q, 0.0) for q in range(3)]
    for T in [int(v) for v in a.tasks.split(",")]:
        Bs = [_B(T, g, dev) for _ in range(3)]
        krons = []
        for q in range(3):
            kp = KronPlan(datas[q], T).set_noise(0.1)
            kp.set_task_covar(Bs[q])
            krons.append(kp)
        V = torch.randn(n * T, t, device=dev, generator=g)
        for Q in [int(v) for v in a.terms.split(",")]:
            lp = LcmPlan(datas[:Q], T).set_noise(0.1)
            lp.set_term_covars(torch.stack(Bs[:Q]))
            calls = [lambda: lp.kmv(V)] + [lambda k=k: k.kmv(V) for k in krons[:Q]]
            for f in calls:   # warm every shape
                f(); f()
            ts = [[] for _ in calls]
            for _ in range(a.reps):
                for i, f in enumerate(calls):
                    ts[i].append(_time(f))
            med = [statistics.median(v) for v in ts]
            y = torch.randn(n * T, device=dev, generator=g)
            tp = 10
            eps1 = torch.randn(15, tp, device=dev, generator=g)
            eps2 = torch.randn(n * T, tp, device=dev, generator=g)
            rad = torch.randint(0, 2, (n * T, tp), device=dev, generator=g).float() * 2 - 1
            lp.mll(y, eps1, eps2, rad, num_probes=tp, precond_rank=15, min_precond_size=1, warn=False)
            mll_ms = _time(lambda: lp.mll(y, eps1, eps2, rad, num_probes=tp, precond_rank=15, min_precond_size=1, warn=False))
            L = torch.randn(n * T, t, device=dev, generator=g)
            lp.terms_grad(L, V)
            grad_ms = _time(lambda: lp.terms_grad(L, V))
            print(json.dumps({"card": name, "power_limit": pl, "n": n, "d": d, "cols": t, "T": T, "Q": Q,
                              "lcm_kmv_ms": round(med[0], 4), "term_kron_kmv_ms": [round(v, 4) for v in med[1:]],
                              "lcm_over_sum_of_terms": round(med[0] / sum(med[1:]), 4), "mll_ms": round(mll_ms, 3),
                              "terms_grad_ms": round(grad_ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
