"""Masked Kronecker K.V (settings.observation_nan_policy("mask") on a MultitaskKernel model) against the unmasked Kronecker K.V and
against a Hadamard plan over the same observed rows (N = 20 000, d = 10, RBF, 11 columns, T in {2, 4, 8}, a random B of rank 2,
observed fraction rho in {1, 0.9, 0.7, 0.5, 0.3} drawn uniformly over the N T entries), plus one MLL evaluation on each.

    python tools/kron_mask_bench.py [--n 20000] [--d 10] [--reps 20] [--tasks 2,4,8] [--rho 1,0.9,0.7,0.5,0.3]

Prints one JSON line per (T, rho) with the card name and power limit.  The three products alternate call by call, so clock drift
hits them alike; times are CUDA-event medians of whole gp_kmv calls:
  (a) kron       the unmasked Kronecker plan, [N T, 11];
  (b) masked     the same plan with the observed rows set (gp_plan_set_kron_observed), [rho N T, 11];
  (c) hadamard   a Hadamard plan over the rho N T observed (point, task) pairs, [rho N T, 11].
`masked_over_kron` is (b) / (a); `hadamard_over_masked` > 1 means the masked Kronecker operator is the faster form at this rho.
The MLL times are one gp_mll call each (preconditioner rank 100, 10 probes, noise 0.1) on (b) and (c)."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpytorch_b200.engine import KronPlan, Plan  # noqa: E402
from kron_bench import _card, _time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--d", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tasks", default="2,4,8")
    ap.add_argument("--rho", default="1,0.9,0.7,0.5,0.3")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n, d, t, tpn = a.n, a.d, 11, 10
    x = torch.rand(n, d, device=dev, generator=g)
    name, pl = _card()
    data = Plan(x).set_hypers("rbf", 0.5, 1.0, 0.0)
    for T in [int(v) for v in a.tasks.split(",")]:
        F = torch.randn(T, 2, device=dev, generator=g)
        B = F @ F.t() + torch.diag(0.5 + torch.rand(T, device=dev, generator=g))
        kp = KronPlan(data, T).set_noise(0.1)
        kp.set_task_covar(B)
        mp = KronPlan(data, T).set_noise(0.1)
        mp.set_task_covar(B)
        VT = torch.randn(n * T, t, device=dev, generator=g)
        for rho in [float(v) for v in a.rho.split(",")]:
            keep = torch.rand(n * T, device=dev, generator=g) < rho if rho < 1 else torch.ones(n * T, dtype=torch.bool, device=dev)
            rows = keep.nonzero().reshape(-1)
            m = rows.numel()
            mp.set_observed(rows if m < n * T else None, None)
            hp = Plan(x[rows // T].contiguous()).set_hypers("rbf", 0.5, 1.0, 0.1)
            hp.set_tasks(rows % T, None, T).set_task_covar(B)
            Vm = VT[:m].contiguous()
            out_m, out_h = mp.kmv(Vm), hp.kmv(Vm)
            rel = float((out_m - out_h).abs().max() / out_h.abs().max())
            for _ in range(3):
                kp.kmv(VT), mp.kmv(Vm), hp.kmv(Vm)
            ta, tb, tc = [], [], []
            for _ in range(a.reps):
                ta.append(_time(lambda: kp.kmv(VT)))
                tb.append(_time(lambda: mp.kmv(Vm)))
                tc.append(_time(lambda: hp.kmv(Vm)))
            ma, mb, mc = statistics.median(ta), statistics.median(tb), statistics.median(tc)
            y = torch.randn(m, device=dev, generator=g)
            eps1 = torch.randn(100, tpn, device=dev, generator=g)
            eps2 = torch.randn(m, tpn, device=dev, generator=g)
            rad = torch.randint(0, 2, (m, tpn), device=dev, generator=g).float() * 2 - 1
            mll_m = lambda: mp.mll(y, eps1, eps2, rad, num_probes=tpn, precond_rank=100, warn=False)  # noqa: E731
            mll_h = lambda: hp.mll(y, eps1, eps2, rad, num_probes=tpn, precond_rank=100, warn=False)  # noqa: E731
            rm, _ = mll_m()
            rh, _ = mll_h()
            t_mm, t_mh = _time(mll_m), _time(mll_h)
            print(json.dumps({"T": T, "rho": rho, "n": n, "d": d, "t": t, "rows": m, "kmv_kron_ms": round(ma, 4),
                              "kmv_masked_ms": round(mb, 4), "kmv_hadamard_ms": round(mc, 4), "masked_over_kron": round(mb / ma, 3),
                              "hadamard_over_masked": round(mc / mb, 3), "masked_vs_hadamard_rel": f"{rel:.2e}",
                              "mll_masked_ms": round(t_mm, 3), "mll_hadamard_ms": round(t_mh, 3), "mll_masked_cg_iters": rm.cg_iters,
                              "mll_hadamard_cg_iters": rh.cg_iters, "card": name, "power_limit": pl}), flush=True)
            hp.close()
        kp.close()
        mp.close()


if __name__ == "__main__":
    main()
