"""Derivative-observation operator (RBFKernelGrad, or Matern52KernelGrad with --kernel matern52) against the plain K.V of the same
kernel on the same points (N = 20 000, t = 11 columns,
d in {2, 5, 10}), one MLL evaluation and the lengthscale + outputscale gradient pass on it, and the dense fp32 torch form of the
value / gradient covariance (from its block table) at the largest N whose matrix fits in memory, and the pivoted Cholesky that
the MLL's preconditioner starts from, on the derivative and on the plain plan.

    python tools/deriv_bench.py [--n 20000] [--ds 2,5,10] [--reps 20] [--kernel rbf|matern52]

Prints one JSON line per d with the card name and power limit.  Times are CUDA-event medians of whole calls; before every timed
call a 256 MB buffer is rewritten so that L2 (50 MB) holds none of the operands:
  kmv_plain   the plain plan of the same kernel, [N, 11];
  kmv_deriv   the derivative plan, [N (d+1), 11] (derivative kernel over 1 to 3 column chunks + the split sum + finish);
  deriv_over_plain, and the derivative kernel's FP32 rate: 2 (3 d + 3) t flops per pair (2 (3 d + 4) t for Matern-5/2) plus 3 d
  for the distance, over kmv_deriv, against the data sheet's 67 TFLOP/s;
  kmv_rbf_deriv  (--kernel matern52 only) the RBF derivative plan on the same points, timed interleaved with kmv_deriv, and
              m52_over_rbf_deriv;
  mll         gp_mll (pivoted-Cholesky rank 100, 10 probes, per-row noise);
  grad        gp_bilinear_grad with 11 columns (lengthscale(s) and outputscale);
  dense       the materialised fp32 N (d+1) x N (d+1) matrix (from the block table) times V, at dense_n points;
  pivots      the pivoted Cholesky (rank 100, tolerance 1e-3, as gp_mll asks for it) of the derivative plan and of the plain plan on
              the same points: the rank reached and whether it stopped on a non-positive or NaN residual diagonal (the condition on
              which gp_mll drops its preconditioner), and the MLL's preconditioner rank on the plain plan.
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

from gpytorch_b200.engine import DerivPlan, Plan  # noqa: E402

PEAK_FP32 = 67e12


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=10).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


_FLUSH = None


def _time(fn):
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(64 * 1024 * 1024, device="cuda:0")
    _FLUSH.fill_(1.0)   # evicts L2
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def _dense(x, ls, os_):
    """The value / gradient covariance materialised in fp32 from its block table ([0,0] = k, [0,b] = k u_b, [a,0] = -k u_a,
    [a,b] = k (delta_ab / l^2 - u_a u_b)) over [N, d+1, N, d+1], i.e. interleaved rows: what a dense implementation stores."""
    n, d = x.shape
    D = x[:, None, :] - x[None, :, :]                      # [n, n, d]
    u = D / ls ** 2
    k = torch.exp(-0.5 * (D / ls).square().sum(-1))        # [n, n]
    K = torch.empty(n, d + 1, n, d + 1, device=x.device)
    K[:, 0, :, 0] = k
    ku = k[..., None] * u
    K[:, 0, :, 1:] = ku
    K[:, 1:, :, 0] = -ku.permute(0, 2, 1)
    K[:, 1:, :, 1:] = (k[..., None, None] * (torch.eye(d, device=x.device) / ls ** 2 - u[..., :, None] * u[..., None, :])).permute(0, 2, 1, 3)
    return os_ * K.reshape(n * (d + 1), n * (d + 1))


def _dense_m52(x, ls, os_):
    """The Matern-5/2 value / gradient covariance materialised in fp32 from its block table ([0,0] = (1 + rho + rho^2/3) e,
    [0,b] = A u_b, [a,0] = -A u_a, [a,b] = A delta_ab / l^2 - B u_a u_b, A = (5/3)(1 + rho) e, B = (25/3) e), interleaved rows."""
    n, d = x.shape
    D = x[:, None, :] - x[None, :, :]
    u = D / ls ** 2
    rho = (5.0 * (D / ls).square().sum(-1)).sqrt()
    e = torch.exp(-rho)
    A = (5.0 / 3.0) * (1 + rho) * e
    B = (25.0 / 3.0) * e
    K = torch.empty(n, d + 1, n, d + 1, device=x.device)
    K[:, 0, :, 0] = (1 + rho + rho.square() / 3) * e
    Au = A[..., None] * u
    K[:, 0, :, 1:] = Au
    K[:, 1:, :, 0] = -Au.permute(0, 2, 1)
    K[:, 1:, :, 1:] = (A[..., None, None] * torch.eye(d, device=x.device) / ls ** 2
                       - B[..., None, None] * u[..., :, None] * u[..., None, :]).permute(0, 2, 1, 3)
    return os_ * K.reshape(n * (d + 1), n * (d + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--ds", default="2,5,10")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--kernel", choices=["rbf", "matern52"], default="rbf")
    a = ap.parse_args()
    kind = a.kernel
    dense = _dense if kind == "rbf" else _dense_m52
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n, t = a.n, 11
    name, pl = _card()
    free = torch.cuda.mem_get_info(0)[0]
    for d in [int(v) for v in a.ds.split(",")]:
        x = torch.rand(n, d, device=dev, generator=g)
        ls = 0.5 * d ** 0.5
        data = Plan(x).set_hypers(kind, ls, 1.0, 0.0)
        dp = DerivPlan(data, kind).set_noise(0.0)
        dp.set_noise_diag((0.01 + 0.05 * torch.rand(d + 1, device=dev, generator=g)).repeat(n))
        V1 = torch.randn(n, t, device=dev, generator=g)
        VD = torch.randn(n * (d + 1), t, device=dev, generator=g)
        for _ in range(3):
            data.kmv(V1), dp.kmv(VD)
        rbf_dp = None
        if kind != "rbf":   # the RBF derivative operator on the same points, for the comparison
            rbf_dp = DerivPlan(Plan(x).set_hypers("rbf", ls, 1.0, 0.0)).set_noise(0.0)
            for _ in range(3):
                rbf_dp.kmv(VD)
        ta, tb, tr = [], [], []
        for _ in range(a.reps):
            ta.append(_time(lambda: data.kmv(V1)))
            tb.append(_time(lambda: dp.kmv(VD)))
            if rbf_dp is not None:
                tr.append(_time(lambda: rbf_dp.kmv(VD)))
        ma, mb = statistics.median(ta), statistics.median(tb)
        extra = {}
        if rbf_dp is not None:
            mr = statistics.median(tr)
            extra = {"kmv_rbf_deriv_ms": round(mr, 4), "m52_over_rbf_deriv": round(mb / mr, 3),
                     "kmv_deriv_minmax_ms": [round(min(tb), 4), round(max(tb), 4)],
                     "kmv_rbf_deriv_minmax_ms": [round(min(tr), 4), round(max(tr), 4)]}
            rbf_dp.close()
        flops = float(n) * n * (2 * (3 * d + (3 if kind == "rbf" else 4)) * t + 3 * d)
        tpn = 10
        N = n * (d + 1)
        y = torch.randn(N, device=dev, generator=g)
        eps1 = torch.randn(100, tpn, device=dev, generator=g)
        eps2 = torch.randn(N, tpn, device=dev, generator=g)
        rad = torch.randint(0, 2, (N, tpn), device=dev, generator=g).float() * 2 - 1
        run_mll = lambda: dp.mll(y, eps1, eps2, rad, num_probes=tpn, precond_rank=100, warn=False)  # noqa: E731
        res, _ = run_mll()
        t_mll = statistics.median([_time(run_mll) for _ in range(3)])
        Lf = torch.randn(N, t, device=dev, generator=g)
        Rf = torch.randn(N, t, device=dev, generator=g)
        dp.bilinear_grad(Lf, Rf)
        t_grad = statistics.median([_time(lambda: dp.bilinear_grad(Lf, Rf)) for _ in range(3)])
        # pivoted Cholesky as gp_mll runs it (rank 100, tolerance 1e-3) on the derivative plan and on the plain plan over the same
        # points; status 5 (GP_W_PIVCHOL_NAN) = a non-positive or NaN maximum of the residual diagonal, and gp_mll then drops the
        # preconditioner
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            lt_d, _, st_d = dp.pivoted_cholesky(100, 1e-3)
            data.set_hypers(kind, ls, 1.0, float(0.03))
            lt_p, _, st_p = data.pivoted_cholesky(100, 1e-3)
            res_p, _ = data.mll(torch.randn(n, device=dev, generator=g), eps1, torch.randn(n, tpn, device=dev, generator=g),
                                torch.randint(0, 2, (n, tpn), device=dev, generator=g).float() * 2 - 1, num_probes=tpn,
                                precond_rank=100, warn=False)
        # dense: the largest n whose fp32 matrix ((d+1)^2 n^2 floats) and its temporaries (three [n, n, d, d] Hessian blocks, a few
        # [n, n, d]) fit in 80 % of the memory that was free at the start
        dn = int((0.8 * free / (4.0 * ((d + 1) ** 2 + 3 * d * d + 4 * d))) ** 0.5)
        dn = max(64, min(dn, n))
        xd = x[:dn].contiguous()
        Vd = torch.randn(dn * (d + 1), t, device=dev, generator=g)
        try:
            dense(xd, ls, 1.0) @ Vd
            torch.cuda.synchronize()
            t_dense = statistics.median([_time(lambda: dense(xd, ls, 1.0) @ Vd) for _ in range(3)])
        except torch.OutOfMemoryError:
            t_dense = None
        torch.cuda.empty_cache()
        dsub = DerivPlan(Plan(xd).set_hypers(kind, ls, 1.0, 0.0), kind).set_noise(0.0)
        dsub.kmv(Vd)
        t_sub = statistics.median([_time(lambda: dsub.kmv(Vd)) for _ in range(5)])
        print(json.dumps({"d": d, "n": n, "t": t, "kmv_plain_ms": round(ma, 4), "kmv_deriv_ms": round(mb, 4),
                          "deriv_over_plain": round(mb / ma, 2), "deriv_tflops": round(flops / (mb * 1e-3) / 1e12, 2),
                          "deriv_share_of_fp32_peak": round(flops / (mb * 1e-3) / PEAK_FP32, 3),
                          "mll_ms": round(t_mll, 2), "mll_cg_iters": res.cg_iters, "mll_precond_rank": res.precond_rank,
                          "grad_ms": round(t_grad, 3), "pivchol_deriv_rank": lt_d.size(0), "pivchol_deriv_status": st_d,
                          "pivchol_plain_rank": lt_p.size(0), "pivchol_plain_status": st_p, "mll_plain_precond_rank": res_p.precond_rank, "dense_n": dn, "dense_fp32_ms": None if t_dense is None else round(t_dense, 2),
                          "deriv_at_dense_n_ms": round(t_sub, 3), **extra, "card": name, "power_limit": pl}), flush=True)
        dp.close()
        dsub.close()


if __name__ == "__main__":
    main()
