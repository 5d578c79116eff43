"""Pivoted-Cholesky timings on one GPU at the benchmark's C2 (N = 50,000, d = 10) and C3 (N = 200,000, d = 20, Matern-5/2) sizes,
rank 100, and of a kernel sum (RBF + Matern-5/2, N = 50,000, d = 6) at rank 40, where three CTAs per SM fit, for two builds of the
library run alternately in one call (A/B), with their pivots and factors compared bit for bit.

    python tools/pivchol_bench.py [--lib-a PATH] [--lib-b PATH] [--rounds 5] [--reps 20] [--out DIR]

--lib-a defaults to gpytorch_b200/lib/parent/libgpbbmm.so, a build of the commit to compare against, made for example with
    git worktree add /tmp/parent HEAD^ && (cd /tmp/parent && python -m gpytorch_b200.build)
    mkdir -p gpytorch_b200/lib/parent && cp /tmp/parent/gpytorch_b200/lib/libgpbbmm.so gpytorch_b200/lib/parent/
--lib-b defaults to this tree's gpytorch_b200/lib/libgpbbmm.so.

Each round runs one child process per library (GPBBMM_LIB selects the shared object); a child times --reps calls of
Plan.pivoted_cholesky with CUDA events after one warm-up call and saves its last factor and pivots under --out.  The card's name
and power limit are printed first, from the same run.  Prints JSON lines; the last one holds the per-size medians, the spread
between rounds and whether the two builds' factors are bit-identical.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
SIZES = {"c2": (50000, 10, "rbf", 1.0, 100), "c3": (200000, 20, "matern52", 1.0, 100), "sum": (50000, 6, "sum", 1.0, 40)}
TOL = 0.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = "unknown", "unknown"
    return {"card": name, "power_limit": power}


def child(size, reps, save):
    sys.path.insert(0, ROOT)
    import torch

    from gpytorch_b200.engine import Plan
    from oracle import mll as om

    n, d, kind, ls, rank = SIZES[size]
    x, _ = om.synthetic_problem(n, d, 0, torch.float32)
    terms = []
    if kind == "sum":
        terms = [Plan(x[:, :3].contiguous().cuda()).set_hypers("rbf", 0.6, 1.2, 0.0), Plan(x.cuda()).set_hypers("matern52", ls, 0.7, 0.0)]
        p = Plan(x.cuda()).set_sum(terms).set_hypers("rbf", [1.0], 1.0, 0.1)
    else:
        p = Plan(x.cuda()).set_hypers(kind, ls, 1.0, 0.1)
    lt, piv, _ = p.pivoted_cholesky(rank, TOL)      # warm-up: module load, buffers
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        lt, piv, _ = p.pivoted_cholesky(rank, TOL)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    torch.save({"lt": lt.cpu(), "piv": piv.cpu()}, save)
    p.close()
    for q in terms:
        q.close()
    print(json.dumps({"ms": times}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", default=os.path.join(ROOT, "gpytorch_b200", "lib", "parent", "libgpbbmm.so"))
    ap.add_argument("--lib-b", default=os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="where the children save their factors (default: a temporary directory)")
    ap.add_argument("--child", default=None)
    ap.add_argument("--save", default=None)
    args = ap.parse_args()
    if args.child:
        child(args.child, args.reps, args.save)
        return
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="pivchol_bench_")
    os.makedirs(args.out, exist_ok=True)
    print(json.dumps(card()), flush=True)
    libs = {"a": os.path.abspath(args.lib_a), "b": os.path.abspath(args.lib_b)}
    res = {s: {k: [] for k in libs} for s in SIZES}
    for r in range(args.rounds):
        for size in SIZES:
            for k in (("a", "b") if r % 2 == 0 else ("b", "a")):
                save = os.path.join(args.out, f"{size}_{k}.pt")
                env = dict(os.environ, GPBBMM_LIB=libs[k])
                out = subprocess.run([sys.executable, __file__, "--child", size, "--reps", str(args.reps), "--save", save],
                                     env=env, capture_output=True, text=True, check=True).stdout
                ms = json.loads(out.strip().splitlines()[-1])["ms"]
                res[size][k].append(statistics.median(ms))
                print(json.dumps({"round": r, "size": size, "lib": k, "ms": ms}), flush=True)
    import torch

    summary = {"ranks": {s: v[4] for s, v in SIZES.items()}, "libs": libs}
    for size in SIZES:
        fa, fb = torch.load(os.path.join(args.out, f"{size}_a.pt")), torch.load(os.path.join(args.out, f"{size}_b.pt"))
        summary[size] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in res[size].items()}
        summary[size]["identical"] = bool(torch.equal(fa["lt"], fb["lt"]) and torch.equal(fa["piv"], fb["piv"]))
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
