"""The SKI backend (csrc/ski.cu) at benchmark scale and at its launch edges, entry by entry against the chunked fp64 reference of
tests/ski_scale_oracle.py: the C5 geometry (N = 10^6, d = 3, 100^3 grid), grids over 64 nodes per dimension, more tiles and slabs
than resident CTAs, d = 4, crowded, empty and one-point tiles, points on both sides of every tile boundary.  Each case names the
paths it reaches; tests/test_ski_scale_host.py recomputes the launch geometry and checks that it reaches them.

Entrywise bound, derived, not tuned (u = 2^-24; first order; |.| entrywise; W the interpolation matrix of the fp32 points, S its
support pattern (ones on the 4^d nodes of a row), K = T_0 x ... x T_{d-1} >= 0, s the outputscale):
  * Weights.  The plan's 1-D weights and the reference's fp32 weights differ by at most 32 u each and the reference's product of d
    of them adds d - 1 roundings: 33 d u per product weight (tests/test_gpu_ski_predict.py).  The scatter and gather form the
    product weight with d - 1 more roundings of numbers <= 1 in magnitude: |W~ - W| <= 34 d u S.
  * Scatter, U = W^T V.  Node m accumulates its points' w v with fmaf in shared memory, one chain per (tile, part) block, then
    red.add's each block's sum into the grid in any order.  A term passes through at most (points touching m) + (blocks touching m)
    <= 2 m_node roundings, m_node = how many points have m among their nodes (a bincount of the reference's indices), plus the
    d - 1 of its weight: |U~ - U|_m <= u (2 m_node + d) (|W|^T |V|)_m + 34 d u (S^T |V|)_m.
  * Toeplitz factors.  T_i in fp32 from expf within eps_T = (3 R^2 + 10 R + 10) u relative, R = sqrt(5) max_i (G_i - 1) step_i / l
    (tests/test_gpu_ski_precond.py); the derivative factors l dT_i/dl take at most 6 more roundings: eps_T + 6 u.
  * Mode products, d of them, 3xTF32 mma.sync.  T = T_hi + T_lo and B = B_hi + B_lo with round-to-nearest tf32 parts leave
    residuals <= 2^-22 |T|, 2^-22 |B|, and the dropped T_lo B_lo is <= 2^-22 |T| |B|; tf32 products are exact in fp32.  The
    accumulation inside the tensor core aligns and truncates: counted conservatively as one 2^-22 loss per product of the output
    (G_i of them) plus one for the fp32 store: per mode (G_i + 4) 2^-22 of |T_i| |B|.  Over the d modes, with U~ as input:
      |Y~ - K U|  <=  K ( |U~ - U| + (sum_i (G_i + 4) 2^-22 + d eps_T) |W|^T |V| ) =: E_Y,    Y_mag = K |W|^T |V|.
  * gp_ski_grid_matmul (s K W^T V): the export multiplies by s, one rounding: s (E_Y + u Y_mag).
  * Gather, Plan.kmv.  out_r = sum_q w~_q Y~[node_q]: per lane an fmaf chain of 4^d / 8 terms and a 3-level shuffle tree, plus
    the weight's d - 1 roundings, <= 4^d + d in all; then s times the sum and fmaf(noise, v, .) in the finish kernel, 2 more:
      |out - s W K W^T V - noise V|  <=  s (|W| E_Y + (4^d + d) u |W| Y_mag + 34 d u S Y_mag) + 2 u (s |W| Y_mag + noise |V|).
  * gp_ski_interp_matmul (W C): the bound of tests/test_gpu_ski_predict.py, (4^d + 2 d) u |W| |C| + 33 d u S |C|; repeated calls
    bit-identical (no atomics).
  * Plan.bilinear_grad.  d/ds = <W^T L, K W^T R> and d/dl = (s / l) sum_i <W^T L, K_i W^T R> (K_i with l dT_i/dl in place of T_i),
    each a sweep of d mode products between two scatters, then an fp64 dot of fp32 products (exact) over M t terms.  With E_A,
    E_B the scatter bounds of A = W^T L and B = W^T R:  |<A~, K~_j B~> - <A, K_j B>| <= <E_A, K_j B_mag> + <A_mag, K_j E_B>
    + (sum_i (G_i + 4) 2^-22 + d eps_T (+ 6 u for j > 0)) <A_mag, K_j B_mag> + 1e-9 <A_mag, K_j B_mag> (fp64 sum of <= 10^8 terms).
    The reference is fp64 autograd through the chunked product with l and s as leaves.
  * Plan.ski_input_grad: the bound of tests/test_gpu_dkl.py with 2 max m_node (the scatter above) in place of n.  Rows with a
    coordinate within 1e-4 of the nodes where the one-hot cells begin are left out (the derivative jumps there).
Every case prints its largest err / bound per entry point; test_zz_report prints the largest over the cases with the card's name
and power limit.  Most of the file's time is the CPU reference: about 100 s in all on an H100 machine.
"""
import math
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu

import ski_scale_oracle as so  # noqa: E402
from dkl_oracle import ski_input_grad  # noqa: E402

U = 2.0 ** -24
NOISE = 0.1
RATIOS = {}


def _record(entry, case, err, bound):
    r = float((err / bound).max())
    RATIOS[(entry, case)] = max(r, RATIOS.get((entry, case), 0.0))
    print(f"\n{case:18s} {entry:12s} max err / bound = {r:.3e}")
    assert torch.isfinite(err).all() and r <= 1.0, (entry, case, r)


def _eps_t(case, lo, step):
    R = max(math.sqrt(5.0) * (g - 1) * s / case.ls for g, s in zip(case.sizes, step))
    return (3 * R * R + 10 * R + 10) * U


def _mode_eps(case):
    return sum((g + 4) * 2.0 ** -22 for g in case.sizes)


def _scatter_q(W, m, V, d):
    """(|W|^T |V|, the scatter bound / u): (2 m_node + d) |W|^T |V| + 34 d S^T |V|."""
    mag = W.wt(V.abs(), "abs")
    return mag, (2 * m + d).unsqueeze(1) * mag + 34 * d * W.wt(V.abs(), "support")


def _plan(dev, case, x, lo, step):
    from gpytorch_b200.engine import Plan

    p = Plan(x.to(dev)).set_ski(case.sizes, lo, step).set_hypers(case.kind, case.ls, case.outputscale, NOISE)
    assert p.info()["backend"] == "ski"
    return p


@pytest.fixture(scope="module")
def prepared():
    cache = {}

    def get(case):
        if case.name not in cache:
            cache.clear()                      # one case at a time: the C5 interpolation data is ~1 GB
            x, axes, lo, step = so.case_points(case)
            W = so.Interp(axes, x)
            cache[case.name] = (x, axes, lo, step, W, W.node_counts(), so.regular_axes(lo, step, case.sizes))
        return cache[case.name]

    return get


@pytest.mark.parametrize("case", so.CASES, ids=lambda c: c.name)
def test_products_entrywise(cuda_dev, prepared, case):
    x, axes, lo, step, W, m, reg = prepared(case)
    d, n, M, OS = len(case.sizes), case.n, W.M, case.outputscale
    g = torch.Generator().manual_seed(100 + case.seed)
    tmax = max(case.t)
    V = torch.randn(n, tmax, generator=g)
    V64 = V.double()
    cols = so.toeplitz_columns(case.kind, reg, case.ls)
    Umag, Q = _scatter_q(W, m, V64, d)
    Q += (_mode_eps(case) + d * _eps_t(case, lo, step)) / U * Umag
    Y, Ymag, EY = so.kuu(cols, torch.cat([W.wt(V64), Umag, U * Q], 1)).split(tmax, 1)
    out_ref = OS * W.w(Y)
    WY = W.w(torch.cat([EY, Ymag], 1), "abs")
    out_bnd = OS * (WY[:, :tmax] + (4 ** d + d) * U * WY[:, tmax:] + 34 * d * U * W.w(Ymag, "support")) + 2 * U * OS * WY[:, tmax:]
    grid_ref, grid_bnd = OS * Y, OS * (EY + U * Ymag)
    p = _plan(cuda_dev, case, x, lo, step)
    Vd = V.to(cuda_dev)
    for t in case.t:
        got = p.kmv(Vd[:, :t].contiguous()).double().cpu()
        _record("kmv", case.name, (got - out_ref[:, :t]).abs(), out_bnd[:, :t])
        got = p.kmv(Vd[:, :t].contiguous(), add_noise=True).double().cpu()
        _record("kmv+noise", case.name, (got - out_ref[:, :t] - NOISE * V64[:, :t]).abs(),
                out_bnd[:, :t] + 2 * U * NOISE * V64[:, :t].abs())
        got = p.ski_grid_matmul(Vd[:, :t].contiguous()).double().cpu()
        _record("grid_matmul", case.name, (got - grid_ref[:, :t]).abs(), grid_bnd[:, :t])
    del Y, Ymag, EY, WY, out_ref, out_bnd, grid_ref, grid_bnd
    Cg = torch.randn(M, tmax, generator=g)
    C64 = Cg.double()
    ref = W.w(C64)
    bnd = (4 ** d + 2 * d) * U * W.w(C64.abs(), "abs") + 33 * d * U * W.w(C64.abs(), "support")
    Cd = Cg.to(cuda_dev)
    for t in case.t:
        got = p.ski_interp_matmul(Cd[:, :t].contiguous())
        _record("interp", case.name, (got.double().cpu() - ref[:, :t]).abs(), bnd[:, :t])
        assert torch.equal(p.ski_interp_matmul(Cd[:, :t].contiguous()), got)
    p.close()


GRAD_CASES = [c for c in so.CASES if c.grads]


@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: c.name)
def test_bilinear_grad_entrywise(cuda_dev, prepared, case):
    x, axes, lo, step, W, m, reg = prepared(case)
    d, n, OS = len(case.sizes), case.n, case.outputscale
    g = torch.Generator().manual_seed(200 + case.seed)
    L, R = torch.randn(n, 2, generator=g), torch.randn(n, 2, generator=g)
    A, B = W.wt(L.double()), W.wt(R.double())
    Amag, QA = _scatter_q(W, m, L.double(), d)
    Bmag, QB = _scatter_q(W, m, R.double(), d)
    ls = torch.tensor(case.ls, dtype=torch.float64, requires_grad=True)
    osc = torch.tensor(OS, dtype=torch.float64, requires_grad=True)
    val = osc * (A * so.kuu(so.toeplitz_columns(case.kind, reg, ls), B)).sum()
    val.backward()
    base = _mode_eps(case) + d * _eps_t(case, lo, step)
    bounds = []
    for j in range(d + 1):
        cols = so.toeplitz_columns(case.kind, reg, case.ls, None if j == 0 else j - 1)
        KB = so.kuu([c.abs() for c in cols], torch.cat([Bmag, U * QB], 1))
        mag = float((Amag * KB[:, :2]).sum())
        bounds.append(U * float((QA * KB[:, :2]).sum()) + float((Amag * KB[:, 2:]).sum())
                      + (base + (6 * U if j else 0.0) + 1e-9) * mag)
    p = _plan(cuda_dev, case, x, lo, step)
    gl, go = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    p.close()
    _record("d/ds", case.name, torch.tensor(abs(go - osc.grad.item())), torch.tensor(bounds[0]))
    _record("d/dl", case.name, torch.tensor(abs(gl[0] - ls.grad.item())), torch.tensor(OS / case.ls * sum(bounds[1:])))


@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: c.name)
def test_input_grad_entrywise(cuda_dev, prepared, case):
    x, axes, lo, step, W, m, reg = prepared(case)
    d, n, t = len(case.sizes), case.n, 2
    g = torch.Generator().manual_seed(300 + case.seed)
    L, R = torch.randn(n, t, generator=g), torch.randn(n, t, generator=g)
    p = _plan(cuda_dev, case, x, lo, step)
    got = p.ski_input_grad(L.to(cuda_dev), R.to(cuda_dev)).double().cpu()
    p.close()
    ref, mag = ski_input_grad(case.kind, x.double(), reg, case.ls, case.outputscale, L.double(), R.double())
    k = 2 * float(m.max()) + 4 * sum(case.sizes) + 2 * 4 ** d + 2 * t + 16 + 20 * max(case.sizes)
    keep = torch.ones(n, dtype=torch.bool)
    for i, ax in enumerate(reg):
        for e in (float(ax[1]), float(ax[-2])):
            keep &= (x[:, i].double() - e).abs() >= 1e-4
    _record("input_grad", case.name, (got - ref).abs()[keep], (k * U * mag + 1e-30)[keep])


def test_zz_report_error_fraction_of_bound(cuda_dev):
    """Largest observed |engine - fp64| / bound per entry point over this module's cases (printed with -s)."""
    name = torch.cuda.get_device_name(0)
    smi = shutil.which("nvidia-smi")
    q = subprocess.run([smi, "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True) if smi else None
    name += f", power limit {(q.stdout.strip() if q else '') or 'unknown'}"
    entries = sorted({e for e, _ in RATIOS})
    for e in entries:
        r, c = max((v, cs) for (ee, cs), v in RATIOS.items() if ee == e)
        print(f"[{name}] ski {e:12s} max err / bound = {r:.3e} ({c})")
    for (e, c), r in sorted(RATIOS.items()):
        if c == "c5":
            print(f"[{name}] ski C5 {e:12s} err / bound = {r:.3e}")
    assert all(r <= 1.0 for r in RATIOS.values())
