"""Edges of the kernels that turn K.V into the MLL: SLQ (slq.cu), the preconditioner factorisation (pivchol.cu: gram / chol_small /
cinv / wsolve / probes), the mBCG bookkeeping (cg.cu) and Lanczos (lanczos.cu).  Every comparison is against a plain fp64
computation on the same fp32 values the device sees.

Stated tolerances:
  SLQ              |gpu - ref| <= 1e-9 (n/t_p) sum |z_j^2 log lambda_j| + 1e-12: two backward-stable fp64 eigen-solvers of
                   identical fp32 tridiagonals; a non-finite entry in a probe's leading block gives NaN
  preconditioner   log det P and P^-1 v within the first-order effect of the fp32 Gram chunks: |E_ab| <= gamma (|X|^T |X|)_ab,
                   gamma = 66 u (64-term fp32 chunks + 2 roundings of the 1/d scaling), X = S^-1/2 L, M = I + X^T X:
                   |d log det| <= gamma sum_ab |M^-1|_ab (|X|^T|X|)_ab ;  |d P^-1 v| <= gamma |S^-1/2 X M^-1|_2 | |X|^T|X| |b| |
                   (b = M^-1 X^T S^-1/2 v) + 2u |W|_F |W|_2 |v| (W stored in fp32) + k 2^-53 cond(M) |v| / s_min (fp64 part)
  probes           entrywise (k + 2) u (|L|^T |eps1| + s^1/2 |eps2|): k fp32 FMAs plus the fp32 square root of the noise
  mBCG             same iters / tridiag_size; tridiagonals rel 1e-4 (where the oracle's fp32 and fp64 runs agree to 1e-5); solves
                   per column rel 5e-4; resid per column max(1e-3 |o64|, 3 |o32 - o64|); after Krylov exhaustion (n = 7)
                   |gpu - o64| <= max(1e-3 |o64|, 3 |o32 - o64|) entrywise; TMAT outside the leading block exactly 0;
                   strided calls bit-identical
  Lanczos          Ritz values rel 1e-4 (full run, N = 40) / 1e-3 (low-rank operator) of the exact spectrum; Q^T Q = I to 1e-5;
                   |Q^T A Q - T| <= 1e-3
"""
import ctypes as C
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import kernels as ok, linalg as ol, mll as om  # noqa: E402

U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def Plan(cuda_dev):
    from gpytorch_b200.engine import Plan as P

    return P


@pytest.fixture(scope="module")
def lib(cuda_dev):
    from gpytorch_b200 import _lib

    return _lib


def _p(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


# ---------------------------------------------------------------------------------------------------------
# SLQ in isolation: fp32 tridiagonals built here, padded pitch, gp_slq_logdet through ctypes
# ---------------------------------------------------------------------------------------------------------
SLQ_N = 1000
SPECTRA = ["well", "spread", "clustered", "split", "indefinite", "mixed_sign"]


def make_tridiag(kind, J, nt, seed):
    """[nt, J] diagonals and [nt, J-1] off-diagonals (fp32)."""
    g = torch.Generator().manual_seed(seed)
    m = max(J - 1, 0)
    if kind == "clustered":
        return torch.ones(nt, J), torch.full((nt, m), 1e-9)
    if kind == "spread":   # eigenvalues ~ the diagonal: D^-1/2 T D^-1/2 = I + off-diagonals of 1e-3 or less
        d = 10.0 ** (torch.rand(nt, J, generator=g, dtype=torch.float64) * 10 - 6)
        e = 1e-3 * torch.rand(nt, m, generator=g, dtype=torch.float64) * (d[:, :-1] * d[:, 1:]).sqrt()
        return d.float(), e.float()
    if kind == "indefinite":
        return torch.rand(nt, J, generator=g) * 4 - 2, 0.1 + 0.9 * torch.rand(nt, m, generator=g)
    d = 2 + torch.rand(nt, J, generator=g)            # diagonally dominant: SPD
    e = 0.1 + 0.8 * torch.rand(nt, m, generator=g)
    if kind == "split" and m > 0:
        e[:, m // 2] = 0.0
    if kind == "mixed_sign":
        e = e * (torch.randint(0, 2, e.shape, generator=g) * 2 - 1)
    return d, e


def dense_tridiag(d, e):
    T = torch.diag_embed(d)
    if e.size(-1):
        T = T + torch.diag_embed(e, 1) + torch.diag_embed(e, -1)
    return T


def padded(T, ldt, pad_nan=True):
    """[nt, ldt, ldt] with T in the leading block, 1e30 around it and NaN on the padding's diagonal / sub-diagonal (the
    entries an over-running read of d / e would take first)."""
    nt, J, _ = T.shape
    out = torch.full((nt, ldt, ldt), 1e30)
    out[:, :J, :J] = T
    if pad_nan and ldt > J:
        idx = torch.arange(J, ldt)
        out[:, idx, idx] = float("nan")
        out[:, J, J - 1] = float("nan")
        out[:, J - 1, J] = float("nan")
    return out


def slq_raw(lib, plan, tmat_dev, nt, ldt, J, n):
    out = C.c_double()
    st = lib.load().gp_slq_logdet(plan._h, _p(tmat_dev), nt, ldt, J, n, C.byref(out))
    lib.check(st)
    return out.value


def slq_scale(T64, n):
    """(n / t_p) sum_i sum_j |z_ij^2 log lambda_ij| with the reference's masking."""
    evals, evecs = ol.tridiag_to_diag(T64)
    return float(n / T64.size(0) * (evecs[..., 0, :].pow(2) * evals.log().abs()).sum())


@pytest.fixture(scope="module")
def slq_plan(Plan, cuda_dev):
    p = Plan(torch.rand(16, 2).to(cuda_dev)).set_hypers("rbf", 1.0, 1.0, 0.1)
    yield p
    p.close()


@pytest.mark.parametrize("kind", SPECTRA)
@pytest.mark.parametrize("J,nt", [(1, 1), (2, 10), (3, 64), (20, 1), (20, 10), (64, 64), (255, 10), (256, 64), (256, 1)])
def test_slq_matches_fp64_eigh(lib, slq_plan, cuda_dev, kind, J, nt):
    if kind == "split" and J < 2:
        pytest.skip("no off-diagonal to split")
    d, e = make_tridiag(kind, J, nt, seed=J * 100 + nt)
    T = dense_tridiag(d, e)
    ldt = J + 7
    got = slq_raw(lib, slq_plan, padded(T, ldt).to(cuda_dev), nt, ldt, J, SLQ_N)
    T64 = T.double()
    ref = ol.slq_logdet(T64, SLQ_N)
    bound = 1e-9 * slq_scale(T64, SLQ_N) + 1e-12
    assert abs(got - ref) <= bound, (got, ref, bound)
    if kind == "indefinite":
        assert (torch.linalg.eigvalsh(T64) < 0).any()   # the masking is exercised


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("where", ["diag0", "diag3", "diag7", "off3"])
def test_slq_non_finite_tridiagonal_gives_nan(lib, slq_plan, cuda_dev, bad, where):
    # InvQuadLogdet.forward (oracle.linalg.inv_quad_logdet): NaN in any probe's tridiagonal -> NaN log-det; eigh of an Inf
    # entry gives NaN eigenvalues, so an Inf does the same
    J, nt, ldt = 8, 10, 15
    d, e = make_tridiag("well", J, nt, seed=3)
    T = dense_tridiag(d, e)
    clean = slq_raw(lib, slq_plan, padded(T, ldt).to(cuda_dev), nt, ldt, J, SLQ_N)
    assert math.isfinite(clean) and clean == pytest.approx(ol.slq_logdet(T.double(), SLQ_N), rel=1e-12)
    a = int(where[-1])
    Tb = T.clone()
    if where.startswith("diag"):
        Tb[4, a, a] = bad
    else:
        Tb[4, a + 1, a] = bad
        Tb[4, a, a + 1] = bad
    assert math.isnan(slq_raw(lib, slq_plan, padded(Tb, ldt).to(cuda_dev), nt, ldt, J, SLQ_N))


def test_slq_ignores_non_finite_padding(lib, slq_plan, cuda_dev):
    J, nt, ldt = 20, 64, 27
    d, e = make_tridiag("well", J, nt, seed=4)
    T = dense_tridiag(d, e)
    tight = slq_raw(lib, slq_plan, T.contiguous().to(cuda_dev), nt, J, J, SLQ_N)
    for pad in (padded(T, ldt, pad_nan=True), padded(T, ldt, pad_nan=False)):
        pad[:, J:, :] = float("nan")
        pad[:, :, J:] = float("inf")
        assert slq_raw(lib, slq_plan, pad.to(cuda_dev), nt, ldt, J, SLQ_N) == tight


@pytest.mark.parametrize("nt,ldt,J", [(4, 8, 0), (4, 264, 257), (4, 9, 10), (0, 8, 8), (65, 8, 8)])
def test_slq_rejects_bad_shapes_without_launching(lib, slq_plan, cuda_dev, nt, ldt, J):
    buf = torch.ones(max(nt, 1), ldt, ldt, device=cuda_dev)
    before = slq_plan.launches()
    with pytest.raises(RuntimeError, match="bad SLQ shape"):
        slq_raw(lib, slq_plan, buf, nt, ldt, J, SLQ_N)
    assert slq_plan.launches() == before


# ---------------------------------------------------------------------------------------------------------
# preconditioner factorisation: gp_precond_build / gp_precond_probes vs QR of [L; S^1/2] in fp64
# ---------------------------------------------------------------------------------------------------------
GAMMA_GRAM = 66 * U32


def precond_bounds(Lt32, noise, W32, v64):
    """First-order bounds (see the module header) for log det P and for every column of P^-1 v."""
    L = Lt32.double().t()                                   # [n, k]
    n, k = L.shape
    s = noise.double().reshape(-1) if torch.is_tensor(noise) else torch.full((n,), float(noise), dtype=torch.float64)
    X = L / s.sqrt().unsqueeze(-1)
    M = torch.eye(k, dtype=torch.float64) + X.t() @ X
    Minv = torch.linalg.inv(M)
    Gabs = X.abs().t() @ X.abs()
    s_min = s.min().item()
    cond = torch.linalg.cond(M).item()
    ld_bound = GAMMA_GRAM * (Minv.abs() * Gabs).sum().item() + 1e-13 * n * (1 + abs(math.log(s_min)))
    A = (X @ Minv) / s.sqrt().unsqueeze(-1)                 # S^-1/2 X M^-1
    b = Minv @ (X.t() @ (v64 / s.sqrt().unsqueeze(-1)))     # [k, c]
    W = W32.double() if torch.is_tensor(noise) else W32.double() / math.sqrt(float(noise))   # the factor of P^-1 = S^-1 - W W^T
    vn = v64.norm(dim=0)
    ap_bound = (GAMMA_GRAM * torch.linalg.matrix_norm(A, 2).item() * (Gabs @ b.abs()).norm(dim=0)
                + 2 * U32 * W.norm() * torch.linalg.matrix_norm(W, 2) * vn
                + k * 2.0 ** -53 * cond * vn / s_min)
    return ld_bound, ap_bound


def check_precond(p, lt, noise, seed):
    n = lt.size(1)
    W, logdet, st = p.precond_build(lt)
    assert st == 0
    Lt32 = lt.cpu()
    pre = ol.build_preconditioner(Lt32.double().t().contiguous(), noise.double() if torch.is_tensor(noise) else noise)
    v = torch.randn(n, 4, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    wd = W.double().cpu()
    if torch.is_tensor(noise):
        got = v / noise.double().unsqueeze(-1) - wd @ (wd.t() @ v)
    else:
        got = (v - wd @ (wd.t() @ v)) / noise
    ld_bound, ap_bound = precond_bounds(Lt32, noise, W.cpu(), v)
    assert abs(logdet - pre.logdet) <= ld_bound, (logdet, pre.logdet, ld_bound)
    err = (got - pre.apply(v)).norm(dim=0)
    assert torch.all(err <= ap_bound), (err, ap_bound)
    return W


def _noise32(x):
    return float(torch.tensor(x, dtype=torch.float32))


@pytest.mark.parametrize("k,n,noise", [
    (1, 2, 0.1), (1, 4097, 1e-4), (63, 1000, 10.0), (64, 65, 0.1), (64, 4097, 1e-4), (65, 1000, 1e-4), (65, 66, 10.0),
    (127, 4097, 0.1), (128, 129, 1e-4), (128, 1000, 0.1), (128, 4097, 10.0), (128, 4097, 1e-4)])
def test_precond_dense_factor_matches_qr(Plan, cuda_dev, k, n, noise):
    """A dense random L isolates the factorisation (Gram tiles, their mirror, Cholesky, C^-1, W) from the pivoting."""
    g = torch.Generator().manual_seed(k * 7 + n)
    lt = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(cuda_dev)
    p = Plan(torch.rand(n, 2, generator=g).to(cuda_dev)).set_hypers("rbf", 1.0, 1.0, noise)
    check_precond(p, lt, _noise32(noise), seed=k + n)
    p.close()


@pytest.mark.parametrize("k,n", [(65, 1000), (128, 4097)])
def test_precond_per_row_noise_matches_qr(Plan, cuda_dev, k, n):
    g = torch.Generator().manual_seed(k + n)
    lt = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(cuda_dev)
    dvec = (10.0 ** (-3 * torch.rand(n, generator=g))).float()           # 1e-3 ... 1
    p = Plan(torch.rand(n, 2, generator=g).to(cuda_dev)).set_hypers("rbf", 1.0, 1.0, 0.5)
    p.set_noise_diag(dvec.to(cuda_dev))
    check_precond(p, lt, dvec, seed=n)
    p.close()


@pytest.mark.parametrize("noise", [1e-4, 10.0])
def test_precond_engine_factor_small_noise(Plan, cuda_dev, noise):
    """The engine's own pivoted-Cholesky factor at the rank limit (k = 128): near-dependent columns, 1/sigma^2 amplification."""
    n = 4097
    x, _ = om.synthetic_problem(n, 6, 2, torch.float32)
    p = Plan(x.to(cuda_dev)).set_hypers("matern52", 0.8, 1.0, noise)
    lt, _, _ = p.pivoted_cholesky(128, 0.0)
    assert lt.size(0) == 128
    W = check_precond(p, lt, _noise32(noise), seed=1)
    # probes at the rank limit, entrywise against z = L eps1 + sigma eps2
    L64 = lt.double().cpu().t()
    s = _noise32(noise)
    for tp in (1, 15, 16):
        eps1, eps2, _ = om.make_probe_noise(n, 128, tp, 5 + tp)
        z = p.precond_probes(lt, eps1.to(cuda_dev), eps2.to(cuda_dev)).double().cpu()
        ref = L64 @ eps1.double() + math.sqrt(s) * eps2.double()
        bound = (128 + 2) * U32 * (L64.abs() @ eps1.double().abs() + math.sqrt(s) * eps2.double().abs())
        assert torch.all((z - ref).abs() <= bound), tp
    p.close()


def test_precond_rejections(Plan, cuda_dev):
    n = 300
    x = torch.rand(n, 2).to(cuda_dev)
    p = Plan(x).set_hypers("rbf", 1.0, 1.0, 0.1)
    with pytest.raises(RuntimeError, match="not in"):
        p.precond_build(torch.empty(0, n, device=cuda_dev))
    with pytest.raises(RuntimeError, match="not in"):
        p.precond_build(torch.randn(129, n, device=cuda_dev))
    p.set_hypers("rbf", 1.0, 1.0, 0.0)
    with pytest.raises(RuntimeError, match="noise > 0"):
        p.precond_build(torch.randn(4, n, device=cuda_dev))
    p.close()


# ---------------------------------------------------------------------------------------------------------
# mBCG bookkeeping vs oracle.linalg.linear_cg
# ---------------------------------------------------------------------------------------------------------
def mbcg_raw(lib, p, rhs, t, n_tridiag, tol, max_iter, mti, W=None, ldr=None, lds=None, tmat_fill=float("nan")):
    """gp_mbcg with explicit strides; TMAT is pre-filled with `tmat_fill` (the call must zero it)."""
    n = rhs.size(0)
    ldr = ldr or rhs.stride(0)
    lds = lds or t
    solves = torch.full((n, lds), -7.0, device=rhs.device)
    tmat = torch.full((max(n_tridiag, 1), mti, mti), tmat_fill, device=rhs.device)
    it, js = C.c_int(), C.c_int()
    resid = (C.c_float * 16)()
    st = lib.load().gp_mbcg(p._h, _p(rhs), ldr, t, n_tridiag, float(tol), int(max_iter), int(mti), _p(W),
                            0 if W is None else W.size(1), _p(solves), lds, _p(tmat), C.byref(it), C.byref(js), resid)
    lib.check(st, warn=False)
    return solves, tmat, it.value, js.value, [resid[i] for i in range(t)]


def mbcg_problem(n, t, zero_col, seed):
    x, _ = om.synthetic_problem(n, 10, seed, torch.float32)
    g = torch.Generator().manual_seed(seed + 1)
    rhs = torch.randn(n, t, generator=g, dtype=torch.float64)
    rhs = rhs / rhs.norm(dim=0) * torch.logspace(-6, 6, t, dtype=torch.float64)   # column norms 1e-6 ... 1e6
    if zero_col is not None:
        rhs[:, zero_col] = 0.0
    return x, rhs.float()


def oracle_cg(A64, rhs32, n_tridiag, tol, max_iter, mti, pre64=None, pre32=None):
    """fp64 and fp32 runs of the oracle on the same fp32 right-hand side."""
    out = []
    for A, rhs, pre in ((A64, rhs32.double(), pre64), (A64.float(), rhs32, pre32)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            r = ol.linear_cg(lambda v: A @ v, rhs, n_tridiag=n_tridiag, tolerance=tol, max_iter=max_iter,
                             max_tridiag_iter=mti, preconditioner=None if pre is None else pre.apply, return_info=True)
        out.append((r[0], r[1] if n_tridiag else None, r[-1]))
    return out


def close(gpu, o64, o32, floor=1e-4):
    """|gpu - o64| <= max(floor |o64|, 3 |o32 - o64|) entrywise: where the oracle's fp32 and fp64 runs agree this is a plain
    relative bound; past a converged column or an exhausted Krylov space they part ways and the gpu must stay as close to
    fp64 as the reference's own fp32 run."""
    gpu, o64, o32 = gpu.double().cpu(), o64.double(), o32.double()
    return bool(torch.all((gpu - o64).abs() <= torch.maximum(floor * o64.abs(), 3 * (o32 - o64).abs())))


def colrel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm(dim=0) / b.norm(dim=0).clamp_min(1e-300))


# (backend, precond rank or 0, t, n_tridiag, max_tridiag_iter, max_iter, n, zero column).  sigma^2 = 1, RBF l = 1, d = 10: without a
# preconditioner the fp32 and fp64 recurrences part ways once a column reaches a ~1e-5 residual (after ~10 steps here), so the
# runs of 20 and 37 steps use a rank-100 preconditioner, under which the oracle's fp32 and fp64 tridiagonals agree to ~1e-6
MBCG_CASES = [
    ("tcgen05", 0, 1, 1, 1, 1000, 64, None),
    ("simt", 16, 2, 0, 5, 5, 1001, None),
    ("tcgen05", 32, 15, 15, 20, 1000, 4099, 3),
    ("simt", 100, 16, 1, 37, 1000, 1001, 9),
    ("tcgen05", 64, 1, 1, 5, 5, 4099, None),
    ("simt", 0, 15, 0, 20, 1000, 64, 0),
    ("tcgen05", 100, 2, 2, 37, 1000, 4099, None),
    ("simt", 100, 16, 16, 20, 1000, 1001, None),
]


@pytest.mark.parametrize("backend,rank,t,nt,mti,max_iter,n,zero_col", MBCG_CASES)
def test_mbcg_bookkeeping_matches_oracle(Plan, lib, cuda_dev, backend, rank, t, nt, mti, max_iter, n, zero_col):
    noise = 1.0
    x, rhs = mbcg_problem(n, t, zero_col, seed=n + t)
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 1.0, 1.0, True) + noise * torch.eye(n, dtype=torch.float64)
    p = Plan(x.to(cuda_dev), backend=backend).set_hypers("rbf", 1.0, 1.0, noise)
    assert p.info()["backend"] == backend
    W, pre64, pre32 = None, None, None
    if rank:
        lt, _, _ = p.pivoted_cholesky(rank, 0.0)
        W, _, _ = p.precond_build(lt)
        L32 = lt.cpu().t().contiguous()
        pre64, pre32 = ol.build_preconditioner(L32.double(), noise), ol.build_preconditioner(L32, noise)
    (s64, t64, i64), (s32, t32, i32) = oracle_cg(A, rhs, nt, 1.0, max_iter, mti, pre64, pre32)
    assert i32.iters == i64.iters          # precondition: the oracle's own fp32 and fp64 runs take the same number of steps
    sg, tg, iters, J, resid = mbcg_raw(lib, p, rhs.to(cuda_dev), t, nt, 1.0, max_iter, mti, W)
    assert iters == i64.iters
    nz = rhs.norm(dim=0) > 0
    assert torch.all(colrel(sg, s64)[nz] < 5e-4), colrel(sg, s64)
    if zero_col is not None:
        assert torch.all(sg[:, zero_col] == 0)
    assert close(torch.tensor(resid), i64.residual_norms, i32.residual_norms, 1e-3), (resid, i64.residual_norms)
    if nt:
        assert t32.shape == t64.shape                      # precondition, as above
        assert J == t64.size(-1) <= min(mti, n)             # the off-diagonal stop (< 1e-6) may end it earlier
        for c in range(nt):
            assert rel(t32[c], t64[c]) < 1e-5, c           # precondition: the oracle's fp32 and fp64 tridiagonals agree
            assert rel(tg[c, :J, :J], t64[c]) < 1e-4, c
        # everything outside the leading J x J block was zeroed by the call (TMAT was NaN-filled before it)
        outside = torch.ones(mti, mti, dtype=torch.bool)
        outside[:J, :J] = False
        assert torch.all(tg[:, outside.to(cuda_dev)] == 0)
    else:
        assert J == 0
    p.close()


# (without a preconditioner the last step before exhaustion runs on a ~1e-4 residual and its fp32 entries are off by ~3e-2:
# no entrywise bound applies there, so the exhausting run uses the rank-4 preconditioner)
@pytest.mark.parametrize("backend,rank", [("simt", 4)])
def test_mbcg_krylov_exhausted_small_n(Plan, lib, cuda_dev, backend, rank):
    """n = 7 < max_tridiag_iter: the tridiagonal ends by step min(max_tridiag_iter, N) = 7 inside a 20-pitch TMAT, and CG keeps
    iterating on a rounding-level residual (where fp32 and fp64 runs part ways) until the tolerance test at k = 10."""
    n, t, nt, mti = 7, 16, 16, 20
    x, rhs = mbcg_problem(n, t, None, seed=7)
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 1.0, 1.0, True) + torch.eye(n, dtype=torch.float64)
    p = Plan(x.to(cuda_dev), backend=backend).set_hypers("rbf", 1.0, 1.0, 1.0)
    W, pre64, pre32 = None, None, None
    if rank:
        lt, _, _ = p.pivoted_cholesky(rank, 0.0)
        W, _, _ = p.precond_build(lt)
        L32 = lt.cpu().t().contiguous()
        pre64, pre32 = ol.build_preconditioner(L32.double(), 1.0), ol.build_preconditioner(L32, 1.0)
    (s64, t64, i64), (s32, t32, i32) = oracle_cg(A, rhs, nt, 1.0, 1000, mti, pre64, pre32)
    sg, tg, iters, J, _ = mbcg_raw(lib, p, rhs.to(cuda_dev), t, nt, 1.0, 1000, mti, W)
    assert iters == i64.iters == i32.iters
    # with the preconditioner the space is exhausted before step 7 and the off-diagonal stop (< 1e-6) ends the tridiagonal
    # there; whether it fires one step earlier or later depends on rounding, so fp32 and fp64 may differ by one step
    assert J in (t64.size(-1), t32.size(-1)) and J <= n
    m = min(J, t64.size(-1), t32.size(-1))
    # the last steps before exhaustion run on residuals of ~1e-3 of the start: fp32 rounding is amplified by as much
    assert close(tg[:, :m, :m], t64[:, :m, :m], t32[:, :m, :m], 1e-3), (tg[:, :m, :m].cpu() - t64[:, :m, :m]).abs().max()
    assert torch.all(colrel(sg, s64) < 5e-4) or close(sg, s64, s32)
    outside = torch.ones(mti, mti, dtype=torch.bool)
    outside[:J, :J] = False
    assert torch.all(tg[:, outside.to(cuda_dev)] == 0)
    p.close()


def test_mbcg_tridiagonal_stops_on_small_off_diagonal(Plan, lib, cuda_dev):
    """linear_cg stops updating the tridiagonals once every off-diagonal of the step is below 1e-6.  A zero probe column has
    alpha = beta = 0, so its second off-diagonal is exactly 0: the tridiagonal ends at 2 x 2 = I in fp32 and fp64 alike."""
    n, t, nt, mti = 1001, 3, 1, 20
    x, rhs = mbcg_problem(n, t, 0, seed=11)
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 1.0, 1.0, True) + torch.eye(n, dtype=torch.float64)
    (s64, t64, i64), _ = oracle_cg(A, rhs, nt, 1.0, 1000, mti)
    assert t64.shape == (1, 2, 2) and torch.equal(t64[0], torch.eye(2, dtype=torch.float64))
    for backend in ("tcgen05", "simt"):
        p = Plan(x.to(cuda_dev), backend=backend).set_hypers("rbf", 1.0, 1.0, 1.0)
        sg, tg, iters, J, _ = mbcg_raw(lib, p, rhs.to(cuda_dev), t, nt, 1.0, 1000, mti)
        assert J == 2 and iters == i64.iters
        assert torch.equal(tg[0, :2, :2].cpu(), torch.eye(2)) and torch.all(tg[0, 2:, :] == 0) and torch.all(tg[0, :, 2:] == 0)
        assert torch.all(colrel(sg[:, 1:], s64[:, 1:]) < 5e-4)
        p.close()


@pytest.mark.parametrize("backend,rank", [("tcgen05", 16), ("simt", 0)])
def test_mbcg_and_kmv_strides_leave_padding_and_bits(Plan, lib, cuda_dev, backend, rank):
    n, t, nt = 1001, 5, 3
    x, rhs = mbcg_problem(n, t, None, seed=21)
    p = Plan(x.to(cuda_dev), backend=backend).set_hypers("rbf", 1.0, 1.0, 1.0)
    W = None
    if rank:
        lt, _, _ = p.pivoted_cholesky(rank, 0.0)
        W, _, _ = p.precond_build(lt)
    rd = rhs.to(cuda_dev)
    s0, t0, i0, j0, r0 = mbcg_raw(lib, p, rd.contiguous(), t, nt, 1.0, 1000, 20, W)
    ldr, lds = t + 3, t + 6
    big = torch.full((n, ldr), float("nan"), device=cuda_dev)
    big[:, :t] = rd
    s1, t1, i1, j1, r1 = mbcg_raw(lib, p, big, t, nt, 1.0, 1000, 20, W, ldr=ldr, lds=lds)
    assert torch.isnan(big[:, t:]).all() and torch.equal(big[:, :t], rd)
    assert torch.all(s1[:, t:] == -7.0)                       # the solve padding is untouched
    assert torch.equal(s1[:, :t], s0[:, :t]) and torch.equal(t1, t0) and (i1, j1, r1) == (i0, j0, r0)
    # gp_kmv: two 16-column chunks, NaN in the input padding, a sentinel in the output padding
    tv = 20
    v = torch.randn(n, tv, generator=torch.Generator().manual_seed(2)).to(cuda_dev)
    o0 = p.kmv(v, add_noise=True)
    ldv, ldo = tv + 5, tv + 3
    vb = torch.full((n, ldv), float("nan"), device=cuda_dev)
    vb[:, :tv] = v
    ob = torch.full((n, ldo), 123.0, device=cuda_dev)
    lib.check(lib.load().gp_kmv(p._h, _p(vb), ldv, tv, _p(ob), ldo, 1))
    torch.cuda.synchronize()
    assert torch.all(ob[:, tv:] == 123.0) and torch.equal(ob[:, :tv], o0)
    p.close()


# ---------------------------------------------------------------------------------------------------------
# Lanczos vs oracle.linalg.lanczos_tridiag
# ---------------------------------------------------------------------------------------------------------
def test_lanczos_max_iter_beyond_n(Plan, cuda_dev):
    n, noise = 40, 0.5
    x, _ = om.synthetic_problem(n, 3, 4, torch.float32)
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 0.7, 1.0, True) + noise * torch.eye(n, dtype=torch.float64)
    init = torch.randn(n, generator=torch.Generator().manual_seed(1))
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", 0.7, 1.0, noise)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        Q, T = p.lanczos(init.to(cuda_dev), 60)
    J = T.size(0)
    assert 1 <= J <= n and Q.shape == (n, J)
    ritz = torch.linalg.eigvalsh(T.double().cpu())
    ev = torch.linalg.eigvalsh(A)
    nearest = (ritz.unsqueeze(-1) - ev.unsqueeze(0)).abs().min(-1)
    assert torch.all(nearest.values <= 1e-4 * ev[nearest.indices]), (ritz, ev)
    if J == n:
        assert torch.allclose(ritz, ev, rtol=1e-4, atol=0)
    p.close()


@pytest.mark.parametrize("max_iter", [1, 2])
def test_lanczos_one_and_two_steps(Plan, cuda_dev, max_iter):
    n = 1500
    x, _ = om.synthetic_problem(n, 4, 0, torch.float32)
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 0.6, 1.0, True) + 0.1 * torch.eye(n, dtype=torch.float64)
    init = torch.randn(n, 1, dtype=torch.float64, generator=torch.Generator().manual_seed(9)).float()
    Qo, To = ol.lanczos_tridiag(lambda v: A @ v, max_iter, init.double())
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", 0.6, 1.0, 0.1)
    Q, T = p.lanczos(init[:, 0].to(cuda_dev), max_iter)
    assert Q.shape == (n, max_iter) and T.shape == To[0].shape == (max_iter, max_iter)
    # fp32 products of an operator of norm ~|A|: entries within 1e-5 |A|
    assert (T.double().cpu() - To[0]).abs().max() <= 1e-5 * To[0].abs().max()
    assert (Q.double().cpu() - Qo[0]).abs().max() < 1e-5
    p.close()


def test_lanczos_low_rank_operator_exhausts_krylov_space(Plan, cuda_dev):
    """4 distinct points repeated 250 times: K + sigma^2 I has at most 5 distinct eigenvalues, so the Krylov space is
    exhausted after 5 steps and the further steps run on a rounding-level residual."""
    reps, noise, os_ = 250, 0.1, 0.2
    pts = torch.tensor([[0.1, 0.2], [0.7, 0.3], [0.4, 0.9], [0.95, 0.8]])
    x = pts.repeat(reps, 1)
    n = x.size(0)
    K4 = ok.kernel_matrix("rbf", pts.double(), pts.double(), 0.5, os_, True)
    exact = torch.cat([torch.linalg.eigvalsh(reps * K4) + noise, torch.tensor([noise], dtype=torch.float64)])
    A = ok.kernel_matrix("rbf", x.double(), x.double(), 0.5, os_, True) + noise * torch.eye(n, dtype=torch.float64)
    init = torch.randn(n, generator=torch.Generator().manual_seed(3))
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", 0.5, os_, noise)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        Q, T = p.lanczos(init.to(cuda_dev), 12)
    Qd, Td = Q.double().cpu(), T.double().cpu()
    ritz = torch.linalg.eigvalsh(Td)
    d = ((ritz.unsqueeze(-1) - exact.unsqueeze(0)).abs() / exact.unsqueeze(0)).min(-1).values
    assert torch.all(d <= 1e-3), (ritz, exact)
    assert (Qd.t() @ Qd - torch.eye(Qd.size(1), dtype=torch.float64)).abs().max() < 1e-5
    assert (Qd.t() @ A @ Qd - Td).abs().max() < 1e-3
    p.close()
