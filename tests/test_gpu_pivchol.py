"""The pivoted Cholesky (csrc/pivchol.cu) on its own terms (run with -m gpu on an H100): every factor goes through the fp64
checker of tests/pivchol_oracle.py -- structure, backward identity on the pivot columns, greedy choice, ties by position and the
stop rule -- at rows beyond the resident grid, at position ties, at small and ragged n, at the stop rule and NaN inputs, for the
plain entry sources and a kernel sum, and at ranks past the column cache (rank 200)."""
import math
import warnings

import pytest
import torch

import pivchol_oracle as po
import ppoly_oracle as ppo

pytestmark = pytest.mark.gpu

PCP_THREADS = 384
MAX_CTAS_PER_SM = 5     # 2048 threads per SM / 384


@pytest.fixture(scope="module")
def Plan(cuda_dev):
    from gpytorch_b200.engine import Plan as P

    return P


def _host_gb():
    try:
        import psutil

        return psutil.virtual_memory().available / 1e9
    except Exception:
        return 0.0


def _grid_stride_n(cuda_dev):
    """n = 2 * 5 * 384 * SMs + 1: whatever occupancy the runtime picks, every thread of the grid owns at least two rows."""
    props = torch.cuda.get_device_properties(cuda_dev)
    assert props.max_threads_per_multi_processor // PCP_THREADS <= MAX_CTAS_PER_SM
    return 2 * MAX_CTAS_PER_SM * PCP_THREADS * props.multi_processor_count + 1


def _stationary(kind, r2, alpha=None):
    r = r2.sqrt()
    if kind == "rbf":
        return torch.exp(-0.5 * r2)
    if kind == "matern12":
        return torch.exp(-r)
    if kind == "matern32":
        return (1 + math.sqrt(3) * r) * torch.exp(-math.sqrt(3) * r)
    if kind == "matern52":
        return (1 + math.sqrt(5) * r + 5.0 / 3.0 * r2) * torch.exp(-math.sqrt(5) * r)
    if kind == "rq":
        return (1 + r2 / (2 * alpha)) ** (-alpha)
    raise ValueError(kind)


def _col_fn(kind, x, ls, S, alpha=None, power=None, offset=None, q=None):
    """col(i) -> K[:, i] in fp64 from direct differences of the fp32 inputs (held in fp64)."""
    x = x.double().cpu()

    def col(i):
        if kind == "poly":
            return S * (x @ x[i] + offset) ** power
        if kind == "ppoly":
            return ppo.kernel(x, x[i:i + 1], ls, q, S)[:, 0]
        d = (x - x[i]) / ls
        return S * _stationary(kind, (d * d).sum(-1), alpha)
    return col


def _eps(kind, x, ls, S, power=None, offset=None):
    d = x.size(1)
    if kind == "poly":
        a = float((x.double() * x.double()).sum(-1).max()) + offset
        return po.generic_entry_bound(S * a ** power, d, power * a)
    span = float((x.double().amax(0) - x.double().amin(0)).pow(2).sum()) / (ls * ls)
    return po.generic_entry_bound(S, d, 0.5 * span)


def _run(p, rank, tol):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        lt, piv, st = p.pivoted_cholesky(rank, tol)
    torch.cuda.synchronize()
    return lt, piv, st


def _check(lt, piv, st, diag, col, tol, eps, rank):
    return po.check_factor(lt, piv, lt.size(0), st, diag, col, tol, eps, rank)


# ---------------------------------------------------------------------------------------------------------
# rows beyond the resident grid
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,rank", [("rbf", 15), ("rbf", 60), ("rbf", 100), ("rbf", 128), ("matern52", 60)])
def test_grid_stride_rows(Plan, cuda_dev, kind, rank):
    if _host_gb() < 6:
        pytest.skip("the fp64 pivot columns of n = 5e5 rows need ~1 GB of host memory and the checker twice that")
    n = _grid_stride_n(cuda_dev)
    d, ls, S = 3, 0.35, 1.3
    x = torch.rand(n, d, generator=torch.Generator().manual_seed(rank))
    p = Plan(x.to(cuda_dev)).set_hypers(kind, ls, S, 0.1)
    lt, piv, st = _run(p, rank, 0.0)
    p.close()
    assert st == 0 and lt.size(0) == rank
    # pivots in the later passes of the grid were chosen (rows owned as a thread's second or third row)
    assert int((piv.cpu() >= n // 2).sum()) >= 1
    _check(lt, piv, st, torch.full((n,), float(torch.tensor(S)), dtype=torch.float64), _col_fn(kind, x, ls, S), 0.0,
           _eps(kind, x, ls, S), rank)


def test_grid_stride_kernel_sum(Plan, cuda_dev):
    if _host_gb() < 6:
        pytest.skip("the fp64 pivot columns of n = 5e5 rows need ~1 GB of host memory")
    n, rank = _grid_stride_n(cuda_dev), 40
    x = torch.rand(n, 3, generator=torch.Generator().manual_seed(8))
    xd = x.to(cuda_dev)
    pa = Plan(xd).set_hypers("rbf", 0.4, 1.2, 0.0)
    pb = Plan(xd).set_hypers("matern32", 0.9, 0.7, 0.0)
    ps = Plan(xd).set_sum([pa, pb]).set_hypers("rbf", [1.0], 1.0, 0.1)
    lt, piv, st = _run(ps, rank, 0.0)
    ps.close(), pa.close(), pb.close()
    ca, cb = _col_fn("rbf", x, 0.4, 1.2), _col_fn("matern32", x, 0.9, 0.7)
    diag = torch.full((n,), float(torch.tensor(1.2) + torch.tensor(0.7)), dtype=torch.float64)
    eps = _eps("rbf", x, 0.4, 1.2) + _eps("matern32", x, 0.9, 0.7) + 2 * po.U32 * 1.9
    assert st == 0 and lt.size(0) == rank
    _check(lt, piv, st, diag, lambda i: ca(i) + cb(i), 0.0, eps, rank)


# ---------------------------------------------------------------------------------------------------------
# position ties: bit-identical duplicate rows, decided by the earliest position of the running permutation
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("big", [False, True])
def test_position_ties(Plan, cuda_dev, big):
    """Small n: every point 3 times at scattered indices.  Grid-stride n: 200 points, each about n / 200 times, so that the low
    rows the first swaps move to later positions are copies of later pivots (with n / 3 points they almost never are)."""
    if big and _host_gb() < 6:
        pytest.skip("the fp64 pivot columns of n = 5e5 rows need ~1 GB of host memory")
    n = _grid_stride_n(cuda_dev) if big else 3000
    D, rank, ls = (200 if big else n // 3), 60, 0.3
    g = torch.Generator().manual_seed(21)
    base = torch.rand(D, 3, generator=g)
    x = base[torch.randperm(n, generator=g) % D].contiguous()     # scattered copies of D points
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", ls, 1.0, 0.1)
    lt, piv, st = _run(p, rank, 0.0)
    p.close()
    assert st == 0 and lt.size(0) == rank < D
    out = _check(lt, piv, st, torch.ones(n, dtype=torch.float64), _col_fn("rbf", x, ls, 1.0), 0.0, _eps("rbf", x, ls, 1.0), rank)
    assert out["ties"] >= rank // 2
    assert out["ties_by_position"] >= 1, "no tie was decided by a position that differs from the index order"


# ---------------------------------------------------------------------------------------------------------
# small and ragged n
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 383, 384, 385, 767])
def test_small_and_ragged_n(Plan, cuda_dev, n):
    x = torch.rand(n, 2, generator=torch.Generator().manual_seed(n)) * 4
    ls = 0.5
    col, eps = _col_fn("matern32", x, ls, 1.0), _eps("matern32", x, ls, 1.0)
    p = Plan(x.to(cuda_dev)).set_hypers("matern32", ls, 1.0, 0.1)
    for rank in sorted({1, max(n - 1, 1), n, n + 5}):
        lt, piv, st = _run(p, rank, 0.0)
        assert st in (0, po.GP_W_PIVCHOL_NAN)
        assert 1 <= lt.size(0) <= min(rank, n)
        if st == 0:
            assert lt.size(0) == min(rank, n)
        assert bool(torch.isfinite(lt).all())
        _check(lt, piv, st, torch.ones(n, dtype=torch.float64), col, 0.0, eps, min(rank, n))
    p.close()


# ---------------------------------------------------------------------------------------------------------
# stop rule and NaN
# ---------------------------------------------------------------------------------------------------------
def test_stop_rule_tolerance_sweep(Plan, cuda_dev):
    n, ls = 2000, 1.2
    x = torch.rand(n, 3, generator=torch.Generator().manual_seed(3))
    col, eps = _col_fn("rbf", x, ls, 1.0), _eps("rbf", x, ls, 1.0)
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", ls, 1.0, 0.1)
    decided, ranks = 0, []
    for tol in (1.0, 0.3, 0.1, 3e-2, 1e-2, 1e-3):
        lt, piv, st = _run(p, 100, tol)
        assert st == 0
        out = _check(lt, piv, st, torch.ones(n, dtype=torch.float64), col, tol, eps, 100)
        decided += out["stop_checked"] and lt.size(0) < 100
        ranks.append(lt.size(0))
    p.close()
    assert ranks == sorted(ranks) and ranks[0] < ranks[-1]
    assert decided >= 1, "no tolerance stopped the factor at a step the fp32 uncertainty decides"


def test_nan_beyond_the_first_pass_and_at_the_first_pivot(Plan, cuda_dev):
    n = _grid_stride_n(cuda_dev)
    x = torch.rand(n, 3, generator=torch.Generator().manual_seed(5))
    for row in (n - 2, 0):      # a row of a later grid pass; the first pivot (constant diagonal: row 0)
        xb = x.clone()
        xb[row, 1] = float("nan")
        p = Plan(xb.to(cuda_dev)).set_hypers("rbf", 0.5, 1.0, 0.1)
        lt, piv, st = _run(p, 30, 0.0)
        p.close()
        assert st == po.GP_W_PIVCHOL_NAN
        assert lt.size(0) == 1 and int(piv[0]) == 0


def test_rank_above_the_numerical_rank(Plan, cuda_dev):
    n = 1500
    x = torch.rand(n, 1, generator=torch.Generator().manual_seed(9))     # 1-D, long lengthscale: numerical rank ~ 10
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", 2.0, 1.0, 0.1)
    lt, piv, st = _run(p, 120, 0.0)
    p.close()
    assert st in (0, po.GP_W_PIVCHOL_NAN)
    if st == 0:
        assert lt.size(0) == 120
    assert bool(torch.isfinite(lt).all())
    _check(lt, piv, st, torch.ones(n, dtype=torch.float64), _col_fn("rbf", x, 2.0, 1.0), 0.0, _eps("rbf", x, 2.0, 1.0), 120)


# ---------------------------------------------------------------------------------------------------------
# entry sources (several CTAs each)
# ---------------------------------------------------------------------------------------------------------
PLAIN = [("rbf", {}), ("matern12", {}), ("matern32", {}), ("matern52", {}), ("rq", {"alpha": 0.7}),
         ("poly", {"power": 3, "offset": 0.5}), ("ppoly", {"q": 2})]


@pytest.mark.parametrize("kind,kw", PLAIN, ids=[k for k, _ in PLAIN])
def test_plain_entry_sources(Plan, cuda_dev, kind, kw):
    n, d, ls, S, rank = 4000, 3, 0.4, 1.1, 50
    x = torch.rand(n, d, generator=torch.Generator().manual_seed(31))
    xd = x.to(cuda_dev)
    if kind == "rq":
        p = Plan(xd).set_hypers_rq(ls, kw["alpha"], S, 0.1)
    elif kind == "poly":
        p = Plan(xd).set_hypers_poly(kw["power"], kw["offset"], S, 0.1)
    elif kind == "ppoly":
        ls = 0.6
        p = Plan(xd).set_hypers_pp(kw["q"], ls, S, 0.1)
    else:
        p = Plan(xd).set_hypers(kind, ls, S, 0.1)
    lt, piv, st = _run(p, rank, 0.0)
    if kind == "poly":   # the diagonal S (|x|^2 + c)^p varies from row to row: the device's own fp32 diagonal
        diag = p.diag().double().cpu()
    else:
        diag = torch.full((n,), float(torch.tensor(S)), dtype=torch.float64)
    p.close()
    # a polynomial kernel of degree 3 in 3 inputs has rank 20: its factor may end once no residual is positive, with status 0
    assert st == 0
    assert lt.size(0) == rank or (kind == "poly" and lt.size(0) >= 20)
    col = _col_fn(kind, x, ls, S, alpha=kw.get("alpha"), power=kw.get("power"), offset=kw.get("offset"), q=kw.get("q"))
    _check(lt, piv, st, diag, col, 0.0, _eps(kind, x, ls, S, kw.get("power"), kw.get("offset")), rank)


# ---------------------------------------------------------------------------------------------------------
# rank past the column cache: the cooperative kernel caches what fits in shared memory and reads the rest from L
# ---------------------------------------------------------------------------------------------------------
def test_rank_200_through_the_plan_and_the_public_function(Plan, cuda_dev, monkeypatch):
    import gpytorch_b200 as gp
    from gpytorch_b200.operators import KernelLinearOperator

    n, d, ls, S, rank = 20000, 4, 0.3, 1.0, 200
    x = torch.rand(n, d, generator=torch.Generator().manual_seed(200))
    col, eps = _col_fn("rbf", x, ls, S), _eps("rbf", x, ls, S)
    p = Plan(x.to(cuda_dev)).set_hypers("rbf", ls, S, 0.1)
    lt, piv, st = _run(p, rank, 0.0)
    assert st == 0 and lt.size(0) == rank
    _check(lt, piv, st, torch.ones(n, dtype=torch.float64), col, 0.0, eps, rank)
    monkeypatch.setenv("GP_PC_STEPWISE", "1")
    lt2, piv2, _ = _run(p, rank, 0.0)
    monkeypatch.delenv("GP_PC_STEPWISE")
    assert torch.equal(piv, piv2) and torch.equal(lt, lt2)
    p.close()
    op = KernelLinearOperator(x.to(cuda_dev), None, "rbf", torch.tensor(ls, device=cuda_dev), torch.tensor(S, device=cuda_dev))
    L, pv = gp.pivoted_cholesky(op, rank, error_tol=0.0, return_pivots=True)
    assert L.shape == (n, rank)
    assert torch.equal(pv, piv) and torch.equal(L.t(), lt)


# ---------------------------------------------------------------------------------------------------------
# composite entry sources: each operator's plan from its feature tests' builders, its dense fp64 K from its oracle.  eps_K is 2e-5
# of the largest |K| entry (of the entry majorant for derivative observations), the row bound those feature tests hold the
# operator's row extraction to.
# ---------------------------------------------------------------------------------------------------------
ROW_REL = 2e-5


def _src_sum_poly(dev, Plan):
    x = torch.rand(3000, 3, generator=torch.Generator().manual_seed(41))
    pa = Plan(x.to(dev)).set_hypers("rbf", 0.4, 1.2, 0.0)
    pb = Plan(x.to(dev)).set_hypers_poly(2, 0.5, 0.3, 0.0)
    p = Plan(x.to(dev)).set_sum([pa, pb]).set_hypers("rbf", [1.0], 1.0, 0.1)
    xd = x.double()
    d = (xd[:, None, :] - xd[None, :, :]) / 0.4
    K = 1.2 * torch.exp(-0.5 * (d * d).sum(-1)) + 0.3 * (xd @ xd.T + 0.5) ** 2
    return p, [pa, pb], K, None, pa.diag().double().cpu() + pb.diag().double().cpu()   # a sum has no diag() of its own


def _src_product(dev, Plan):
    import product_oracle as pro
    from test_gpu_product import TC2, _plans

    x = torch.rand(3000, 4, generator=torch.Generator().manual_seed(42))
    factors = [("rbf", [0, 1, 2], 0.6, 1.2), ("matern12", [3], 1.5, 0.7)]
    p, fp, _ = _plans(dev, factors, x, None, TC2, noise=0.1)
    return p, fp, pro.dense(pro.f32_factors(factors), x), None


def _src_task(dev, Plan):
    import hadamard_oracle as ho

    g = torch.Generator().manual_seed(43)
    n, T = 3000, 4
    x = torch.rand(n, 3, generator=g, dtype=torch.float64).float()
    t = torch.randint(0, T, (n,), generator=g)
    B = torch.diag(torch.tensor([0.5, 2.0, 1.0, 1.5], dtype=torch.float64)) + 0.1
    p = Plan(x.to(dev)).set_hypers("rbf", 0.3, 1.1, 0.1)
    p.set_tasks(t.to(dev), None, T)
    p.set_task_covar(B.float())
    return p, [], ho.hadamard_matrix("rbf", x.double(), x.double(), t, t, 0.3, 1.1, B.float().double(), True), None


def _src_kron(dev, Plan):
    import kron_oracle as kro
    from test_gpu_kron import _kron

    x = torch.rand(1000, 3, generator=torch.Generator().manual_seed(44)).double()
    B = (torch.diag(torch.tensor([0.5, 2.0, 1.0], dtype=torch.float64)) + 0.1).float().double()
    data = Plan(x.float().to(dev)).set_hypers("rbf", 0.3, 1.1, 0.0)
    return _kron(data, 3, B, noise=0.1), [data], kro.kron_matrix("rbf", x, x, 0.3, 1.1, B, True), None


def _src_kron_obs(dev, Plan):
    import kron_mask_oracle as km
    import multitask_oracle as mto
    from test_gpu_kron_mask import LS, OS, _kron

    n, T = 1500, 3
    x = torch.rand(n, 2, generator=torch.Generator().manual_seed(45))
    B = mto.random_B(T, 42)
    rows = km.pattern("frac50", n, T, 43)
    p, _ = _kron(dev, "rbf", x, None, T, B, "simt", rows, None, noise=0.1)
    return p, [], km.mask_matrix("rbf", x, None, LS, OS, B, rows, rows), None


def _src_kron_terms(dev, Plan):
    import lcm_oracle as lo
    from test_gpu_lcm import _build

    lp, datas, terms = _build(dev, 3, 3, ["tcgen05", "simt"], n=1000)
    return lp, datas, lo.dense([dict(tm, x1=tm["x1"].cpu()) for tm in terms]), None


def _src_deriv(dev, Plan, m52=False):
    from gpytorch_b200.engine import DerivPlan

    if m52:
        import m52grad_oracle as o
        dense, major = o.m52grad_dense, o.m52grad_majorant
    else:
        import deriv_oracle as o
        dense, major = o.deriv_dense, o.deriv_majorant
    x = torch.rand(750, 3, generator=torch.Generator().manual_seed(46)).double()
    ls = torch.tensor([0.35, 0.5, 0.7])
    data = Plan(x.float().to(dev)).set_hypers("matern52" if m52 else "rbf", ls.tolist(), 1.1, 0.0)
    p = (DerivPlan(data, "matern52") if m52 else DerivPlan(data)).set_noise(0.1)
    return p, [data], dense(x, x, ls, 1.1), ROW_REL * float(major(x, x, ls, 1.1).max())


def _src_additive(dev, Plan):
    import additive_oracle as ao
    from test_gpu_additive import _hyp, _plan, _points

    x = _points(3000, 3, 47)
    ls, sc = _hyp(3, 9, False)
    p = _plan(dev, "matern32", x, None, ls, sc, 2, noise=0.1)
    return p, [], ao.additive_dense("matern32", x.double(), x.double(), ls, sc, 2), None


def _src_spectral(dev, Plan):
    import spectral_oracle as so
    from test_gpu_spectral import _params, _plan, _points

    x = _points(3000, 2, 48)
    w, mu, v = _params(3, 2, 49)
    p = _plan(dev, x, None, w, mu, v, 0.8, noise=0.1)
    return p, [], so.covariance(x, x, w, mu, v, 0.8), None


SOURCES = {"sum_poly": _src_sum_poly, "product": _src_product, "task": _src_task, "kron": _src_kron, "kron_obs": _src_kron_obs,
           "kron_terms": _src_kron_terms, "deriv": _src_deriv, "m52grad": lambda d, P: _src_deriv(d, P, True),
           "additive": _src_additive, "spectral": _src_spectral}


@pytest.mark.parametrize("src", list(SOURCES))
def test_composite_entry_sources(Plan, cuda_dev, src):
    p, keep, K, eps, *diag = SOURCES[src](cuda_dev, Plan)
    K = K.double().cpu()
    n, rank = K.size(0), 40
    assert n > 4 * PCP_THREADS   # several CTAs
    diag = diag[0] if diag else p.diag().double().cpu()
    lt, piv, st = _run(p, rank, 0.0)
    p.close()
    for q in keep:
        q.close()
    assert st == 0
    # a sum with a polynomial term may end once no residual is positive (rank_stop), with status 0
    assert lt.size(0) == rank or src == "sum_poly"
    eps = ROW_REL * float(K.abs().max()) if eps is None else eps
    _check(lt, piv, st, diag, lambda i: K[:, i], 0.0, eps, rank)


# ---------------------------------------------------------------------------------------------------------
# several-term Kronecker and derivative rows (row r is point r / rep) beyond the resident grid
# ---------------------------------------------------------------------------------------------------------
def test_grid_stride_kron_terms(Plan, cuda_dev):
    if _host_gb() < 6:
        pytest.skip("the fp64 pivot columns of n = 5e5 rows need ~1 GB of host memory")
    from gpytorch_b200.engine import LcmPlan
    import multitask_oracle as mto

    T, rank = 2, 40
    npts = -(-_grid_stride_n(cuda_dev) // T)
    x = torch.rand(npts, 3, generator=torch.Generator().manual_seed(50))
    spec = [("rbf", 0.3, 1.0), ("matern52", 0.8, 0.6)]
    Bs = [mto.random_B(T, 60 + q).float() for q in range(2)]
    datas = [Plan(x.to(cuda_dev)).set_hypers(k, ls, os_, 0.0) for k, ls, os_ in spec]
    lp = LcmPlan(datas, T)
    lp.set_noise(0.1)
    lp.set_term_covars(torch.stack(Bs))
    diag = lp.diag().double().cpu()
    lt, piv, st = _run(lp, rank, 0.0)
    lp.close()
    for q in datas:
        q.close()
    cols = [_col_fn(k, x, ls, os_) for k, ls, os_ in spec]

    def col(i):
        pt, a = i // T, i % T
        return sum(torch.kron(c(pt)[:, None], B.double()[:, a:a + 1])[:, 0] for c, B in zip(cols, Bs))
    kmax = sum(os_ * float(B.double().abs().max()) for (_, _, os_), B in zip(spec, Bs))
    assert st == 0 and lt.size(0) == rank and lt.size(1) >= _grid_stride_n(cuda_dev)
    _check(lt, piv, st, diag, col, 0.0, ROW_REL * kmax, rank)


def test_grid_stride_deriv(Plan, cuda_dev):
    if _host_gb() < 6:
        pytest.skip("the fp64 pivot columns of n = 5e5 rows need ~1 GB of host memory")
    from gpytorch_b200.engine import DerivPlan
    import deriv_oracle as do

    d, rank = 2, 40
    rep = d + 1
    npts = -(-_grid_stride_n(cuda_dev) // rep)
    x = torch.rand(npts, d, generator=torch.Generator().manual_seed(51))
    ls = torch.tensor([0.3, 0.45])
    data = Plan(x.to(cuda_dev)).set_hypers("rbf", ls.tolist(), 1.1, 0.0)
    p = DerivPlan(data).set_noise(0.1)
    diag = p.diag().double().cpu()
    lt, piv, st = _run(p, rank, 0.0)
    p.close(), data.close()
    xd = x.double()
    assert st == 0 and lt.size(0) == rank and lt.size(1) >= _grid_stride_n(cuda_dev)
    _check(lt, piv, st, diag, lambda i: do.deriv_dense(xd, xd[i // rep:i // rep + 1], ls, 1.1)[:, i % rep], 0.0,
           lambda i: ROW_REL * do.deriv_majorant(xd, xd[i // rep:i // rep + 1], ls, 1.1)[:, i % rep], rank)
