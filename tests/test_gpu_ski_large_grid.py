"""KISS-GP grids over 128 nodes per dimension (csrc/ski.cu, ski_mode_banded_kernel), entry by entry against fp64.

Products (Plan.kmv, gp_ski_grid_matmul, gp_ski_interp_matmul) and the hyper-parameter gradient run the cases of
tests/ski_large_grid_oracle.py against the chunked fp64 reference of tests/ski_scale_oracle.py, with the entrywise bound derived in
tests/test_gpu_ski_scale.py and two refinements that keep it meaningful on fine grids:
  * Toeplitz factors.  Entry k of t_i carries its own fp32 error, (3 r_k^2 + 10 r_k + 10) u t_i[k] with r_k = sqrt(5) k step_i / l
    (+ 6 u t_i[k] for l dt_i/dl), instead of the largest r over the grid: the bound adds sum_i K(.., E_i, ..) |W|^T |V|, E_i the
    Toeplitz matrix of those errors.
  * Mode products.  A banded product accumulates at most k_active = min(G, 128 + 2 (band - 1) + 64) terms per output (the k-chunks
    it runs; the skipped ones hold exact zeros), so a banded mode counts (k_active + 4) 2^-22 of |T_i| |B| where the dense one
    counts (G + 4) 2^-22.
Single entries, the pivoted Cholesky, the solves and prediction run through the bounds of tests/test_gpu_ski_precond.py and the
reference's KISS-GP example.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import ski_large_grid_oracle as lo  # noqa: E402
import ski_scale_oracle as so  # noqa: E402
from oracle import linalg as ol  # noqa: E402
from test_gpu_ski_precond import dense64, interp_and_factors, pow2_points  # noqa: E402
import pivchol_oracle as po  # noqa: E402

U = 2.0 ** -24
NOISE = 0.1


def _record(entry, case, err, bound):
    r = float((err / bound).max())
    print(f"\n{case:18s} {entry:12s} max err / bound = {r:.3e}")
    assert torch.isfinite(err).all() and r <= 1.0, (entry, case, r)


def _plan(dev, sizes, x, lo_, step, kind, ls, os_, noise=NOISE):
    from gpytorch_b200.engine import Plan

    p = Plan(x.to(dev)).set_ski(sizes, lo_, step).set_hypers(kind, ls, os_, noise)
    assert p.info()["backend"] == "ski"
    return p


def _fac_err_cols(case, step, cols, deriv_dim=None):
    """Per dimension the error column of the fp32 factor: (3 r^2 + 10 r + 10) u |t| (+ 6 u |t| for a derivative factor)."""
    out = []
    for i, (G, s, c) in enumerate(zip(case.sizes, step, cols)):
        r = math.sqrt(5.0) * torch.arange(G, dtype=torch.float64) * s / case.ls
        e = (3 * r * r + 10 * r + 10) * U + (6 * U if i == deriv_dim else 0.0)
        out.append(e * c.abs())
    return out


def _mode_eps(case, step):
    eps = 0.0
    for G, s in zip(case.sizes, step):
        k = G if G <= lo.DENSE_G else lo.k_active(G, max(lo.band_end(lo.column_fp32(case.kind, G, s, case.ls)),
                                                        lo.band_end(lo.column_fp32(case.kind, G, s, case.ls, True))))
        eps += (k + 4) * 2.0 ** -22
    return eps


def _kuu_err(case, step, cols, Z, deriv_dim=None):
    """sum_i (|T_0| x .. x E_i x .. ) Z: the factors' own fp32 errors propagated through the product."""
    errs = _fac_err_cols(case, step, cols, deriv_dim)
    acol = [c.abs() for c in cols]
    return sum(so.kuu(acol[:i] + [errs[i]] + acol[i + 1:], Z) for i in range(len(cols)))


@pytest.fixture(scope="module")
def prepared():
    cache = {}

    def get(case):
        if case.name not in cache:
            cache.clear()
            x, axes, lo_, step = lo.case_grid(case)
            W = so.Interp(axes, x)
            cache[case.name] = (x, lo_, step, W, W.node_counts(), so.regular_axes(lo_, step, case.sizes))
        return cache[case.name]

    return get


@pytest.mark.parametrize("case", lo.CASES, ids=lambda c: c.name)
def test_products_entrywise(cuda_dev, prepared, case):
    x, lo_, step, W, m, reg = prepared(case)
    d, n, M, OS = len(case.sizes), case.n, W.M, case.outputscale
    g = torch.Generator().manual_seed(100 + case.seed)
    tmax = max(case.t)
    V = torch.randn(n, tmax, generator=g)
    V64 = V.double()
    cols = so.toeplitz_columns(case.kind, reg, case.ls)
    Umag = W.wt(V64.abs(), "abs")
    Q = (2 * m + d).unsqueeze(1) * Umag + 34 * d * W.wt(V64.abs(), "support") + _mode_eps(case, step) / U * Umag
    Y, Ymag, EY = so.kuu(cols, torch.cat([W.wt(V64), Umag, U * Q], 1)).split(tmax, 1)
    EY = EY + _kuu_err(case, step, cols, Umag)
    out_ref = OS * W.w(Y)
    WY = W.w(torch.cat([EY, Ymag], 1), "abs")
    out_bnd = OS * (WY[:, :tmax] + (4 ** d + d) * U * WY[:, tmax:] + 34 * d * U * W.w(Ymag, "support")) + 2 * U * OS * WY[:, tmax:]
    grid_ref, grid_bnd = OS * Y, OS * (EY + U * Ymag)
    p = _plan(cuda_dev, case.sizes, x, lo_, step, case.kind, case.ls, OS)
    Vd = V.to(cuda_dev)
    for t in case.t:
        got = p.kmv(Vd[:, :t].contiguous(), add_noise=True).double().cpu()
        _record("kmv+noise", case.name, (got - out_ref[:, :t] - NOISE * V64[:, :t]).abs(),
                out_bnd[:, :t] + 2 * U * NOISE * V64[:, :t].abs())
        got = p.ski_grid_matmul(Vd[:, :t].contiguous()).double().cpu()
        _record("grid_matmul", case.name, (got - grid_ref[:, :t]).abs(), grid_bnd[:, :t])
    del Y, Ymag, EY, WY, out_ref, out_bnd, grid_ref, grid_bnd
    Cg = torch.randn(M, tmax, generator=g)
    ref = W.w(Cg.double())
    bnd = (4 ** d + 2 * d) * U * W.w(Cg.double().abs(), "abs") + 33 * d * U * W.w(Cg.double().abs(), "support")
    got = p.ski_interp_matmul(Cg.to(cuda_dev))
    _record("interp", case.name, (got.double().cpu() - ref).abs(), bnd)
    p.close()


GRAD_CASES = [c for c in lo.CASES if c.grads]


@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: c.name)
def test_bilinear_grad_entrywise(cuda_dev, prepared, case):
    x, lo_, step, W, m, reg = prepared(case)
    d, n, OS = len(case.sizes), case.n, case.outputscale
    g = torch.Generator().manual_seed(200 + case.seed)
    L, R = torch.randn(n, 2, generator=g), torch.randn(n, 2, generator=g)
    A, B = W.wt(L.double()), W.wt(R.double())
    Amag, Bmag = W.wt(L.double().abs(), "abs"), W.wt(R.double().abs(), "abs")
    QA = (2 * m + d).unsqueeze(1) * Amag + 34 * d * W.wt(L.double().abs(), "support")
    QB = (2 * m + d).unsqueeze(1) * Bmag + 34 * d * W.wt(R.double().abs(), "support")
    ls = torch.tensor(case.ls, dtype=torch.float64, requires_grad=True)
    osc = torch.tensor(OS, dtype=torch.float64, requires_grad=True)
    val = osc * (A * so.kuu(so.toeplitz_columns(case.kind, reg, ls), B)).sum()
    val.backward()
    bounds = []
    for j in range(d + 1):
        dd = None if j == 0 else j - 1
        cols = so.toeplitz_columns(case.kind, reg, case.ls, dd)
        KB = so.kuu([c.abs() for c in cols], torch.cat([Bmag, U * QB], 1))
        mag = float((Amag * KB[:, :2]).sum())
        ferr = float((Amag * _kuu_err(case, step, cols, Bmag, dd)).sum())
        bounds.append(U * float((QA * KB[:, :2]).sum()) + float((Amag * KB[:, 2:]).sum()) + ferr
                      + (_mode_eps(case, step) + 1e-9) * mag)
    p = _plan(cuda_dev, case.sizes, x, lo_, step, case.kind, case.ls, OS)
    gl, go = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    p.close()
    _record("d/ds", case.name, torch.tensor(abs(go - osc.grad.item())), torch.tensor(bounds[0]))
    _record("d/dl", case.name, torch.tensor(abs(gl[0] - ls.grad.item())), torch.tensor(OS / case.ls * sum(bounds[1:])))


def test_input_grad_on_a_large_grid(cuda_dev, prepared):
    from dkl_oracle import ski_input_grad

    case = next(c for c in lo.CASES if c.name == "g1000_rbf")
    x, lo_, step, W, m, reg = prepared(case)
    n, d, t = 100_000, 1, 2
    x = x[:n]
    g = torch.Generator().manual_seed(300)
    L, R = torch.randn(n, t, generator=g), torch.randn(n, t, generator=g)
    p = _plan(cuda_dev, case.sizes, x, lo_, step, case.kind, case.ls, case.outputscale)
    got = p.ski_input_grad(L.to(cuda_dev), R.to(cuda_dev)).double().cpu()
    p.close()
    ref, mag = ski_input_grad(case.kind, x.double(), reg, case.ls, case.outputscale, L.double(), R.double())
    Wn = so.Interp(so.bench_grid(case.sizes)[0], x)
    k = 2 * float(Wn.node_counts().max()) + 4 * sum(case.sizes) + 2 * 4 ** d + 2 * t + 16 + 20 * max(case.sizes)
    keep = torch.ones(n, dtype=torch.bool)
    for i, ax in enumerate(reg):
        for e in (float(ax[1]), float(ax[-2])):
            keep &= (x[:, i].double() - e).abs() >= 1e-4
    _record("input_grad", case.name, (got - ref).abs()[keep], (k * U * mag + 1e-30)[keep])


# ---- single entries and the pivoted Cholesky (ski_rows.cuh from the generating columns) -----------------------------------------
ENTRY_CASES = [([129], "rbf", 0.05, 3001), ([1000], "matern12", 0.1, 3001), ([4097], "rbf", 0.01, 2001), ([129, 4], "matern32", 0.3, 2999),
               ([130, 8, 8, 8], "matern52", 0.4, 1501), ([600, 300], "rbf", 0.05, 2001)]


@pytest.mark.parametrize("sizes,kind,ls,n", ENTRY_CASES, ids=lambda v: str(v))
def test_entries_and_pivoted_cholesky(cuda_dev, sizes, kind, ls, n):
    d = len(sizes)
    x, axes, lo_, steps = pow2_points(sizes, n, seed=n + d)
    p = _plan(cuda_dev, sizes, x, lo_, steps, kind, ls, 1.7)
    first, w, T = interp_and_factors(kind, x, axes, ls)
    K = dense64(first, w, T, 1.7)
    Bm = dense64(first, w, T, 1.0, absw=True)
    R = max(math.sqrt(5.0) * (g - 1) * s / ls for g, s in zip(sizes, steps))
    # + an absolute floor for the fp32 factors' denormal range (expf below 2^-126 keeps fewer than 24 bits; an entry that
    # underflows differs from fp64 by < 2^-149): 16 d such entries per SKI entry, times s and the other dimensions' sums <= 4^d
    bound = 1.01 * 1.7 * d * ((3 * R * R + 10 * R + 10) * U + 42 * U) * Bm + 1.7 * 16 * d * 4 ** d * 2.0 ** -126
    dg = p.diag().double().cpu()
    assert ((dg - K.diagonal()).abs() <= bound.diagonal()).all()
    rows = torch.tensor([0, 5, 7, 13, 14, 15, n // 2, n - 1])
    kr = p.rows(rows.to(cuda_dev)).double().cpu()
    _record("krows", str(sizes), (kr - K[rows]).abs(), bound[rows])
    assert torch.equal(kr[torch.arange(len(rows)), rows], dg[rows])     # the row formula at j = i is the diagonal, bit for bit
    k = 20
    lt, piv, st = p.pivoted_cholesky(k, 0.0)
    assert st == 0 and torch.isfinite(lt).all()
    L64, piv64 = ol.pivoted_cholesky(dg, lambda i: p.rows(torch.tensor([i], device=cuda_dev)).double().cpu()[0], k, 0.0)
    mdg = float(dg.max())
    if min(po.pivot_gaps(dg, L64, piv64)) > 2 ** 4 * (k + 1) * U * mdg:   # no near-tie: the fp64 pivoting is the device's
        assert piv.cpu().tolist() == piv64.tolist()
    # L L^T reproduces the operator on the pivot columns, whichever order near-ties took
    pv = piv.cpu()
    ltd = lt.double().cpu()
    Kp = p.rows(pv.to(cuda_dev)).double().cpu()
    assert float((ltd.T @ ltd[:, pv] - Kp.T).abs().max()) <= 1e-3 * mdg
    p.close()


def test_mll_lanczos_against_dense_on_a_large_grid(cuda_dev):
    """mBCG solve, the MLL's inverse quadratic form and SLQ log det, and Lanczos extremes on a 1-D 2000-node grid against dense
    fp64 (the preconditioned solves run in the API test below)."""
    sizes, kind, ls, n, nz = [2000], "matern32", 0.02, 3000, 0.05
    x, axes, lo_, steps = pow2_points(sizes, n, seed=3, special=False)
    first, w, T = interp_and_factors(kind, x, axes, ls)
    Kh = dense64(first, w, T, 1.3) + nz * torch.eye(n, dtype=torch.float64)
    p = _plan(cuda_dev, sizes, x, lo_, steps, kind, ls, 1.3, nz)
    y = torch.sin(6 * x.double()[:, 0]) + 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    solves, _, info = p.mbcg(y.float().to(cuda_dev)[:, None], 0, 1e-5, 2000)
    ref = torch.linalg.solve(Kh, y)
    assert ((solves[:, 0].double().cpu() - ref).norm() / ref.norm()).item() < 1e-3
    evals = torch.linalg.eigvalsh(Kh)
    init = torch.randn(n, generator=torch.Generator().manual_seed(2)).to(cuda_dev)
    _, tm = p.lanczos(init, 60)
    te = torch.linalg.eigvalsh(tm.double().cpu())
    assert abs(float(te[-1]) - float(evals[-1])) <= 1e-3 * float(evals[-1])
    assert float(te[0]) >= float(evals[0]) * (1 - 1e-3)
    g = torch.Generator().manual_seed(4)
    rank, probes = 15, 10
    eps1, eps2 = torch.randn(n, probes, generator=g), torch.randn(rank, probes, generator=g)
    rad = torch.randint(0, 2, (n, probes), generator=g).float() * 2 - 1
    _, logdet = torch.linalg.slogdet(Kh)
    r, _ = p.mll(y.float().to(cuda_dev), eps1.to(cuda_dev), eps2.to(cuda_dev), rad.to(cuda_dev), probes, rank, 10 ** 9,
                 cg_tol=1e-4, max_cg_iter=3000)
    assert r.inv_quad == pytest.approx(float(y @ ref), rel=1e-3)
    assert r.logdet == pytest.approx(float(logdet), rel=0.05, abs=0.02 * n)
    p.close()


def test_refusals(cuda_dev):
    from gpytorch_b200.engine import Plan

    x = torch.rand(1000, 2, device=cuda_dev)
    for sizes in ([131073, 4], [131072, 1024], [4, 131073]):
        p = Plan(x)
        with pytest.raises(RuntimeError) as e:
            p.set_ski(sizes, [0.0, 0.0], [1e-5, 1e-3])
        assert "grid" in str(e.value)
        p.close()
    p = Plan(x).set_ski([131072, 1023], [0.0, -1e-3], [1.0 / 131000, 1.0 / 1000]).set_hypers("rbf", 0.1, 1.0, 0.1)
    p.close()                                                           # M 16 = 2^31 - 2^21: accepted
    p = Plan(x[:, :1].contiguous()).set_ski([131072], [-1e-5], [1.0 / 131000]).set_hypers("rbf", 0.1, 1.0, 0.1)
    p.close()


# ---- through the API -------------------------------------------------------------------------------------------------------------
def test_reference_kissgp_example_with_choose_grid_size(cuda_dev):
    """The reference's 1-D KISS-GP regression example (sin 2 pi x, 25 Adam steps at lr 0.1, MAE < 0.05 on 51 test points) on 1000
    training points, with grid_size = choose_grid_size(train_x) = 1000 nodes (the outputscale outside the grid kernel, the form
    the accelerated path takes; the operator is the same)."""
    import gpytorch_b200 as gp
    from gpytorch_b200.utils.grid import choose_grid_size

    train_x = torch.linspace(0, 1, 1000, device=cuda_dev)
    train_y = torch.sin(train_x * (2 * math.pi))
    test_x = torch.linspace(0, 1, 51, device=cuda_dev)
    test_y = torch.sin(test_x * (2 * math.pi))
    G = choose_grid_size(train_x)
    assert G == 1000

    class M(gp.models.ExactGP):
        def __init__(self, lik):
            super().__init__(train_x, train_y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), grid_size=G, num_dims=1))

        def forward(self, x):
            return gp.distributions.MultivariateNormal(self.mean_module(x), self.covar_module(x))

    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    model = M(lik).to(cuda_dev)
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    model.train(); lik.train()
    opt = torch.optim.Adam(model.parameters(), lr=0.1)
    losses = []
    for _ in range(25):
        opt.zero_grad()
        loss = -mll(model(train_x), train_y)
        loss.backward()
        losses.append(loss.item())
        opt.step()
    for prm in model.parameters():
        assert prm.grad is not None and prm.grad.norm().item() > 0
    assert losses[-1] < losses[0]
    model.eval(); lik.eval()
    with torch.no_grad():
        pred = lik(model(test_x)).mean
    mae = torch.mean(torch.abs(test_y - pred)).item()
    print(f"\n1-D KISS-GP, G = {G}: loss {losses[0]:.3f} -> {losses[-1]:.3f}, MAE {mae:.4f}")
    assert mae < 0.05


def test_2d_model_with_preconditioner_and_grid_prediction(cuda_dev):
    """ScaleKernel(GridInterpolationKernel(RBF, 300^2)) on 10^5 points: trains with settings.ski_preconditioner (loss decreasing) and
    predicts with settings.ski_grid_prediction, whose mean matches the joint path's."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n = 100_000
    g = torch.Generator().manual_seed(11)
    x = torch.rand(n, 2, generator=g)
    y = torch.sin(4 * x[:, 0]) * torch.cos(3 * x[:, 1]) + 0.05 * torch.randn(n, generator=g)
    xt = torch.rand(500, 2, generator=g)
    x, y, xt = x.to(cuda_dev), y.to(cuda_dev), xt.to(cuda_dev)

    class M(gp.models.ExactGP):
        def __init__(self, lik):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel(), grid_size=300, num_dims=2,
                                                                                       grid_bounds=[(0.0, 1.0)] * 2))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    model = M(lik).to(cuda_dev)
    model.covar_module.base_kernel.base_kernel.lengthscale = 0.2
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    opt = torch.optim.Adam(model.parameters(), lr=0.1)
    model.train(); lik.train()
    losses = []
    with settings.ski_preconditioner(True), settings.probe_seed(3), settings.cg_tolerance(1e-2):
        for _ in range(8):
            opt.zero_grad()
            loss = -mll(model(x), y)
            loss.backward()
            losses.append(loss.item())
            opt.step()
    assert losses[-1] < losses[0]
    model.eval(); lik.eval()
    with torch.no_grad(), settings.eval_cg_tolerance(1e-4), settings.ski_preconditioner(True):
        with settings.ski_grid_prediction(True), settings.fast_pred_var(True):
            pg = model(xt)
            mg, vg = pg.mean, pg.variance
        model._clear_caches()
        with settings.ski_grid_prediction(False):
            mj = model(xt).mean
    ref = (torch.sin(4 * xt[:, 0]) * torch.cos(3 * xt[:, 1]))
    assert torch.isfinite(vg).all() and (vg > -1e-4).all()
    assert ((mg - mj).norm() / mj.norm()).item() < 1e-2
    assert (mg - ref).abs().mean().item() < 0.05
    print(f"\n2-D 300^2, n = 1e5: loss {losses[0]:.3f} -> {losses[-1]:.3f}, grid vs joint mean rel "
          f"{((mg - mj).norm() / mj.norm()).item():.2e}")
