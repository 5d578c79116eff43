"""The pivoted-Cholesky preconditioner of the SKI operator: single entries (gp_kdiag / gp_krows on SKI plans, csrc/ski_rows.cuh),
gp_pivoted_cholesky on SKI plans, and settings.ski_preconditioner through the solves, the prediction mean cache and CIQ sampling.

Reference.  The fp64 operator is built from the separable form (tests/test_ski_precond_host.py checks it against the oracle's
dense product) with the interpolation weights of oracle/ski.py computed in fp32 on grids whose nodes and spacing are exact
in fp32 (spacing a power of two, first node minus one spacing): the device then forms the same first nodes and the same
t = (x - lo) / step, and its weights differ from the reference's only by the FMA contraction of the cubic polynomials.

Entry bound (test_ski_entries_match_fp64).  Per dimension the device computes a_k = sum_b w_jb (sum_a T_k[.] w_ia) in fp32 from
  * weights within eps_w = 16 u of the reference (|w| <= 1, 4-term Horner polynomials; absolute),
  * T_k entries within eps_T = (3 R^2 + 10 R + 10) u relative (r = |a - b| step / l in 3 roundings, exp of -r^2/2 or of
    -sqrt(2 nu) r; R the largest scaled distance sqrt(5) (G_k - 1) step_k / l_k),
  * 8 FMA roundings,
so |a_k - a_k*| <= (eps_T + 8 u + 2 eps_w) B_k with B_k = (|w_i| + 1)^T T_k[f_i:f_i+4, f_j:f_j+4] (|w_j| + 1) (the ones absorb the
absolute weight errors), and over the product of d factors and the outputscale
  |K - K*| <= 1.01 s d (eps_T + 42 u) prod_k B_k ,   u = 2^-24.
The weights can be negative (Keys' kernel has negative lobes): the bound uses absolute values.

Pivoting (test_ski_pivoted_cholesky_matches_fp64_pivoting).  The oracle's fp64 pivoted Cholesky runs on the device's own diagonal
and rows, so only the pivoting arithmetic differs: step m's numerator K[p, j] - sum_q L_qp L_qj is formed in fp32 from terms
of size <= max diag, so its error is <= 2 (m + 1) u max diag, plus what earlier rows carry; the test asserts
|L_m - L_m*| <= 2^8 (m + 1) u max diag / L_m[p] per row and, for the pivots to be comparable, that every step's winning
diagonal beats the runner-up by more than 2^4 (k + 1) u max diag (the seeds are chosen so; a failure of that assertion is
a pivot flip, not an arithmetic error).  The MLL test pivots the same way and runs the oracle's mBCG on the fp64 operator.

MLL: iteration count equal to the oracle's preconditioned mBCG on the fp64 operator with the same eps1 / eps2, inv-quad and
log-det by the Krylov rule of tests/test_gpu_ski.py, and within 3 % of dense Cholesky through the public API.
CIQ: the bound of tests/test_gpu_ciq_precond.py (derived in its header) with the SKI operator in place of the dense kernel.
"""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import linalg as ol, ski  # noqa: E402
from test_gpu_ciq_precond import _factor64  # noqa: E402
from test_gpu_sampling import _sqrt_psd  # noqa: E402
from test_ski_precond_host import per_dim_interp, separable_diag, toeplitz_factors  # noqa: E402
import pivchol_oracle as po  # noqa: E402

U32 = 2.0 ** -24


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def pow2_grid(sizes):
    """Grid axes exact in fp32: spacing 2^-ceil(log2(G - 2)), first node minus one spacing (the extended grid of create_grid
    over [0, (G - 3) step])."""
    steps = [2.0 ** -math.ceil(math.log2(g - 2)) for g in sizes]
    axes = [(-s + torch.arange(g, dtype=torch.float64) * s).float() for g, s in zip(sizes, steps)]
    return axes, [-s for s in steps], steps


def pow2_points(sizes, n, seed, special=True):
    """n fp32 points inside the grid; special: some in the first / last cell and some exactly on nodes (their diagonal entries
    tie exactly: one-hot weights)."""
    axes, lo, steps = pow2_grid(sizes)
    g = torch.Generator().manual_seed(seed)
    lo_t = torch.tensor(lo, dtype=torch.float64)
    hi_t = torch.tensor([float(a[-1]) for a in axes], dtype=torch.float64)
    st_t = torch.tensor(steps, dtype=torch.float64)
    x = lo_t + st_t + torch.rand(n, len(sizes), generator=g, dtype=torch.float64) * (hi_t - lo_t - 2 * st_t)
    if not special:
        return x.float(), axes, lo, steps
    x[:7] = lo_t + torch.rand(7, len(sizes), generator=g, dtype=torch.float64) * st_t * 0.999
    x[7:14] = hi_t - torch.rand(7, len(sizes), generator=g, dtype=torch.float64) * st_t * 0.999
    x[14] = torch.stack([a[min(3, a.numel() - 1)].double() for a in axes])
    x[15] = torch.stack([a[a.numel() // 2].double() for a in axes])
    return x.float(), axes, lo, steps


def interp_and_factors(kind, x, axes, ls):
    """(first, w (fp64 of the fp32 weights), [T_k] fp64)."""
    first, w = per_dim_interp(axes, x)
    return first, w.double(), toeplitz_factors(kind, [a.double() for a in axes], ls)


def dense64(first, w, T, os_, absw=False):
    """s prod_k W_k T_k W_k^T (W_k [n, G_k] the 1-D interpolation rows: the 4 nodes of a row are distinct, so nothing cancels);
    absw: the majorant B of the entry bound, (|w| + 1) in place of w."""
    n = first.size(0)
    out = torch.full((n, n), float(os_), dtype=torch.float64)
    for k, Tk in enumerate(T):
        Wk = torch.zeros(n, Tk.size(0), dtype=torch.float64)
        Wk.scatter_(1, first[:, k, None] + torch.arange(4), w[:, k].abs() + 1 if absw else w[:, k])
        out *= Wk @ Tk @ Wk.T
    return out


def _ski_plan(cuda_dev, x, lo, steps, sizes, kind, ls, os_, noise):
    from gpytorch_b200.engine import Plan

    return Plan(x.to(cuda_dev)).set_ski(sizes, lo, steps).set_hypers(kind, ls, os_, noise)


ENTRY_CASES = [
    (1, [4], "rbf", [0.3], 1001), (1, [128], "matern12", [0.2], 3001), (2, [128, 4], "matern32", [0.3, 0.5], 2999),
    (2, [33, 17], "rbf", [0.25], 1537), (3, [20, 16, 12], "matern52", [0.3, 0.4, 0.5], 4097), (4, [10, 8, 6, 5], "rbf", [0.4], 777),
    (3, [4, 128, 9], "matern12", [0.6], 2049),
]


@pytest.mark.parametrize("d,sizes,kind,ls,n", ENTRY_CASES)
def test_ski_entries_match_fp64(cuda_dev, d, sizes, kind, ls, n):
    x, axes, lo, steps = pow2_points(sizes, n, seed=n + d)
    lsv = ls[0] if len(ls) == 1 else ls
    p = _ski_plan(cuda_dev, x, lo, steps, sizes, kind, lsv, 1.7, 0.1)
    first, w, T = interp_and_factors(kind, x, axes, torch.tensor(ls, dtype=torch.float64) if len(ls) > 1 else ls[0])
    K = dense64(first, w, T, 1.7)
    B = dense64(first, w, T, 1.0, absw=True)
    lsd = ls * d if len(ls) == 1 else ls
    R = max(math.sqrt(5.0) * (g - 1) * s / l for g, s, l in zip(sizes, steps, lsd))
    eps_t = (3 * R * R + 10 * R + 10) * U32
    bound = 1.01 * 1.7 * d * (eps_t + 42 * U32) * B
    dg = p.diag().double().cpu()
    assert torch.isfinite(dg).all()
    assert ((dg - K.diagonal()).abs() <= bound.diagonal()).all()
    rows = torch.tensor([0, 5, 7, 13, 14, 15, n // 2, n - 1])
    kr = p.rows(rows.to(cuda_dev)).double().cpu()
    err = (kr - K[rows]).abs()
    print(f"\nd={d} {sizes} {kind}: max err / bound {float((err / bound[rows]).max()):.3g}")
    assert (err <= bound[rows]).all()
    assert torch.equal(kr[torch.arange(len(rows)), rows], dg[rows])     # the row formula at j = i is the diagonal, bit for bit
    # ScaleKernel(GridInterpolationKernel(...))(x, diag=True) is the scaled diagonal of the same operator
    import gpytorch_b200 as gp

    k = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(gp.kernels.RBFKernel() if kind == "rbf" else gp.kernels.MaternKernel(
        nu={"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}[kind], ard_num_dims=len(ls) if len(ls) > 1 else None),
        grid_size=sizes, num_dims=d, grid_bounds=[(0.0, 1.0)] * d)).to(cuda_dev)
    k.base_kernel.base_kernel.lengthscale = ls if len(ls) > 1 else ls[0]
    k.outputscale = 1.7
    xd = x.double().clamp(0.0, 1.0)
    dd = k(xd.float().to(cuda_dev), diag=True)
    assert dd.shape == (n,)
    ref = separable_diag(kind, xd, [a.double() for a in ski.create_grid(sizes, [(0.0, 1.0)] * d)], lsv if len(ls) == 1
                         else torch.tensor(ls, dtype=torch.float64), 1.7)
    assert rel(dd, ref) < 1e-4           # fp32 against fp64 interpolation weights: ~G u relative
    p.close()


@pytest.mark.parametrize("d,sizes,kind,ls,n,k,tol,seed", [
    (2, [32, 32], "matern32", 0.25, 600, 15, 1e-3, 2), (3, [16, 12, 10], "matern52", 0.4, 500, 40, 0.0, 7),
    (1, [24], "rbf", 0.3, 1200, 100, 1e-3, 0),          # rank-deficient: prod G_k = 24 < k
])
def test_ski_pivoted_cholesky_matches_fp64_pivoting(cuda_dev, d, sizes, kind, ls, n, k, tol, seed):
    x, axes, lo, steps = pow2_points(sizes, n, seed=seed, special=False)
    p = _ski_plan(cuda_dev, x, lo, steps, sizes, kind, ls, 1.3, 0.05)
    lt, piv, st = p.pivoted_cholesky(k, tol)
    assert st == 0 and torch.isfinite(lt).all()
    diag = p.diag().double().cpu()
    rows = {}

    def get_row(i):
        if i not in rows:
            rows[i] = p.rows(torch.tensor([i], device=cuda_dev)).double().cpu()[0]
        return rows[i]

    L64, piv64 = ol.pivoted_cholesky(diag, get_row, k, tol)
    mdg = float(diag.max())
    if math.prod(sizes) < k:
        assert lt.size(0) <= math.prod(sizes)
        Kd = torch.stack([get_row(i) for i in range(0, n, 37)])
        approx = lt.double().cpu()[:, ::37].T @ lt.double().cpu()
        assert float((approx - Kd).abs().max()) <= 1e-3 * mdg
        p.close()
        return
    gaps = po.pivot_gaps(diag, L64, piv64)
    print(f"\nd={d}: rank {lt.size(0)} (fp64 {piv64.numel()}), smallest pivot gap {min(gaps):.3g} x max diag {mdg:.3g}")
    assert min(gaps) > 2 ** 4 * (k + 1) * U32 * mdg
    assert piv.cpu().tolist() == piv64.tolist()
    assert lt.size(0) == L64.size(1)
    Lt64 = L64.T
    ltd = lt.double().cpu()
    for m in range(ltd.size(0)):
        pm = int(piv64[m])
        assert float((ltd[m] - Lt64[m]).abs().max()) <= 2 ** 8 * (m + 1) * U32 * mdg / float(Lt64[m, pm])
    p.close()


def _mll_problem(n, sizes, seed):
    x, axes, lo, steps = pow2_points(list(sizes), n, seed=seed, special=False)
    g = torch.Generator().manual_seed(seed + 1)
    y = (torch.sin(3 * x.double().sum(-1)) + 0.1 * torch.randn(n, generator=g, dtype=torch.float64)).float()
    return x, y, axes, lo, steps


def test_preconditioned_ski_mll_matches_oracle(cuda_dev):
    """Primitives (pivoted Cholesky, precond_build, N(0, P) probes, mBCG with W, SLQ) against the oracle's preconditioned mBCG on the
    fp64 operator with the same base samples."""
    n, sizes, kind, ls, os_, nz, k, tp, tol = 1500, [32, 32], "matern12", 0.3, 1.4, 0.05, 15, 10, 1.0
    x, y, axes, lo, steps = _mll_problem(n, sizes, seed=1)
    p = _ski_plan(cuda_dev, x, lo, steps, sizes, kind, ls, os_, nz)
    first, w, T = interp_and_factors(kind, x, axes, ls)
    # the oracle pivots on the device's own diagonal and rows (as in the pivoting test) and runs mBCG on the fp64 operator
    dg_dev = p.diag().double().cpu()
    rows = {}

    def dev_row(i):
        if i not in rows:
            rows[i] = p.rows(torch.tensor([i], device=cuda_dev)).double().cpu()[0]
        return rows[i]
    K = dense64(first, w, T, os_)
    g = torch.Generator().manual_seed(3)
    eps1 = torch.randn(k, tp, generator=g)
    eps2 = torch.randn(n, tp, generator=g)
    lt, piv, st = p.pivoted_cholesky(k, 1e-3)
    assert st == 0 and lt.size(0) == k
    wm, logdet_p, st = p.precond_build(lt)
    z = p.precond_probes(lt, eps1.to(cuda_dev), eps2.to(cuda_dev))
    rhs = torch.cat([z / z.norm(dim=0, keepdim=True), y.to(cuda_dev)[:, None]], -1)
    solves, tmat, info = p.mbcg(rhs, tp, tol, 1000, 20, precond_w=wm)
    ld = p.slq_logdet(tmat, n) + logdet_p
    iq = float((solves[:, tp:].double() * y.to(cuda_dev)[:, None].double()).sum())
    outs = {}
    for dt in (torch.float64, torch.float32):
        Kt = K.to(dt)
        L, pv = ol.pivoted_cholesky(dg_dev.to(dt), lambda i: dev_row(i).to(dt), k, 1e-3)
        pre = ol.build_preconditioner(L, nz, pv)
        probes = pre.probes(eps1.to(dt), eps2.to(dt))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            outs[dt] = ol.inv_quad_logdet(lambda v: Kt @ v + nz * v, n, y.to(dt), probes, pre, tol, 1000, 20, return_info=True)
        if dt == torch.float64:
            assert pv.tolist() == piv.cpu().tolist()
            gaps = po.pivot_gaps(dg_dev, L, pv)
            assert min(gaps) > 2 ** 4 * (k + 1) * U32 * float(dg_dev.max())
    (iq64, ld64, info64, _, _), (iq32, ld32, _, _, _) = outs[torch.float64], outs[torch.float32]
    print(f"\niters {info.iters} (oracle {info64.iters}); inv_quad {iq:.6g} / {iq64:.6g}; logdet {ld:.6g} / {ld64:.6g}")
    assert info.iters == info64.iters
    assert abs(iq - iq64) <= max(2e-4 * abs(iq64), 3 * abs(iq32 - iq64))
    assert abs(ld - ld64) <= max(2e-4 * abs(ld64), 3 * abs(ld32 - ld64))
    p.close()


@pytest.mark.parametrize("per_row", [False, True])
def test_preconditioned_ski_mll_through_the_api(cuda_dev, per_row):
    """inv_quad_logdet of K_ski + sigma^2 I (and K_ski + diag(d), FixedNoise) with settings.ski_preconditioner on: within 3 % of dense
    Cholesky, with a rank-15 preconditioner in use."""
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import (AddedDiagLinearOperator, ConstantDiagLinearOperator, DiagLinearOperator,
                                         SKIKernelLinearOperator)

    n, sizes, ls, os_ = 2500, [32, 32], 0.25, 1.4
    x, y, axes, lo, steps = _mll_problem(n, sizes, seed=11)
    first, w, T = interp_and_factors("rbf", x, axes, ls)
    K = dense64(first, w, T, os_)
    if per_row:
        dv = 0.02 + 0.1 * torch.rand(n, generator=torch.Generator().manual_seed(2))
        D = DiagLinearOperator(dv.to(cuda_dev))
        Kh = K + torch.diag(dv.double())
    else:
        D = ConstantDiagLinearOperator(torch.tensor(0.05, device=cuda_dev), n)
        Kh = K + float(torch.tensor(0.05)) * torch.eye(n, dtype=torch.float64)
    kop = SKIKernelLinearOperator(x.to(cuda_dev), "rbf", torch.tensor(ls, device=cuda_dev), torch.tensor(os_, device=cuda_dev),
                                  sizes, lo, steps)
    op = AddedDiagLinearOperator(kop, D)
    with settings.ski_preconditioner(True), settings.probe_seed(3), settings.cg_tolerance(1e-3), settings.num_trace_samples(15):
        iq, ld = op.inv_quad_logdet(y.to(cuda_dev)[:, None], logdet=True)
        assert op._preconditioner()[1].size(0) == 15
    Lc = torch.linalg.cholesky(Kh)
    iq_ref = float((y.double()[:, None] * torch.cholesky_solve(y.double()[:, None], Lc)).sum())
    ld_ref = float(2 * Lc.diagonal().log().sum())
    print(f"\nper_row={per_row}: iq {float(iq):.6g} / {iq_ref:.6g}, logdet {float(ld):.6g} / {ld_ref:.6g}, cg iters {op.last_cg_iters}")
    assert abs(float(iq) - iq_ref) <= 0.03 * abs(iq_ref)
    assert abs(float(ld) - ld_ref) <= 0.03 * abs(ld_ref)


def _ski_model(cuda_dev, x, y, grid_size, d, noise, kind="rbf"):
    import gpytorch_b200 as gp

    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    lik.noise = noise

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ZeroMean()
            base = gp.kernels.RBFKernel() if kind == "rbf" else gp.kernels.MaternKernel(nu=2.5)
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(base, grid_size=grid_size, num_dims=d,
                                                                                       grid_bounds=[(0.0, 1.0)] * d))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    return M().to(cuda_dev), lik


def _oracle_axes(sizes):
    return ski.create_grid(sizes, [(0.0, 1.0)] * len(sizes), dtype=torch.float32)


def test_preconditioner_cuts_mean_cache_iterations_on_a_stiff_problem(cuda_dev):
    """d = 2, 64^2 grid, N = 4000, sigma^2 = 1e-3: with the flag on (default rank 15) the mean-cache solve at eval_cg_tolerance(1e-5)
    takes clearly fewer CG iterations (597 against 1185 and 1199 in two H100 runs; the SKI product is not bit-reproducible, so the
    assertion keeps a margin: at most 60 %), and both posterior means agree with the dense fp64 one.  (At rank 100 the
    preconditioned solve stalls near a relative residual of 1e-5 here: fp32 P^-1 at sigma^2 = 1e-3; DESIGN section 4.6.)"""
    from gpytorch_b200 import operators, settings

    n, m, d, ls0, os0, nz0 = 4000, 40, 2, 0.2, 1.0, 1e-3
    g = torch.Generator().manual_seed(21)
    x = torch.rand(n, d, generator=g)
    y = torch.sin(3 * x.double().sum(-1)).float() + 0.03 * torch.randn(n, generator=g)
    xt = torch.rand(m, d, generator=g)
    axes = _oracle_axes([64, 64])
    xj = torch.cat([x, xt]).double()
    Kj = ski.ski_matmul("rbf", xj, [a.double() for a in axes], ls0, os0, torch.eye(n + m, dtype=torch.float64))
    Kj = 0.5 * (Kj + Kj.t())
    Lc = torch.linalg.cholesky(Kj[:n, :n].to(cuda_dev) + float(torch.tensor(nz0)) * torch.eye(n, dtype=torch.float64, device=cuda_dev))
    mean_ref = Kj[n:, :n].to(cuda_dev) @ torch.cholesky_solve(y.double().to(cuda_dev)[:, None], Lc)[:, 0]
    iters, means = {}, {}
    for flag in (False, True):
        model, lik = _ski_model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), 64, d, nz0)
        model.covar_module.base_kernel.base_kernel.lengthscale = ls0
        model.covar_module.outputscale = os0
        model.eval(); lik.eval()
        with torch.no_grad(), settings.ski_preconditioner(flag), settings.eval_cg_tolerance(1e-5), settings.max_cg_iterations(4000):
            khat = lik(model.forward(x.to(cuda_dev))).lazy_covariance_matrix     # the prior K_ski + sigma^2 I of the mean cache
            with settings._use_eval_tolerance(True):
                _, _, iters[flag] = operators._run_cg(khat, y.to(cuda_dev)[:, None], 0, khat._preconditioner()[0])
            means[flag] = model(xt.to(cuda_dev)).mean
    print(f"\nmean-cache CG iterations: {iters[False]} without, {iters[True]} with the SKI preconditioner; "
          f"mean rel err {rel(means[False], mean_ref):.2e} / {rel(means[True], mean_ref):.2e}")
    assert iters[True] <= 0.6 * iters[False]
    assert rel(means[True], mean_ref) < 1e-2 and rel(means[False], mean_ref) < 1e-2


def test_ski_training_step_with_the_preconditioner(cuda_dev, monkeypatch):
    """test_gpu_ski.py's training step with settings.ski_preconditioner on: loss and gradients against dense fp64 autograd."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.engine import Plan
    from oracle import mll as om

    calls = []
    orig = Plan.pivoted_cholesky
    monkeypatch.setattr(Plan, "pivoted_cholesky", lambda self, *a, **kw: calls.append(1) or orig(self, *a, **kw))
    n, d, sizes, ls0, os0, nz0 = 2000, 2, [26, 26], 0.3, 1.2, 0.25
    x, y = om.synthetic_problem(n, d, 6, torch.float32)
    axes = _oracle_axes(sizes)
    model, lik = _ski_model(cuda_dev, x.to(cuda_dev), y.to(cuda_dev), 26, d, nz0)
    model.covar_module.base_kernel.base_kernel.lengthscale = ls0
    model.covar_module.outputscale = os0
    model.train(); lik.train()
    with settings.ski_preconditioner(True), settings.probe_seed(5), settings.cg_tolerance(1e-3), settings.num_trace_samples(15):
        loss = -gp.mlls.ExactMarginalLogLikelihood(lik, model)(model(x.to(cuda_dev)), y.to(cuda_dev))
        loss.backward()
    assert calls
    ls = torch.tensor(ls0, dtype=torch.float64, requires_grad=True)
    osc = torch.tensor(os0, dtype=torch.float64, requires_grad=True)
    nz = torch.tensor(nz0, dtype=torch.float64, requires_grad=True)
    Kd = ski.ski_matmul("rbf", x.double(), [a.double() for a in axes], ls, osc, torch.eye(n, dtype=torch.float64))
    Kd = 0.5 * (Kd + Kd.t()) + nz * torch.eye(n, dtype=torch.float64)
    Lc = torch.linalg.cholesky(Kd)
    r = y.double().unsqueeze(-1)
    ref = 0.5 * ((r * torch.cholesky_solve(r, Lc)).sum() + 2 * Lc.diagonal().log().sum() + n * math.log(2 * math.pi)) / n
    ref.backward()
    assert loss.item() == pytest.approx(ref.item(), rel=3e-2, abs=2e-3)
    k = model.covar_module

    def raw_grad(p):
        return p.grad.item() / torch.sigmoid(p).item()

    assert raw_grad(k.base_kernel.base_kernel.raw_lengthscale) == pytest.approx(ls.grad.item(), rel=0.2, abs=3e-3)
    assert raw_grad(k.raw_outputscale) == pytest.approx(osc.grad.item(), rel=0.2, abs=3e-3)
    assert raw_grad(lik.raw_noise) == pytest.approx(nz.grad.item(), rel=0.2, abs=3e-3)


@pytest.mark.parametrize("noise,k,t,Q", [(0.05, 30, 4, 15), (1e-2, 100, 16, 8)])
def test_ciq_precond_on_ski_matches_fp64(cuda_dev, noise, k, t, Q):
    """gp_ciq_precond_build + gp_ciq_sqrt_matmul_precond on a SKI plan against K_hat F^-T sum_q w_q (A + tau_q)^-1 b in fp64; the trace of
    the interval is the fp64 sum of the SKI diagonal; fewer msMINRES iterations than unpreconditioned on the true spectrum."""
    from gpytorch_b200.sampling import contour_quadrature

    n, sizes, ls, os_ = 2000, [32, 32], 0.2, 1.3
    x, axes, lo, steps = pow2_points(sizes, n, seed=k + t)
    p = _ski_plan(cuda_dev, x, lo, steps, sizes, "rbf", ls, os_, noise)
    first, w, T = interp_and_factors("rbf", x, axes, ls)
    K = dense64(first, w, T, os_)
    lt, _, st = p.pivoted_cholesky(k, 0.0)
    assert st == 0 and lt.size(0) == k
    u, tr_e, st = p.ciq_precond_build(lt)
    assert st == 0 and torch.isfinite(u).all()
    tr_dev = float(p.diag().double().sum())
    assert abs(tr_e - (tr_dev - float((lt.double() ** 2).sum()))) <= 1e-6 * tr_dev
    assert abs(tr_dev - float(K.trace())) <= 1e-5 * float(K.trace())
    d = torch.full((n,), float(torch.tensor(noise, dtype=torch.float32)), dtype=torch.float64)
    m, M = 0.5, 2.0 * (1.0 + max(tr_e, 1e-6 * float(K.trace())) / float(d.min()))
    tau, wq = contour_quadrature(m, M, Q)
    b = torch.randn(n, t, generator=torch.Generator().manual_seed(k))
    out, info = p.ciq_sqrt_matmul(b.to(cuda_dev), tau, wq, tol=1e-6, max_iter=600, warn=False, precond_u=u)
    assert torch.isfinite(out).all() and info.precond_rank == k
    L, W, finv_t, Khat, A, fnorm = _factor64(K, d, lt, u, cuda_dev)
    e, V = torch.linalg.eigh(A)
    lo_a, hi_a = float(e[0]), float(e[-1])
    assert 0.5 <= lo_a and hi_a <= M
    bd = b.double().to(cuda_dev)
    filt = sum(wj / (e + tj) for tj, wj in zip(tau, wq))
    fz = finv_t @ (V @ (filt[:, None] * (V.T @ bd)))
    ref = Khat @ fz
    nk = float(torch.linalg.matrix_norm(Khat, 2))
    res = torch.tensor(info.residual_norms, dtype=torch.float64)
    for c in range(t):
        gap = sum(wj * (float(res[j, c]) + min(1.0, 2e-5 * (hi_a + tj) / (lo_a + tj))) for j, (tj, wj) in enumerate(zip(tau, wq)))
        bound = fnorm * float(bd[:, c].norm()) * gap + 1e-5 * nk * float(fz[:, c].norm())
        err = float((out.double()[:, c] - ref[:, c]).norm())
        assert err <= bound, (c, err, bound, info.iters)
    lo_k, hi_k = (float(v) for v in torch.linalg.eigvalsh(Khat)[[0, -1]])
    tau0, w0 = contour_quadrature(lo_k, hi_k * 1.01, Q)
    _, info0 = p.ciq_sqrt_matmul(b.to(cuda_dev), tau0, w0, tol=1e-6, max_iter=600, warn=False)
    print(f"\nSKI sigma^2={noise} k={k}: {info.iters} msMINRES iterations preconditioned, {info0.iters} without")
    assert info.iters < info0.iters
    p.close()


def test_rsample_with_ski_preconditioner_matches_fp64(cuda_dev):
    """likelihood(model(x)).rsample with ciq_samples + ciq_preconditioner + ski_preconditioner equals F A^{1/2} xi (fp64 eigh) for the
    same xi, F from the engine's U."""
    from gpytorch_b200 import settings

    n, d = 2000, 2
    g = torch.Generator().manual_seed(8)
    x = torch.rand(n, d, generator=g)
    model, lik = _ski_model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev), 30, d, 0.02)
    model.covar_module.base_kernel.base_kernel.lengthscale = 0.25
    model.covar_module.outputscale = 1.1
    model.train(); lik.train()
    with settings.ciq_samples(True), settings.ciq_preconditioner(True), settings.ski_preconditioner(True), \
            settings.max_preconditioner_size(40), torch.no_grad():
        torch.manual_seed(123)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.rsample(torch.Size([16]))
        op = dist.lazy_covariance_matrix
        lt = op._preconditioner()[1]
        u = op._ciq_cache[1][0]
    m_, M_, infos = op.last_ciq
    assert all(i.precond_rank == lt.size(0) == 40 for i in infos)
    torch.manual_seed(123)
    xi = torch.randn(n, 16, device=cuda_dev).double()
    axes = _oracle_axes([30, 30])
    K = ski.ski_matmul("rbf", x.double(), [a.double() for a in axes], 0.25, 1.1, torch.eye(n, dtype=torch.float64))
    K = 0.5 * (K + K.T)
    dvec = torch.full((n,), float(lik.noise.detach().cpu()), dtype=torch.float64)
    _, _, finv_t, _, A, _ = _factor64(K, dvec, lt, u, cuda_dev)
    ref = torch.linalg.solve(finv_t.T, _sqrt_psd(A) @ xi)          # F = (F^-T)^-T
    err = ((s.double().T - ref).norm(dim=0) / ref.norm(dim=0)).max().item()
    print(f"\nSKI rsample: iters {[i.iters for i in infos]}, [m, M] = [{m_:.3g}, {M_:.3g}], max rel err {err:.2e}")
    assert err <= 1e-3


def test_ski_precond_sample_moments(cuda_dev):
    """N = 64, S = 4096 preconditioned CIQ draws of a SKI model: the moment bound of tests/test_gpu_sampling.py."""
    from gpytorch_b200 import settings

    n, S, d = 64, 4096, 2
    x = torch.rand(n, d, generator=torch.Generator().manual_seed(64))
    model, lik = _ski_model(cuda_dev, x.to(cuda_dev), torch.zeros(n, device=cuda_dev), 10, d, 0.1)
    model.covar_module.base_kernel.base_kernel.lengthscale = 0.5
    model.covar_module.outputscale = 1.2
    model.train(); lik.train()
    with settings.ciq_samples(True), settings.ciq_preconditioner(True), settings.ski_preconditioner(True), \
            settings.min_preconditioning_size(0), settings.max_preconditioner_size(10), torch.no_grad():
        torch.manual_seed(5)
        dist = lik(model(x.to(cuda_dev)))
        s = dist.sample(torch.Size([S])).cpu().double()
        assert all(i.precond_rank == 10 for i in dist.lazy_covariance_matrix.last_ciq[2])
    axes = _oracle_axes([10, 10])
    A = ski.ski_matmul("rbf", x.double(), [a.double() for a in axes], 0.5, 1.2, torch.eye(n, dtype=torch.float64))
    A = 0.5 * (A + A.T) + float(lik.noise.detach().cpu()) * torch.eye(n, dtype=torch.float64)
    Ch = s.T @ s / S
    assert float((Ch - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_flag_off_leaves_ski_unpreconditioned(cuda_dev, monkeypatch):
    """settings.ski_preconditioner off (the default): SKI MLL, prediction and CIQ sampling (even with ciq_preconditioner on) never
    call the pivoted Cholesky, and CIQ reports precond_rank == 0."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.engine import Plan

    def boom(self, *a, **kw):
        raise AssertionError("pivoted Cholesky called on a SKI operator with settings.ski_preconditioner off")

    monkeypatch.setattr(Plan, "pivoted_cholesky", boom)
    n, d = 2500, 2
    g = torch.Generator().manual_seed(4)
    x = torch.rand(n, d, generator=g).to(cuda_dev)
    y = torch.sin(3 * x.sum(-1))
    model, lik = _ski_model(cuda_dev, x, y, 30, d, 0.1)
    model.train(); lik.train()
    assert settings.ski_preconditioner.off()
    with settings.probe_seed(1), settings.cg_tolerance(1e-2):
        loss = -gp.mlls.ExactMarginalLogLikelihood(lik, model)(model(x), y)
        loss.backward()
    with settings.ciq_samples(True), settings.ciq_preconditioner(True), torch.no_grad():
        dist = lik(model(x))
        dist.rsample(torch.Size([4]))
        assert all(i.precond_rank == 0 for i in dist.lazy_covariance_matrix.last_ciq[2])
    model.eval(); lik.eval()
    with torch.no_grad():
        pred = model(torch.rand(10, d, generator=g).to(cuda_dev))
    assert torch.isfinite(pred.mean).all()
