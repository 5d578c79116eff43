"""Kernel products on the device (run with -m gpu): ProductKernel (reference kernels/kernel.py:547-551, :634-690) as ONE engine
operator (gp_plan_set_product, csrc/product.cu).  Every comparison is against the fp64 oracle of tests/product_oracle.py: K.V entry
by entry within its derived bound on product_tc_kernel and product_simt_kernel (every pair of kinds, scalar and ARD lengthscales,
overlapping and disjoint active dimensions, square and cross plans, row / column edges, several column splits, a ring wrap, three
and four factors), rows, diagonal, pivoted Cholesky, the MLL, the hyper-parameter gradients, the refusals, and the public API
(k1 * k2, ScaleKernel over a product, training, prediction, sampling, fixed noise, NaN inputs)."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

import bilinear_oracle as bo  # noqa: E402
import kmv_oracle as ko  # noqa: E402
import product_oracle as po  # noqa: E402
from oracle import linalg as ol, mll as om  # noqa: E402

KINDS = list(bo.KINDS)


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _plans(dev, factors, x1, x2, backends, noise=0.0):
    """(product plan, factor plans, geometry mirror) for factors [(kind, dims, ls, os)]; asserts the kernel and split it reaches."""
    from gpytorch_b200.engine import Plan

    fp = []
    for (kind, dims, ls, os_), be in zip(factors, backends):
        a = po._slice(x1, dims).to(dev)
        b = None if x2 is None else po._slice(x2, dims).to(dev)
        fp.append(Plan(a, b, backend=be).set_hypers(kind, ls, os_, 0.0))
    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev)).set_product(fp).set_hypers("rbf", [1.0], 1.0, noise)
    info = p.info()
    n2 = x1.size(0) if x2 is None else x2.size(0)
    geo = po.geometry(x1.size(0), n2, [len(f[1]) for f in factors], backends, info["n_sm"])
    assert info["backend"] == "product" and info["nsplit"] == geo["nsplit"] and info["kpad"] == geo["KP"], (info, geo)
    return p, fp, geo


def _check(tag, factors, x1, x2, V, backends, noise=0.0, dev=None):
    dev = dev or torch.device("cuda:0")
    p, fp, geo = _plans(dev, factors, x1, x2, backends, noise)
    out = p.kmv(V.to(dev), add_noise=noise > 0)
    ref, bnd = po.kv_and_bound(factors, x1, x2, V.to(dev), geo["path"], geo["nsplit"], geo["T"], noise if x2 is None else 0.0)
    err = (out.double() - ref).abs()
    frac = torch.where(bnd > 0, err / bnd, torch.where(err > 0, torch.inf, 0.0))
    worst = int(frac.argmax())
    assert bool(torch.isfinite(out).all()) and float(frac.max()) <= 1.0, \
        (tag, geo, divmod(worst, frac.size(1)), float(err.view(-1)[worst]), float(bnd.view(-1)[worst]), float(ref.view(-1)[worst]))
    return p, fp, geo, out, ref


TC2, SIMT2 = ("tcgen05", "tcgen05"), ("simt", "simt")


@pytest.mark.parametrize("backends", [TC2, SIMT2])
def test_every_pair_of_kinds_within_bound(cuda_dev, backends):
    """16 ordered pairs of kinds; scalar and ARD lengthscales, overlapping ([0, 1, 2] x [2, 3]) and disjoint active dimensions,
    square (N not a multiple of 128 / 64) and cross plans; single entries through identity columns."""
    n, m, d = 333, 457, 5
    x1, x2 = ko.points(n, d, 1), ko.points(m, d, 2)
    for ia, ka in enumerate(KINDS):
        for ib, kb in enumerate(KINDS):
            ard = (ia + ib) % 2 == 1
            dims_a, dims_b = ([0, 1, 2], [2, 3]) if ia <= ib else ([0, 1], [2, 3, 4])
            la = [0.5, 0.8, 1.1][: len(dims_a)] if ard else 0.7
            factors = [(ka, dims_a, la, 1.3), (kb, dims_b, 0.6, 0.7)]
            square = (ia + 2 * ib) % 3 != 0
            xb = None if square else x2
            cols = n if square else m
            V, _ = ko.identity_cols(cols, [0, 63, 64, cols - 1])
            V = torch.cat([V, torch.randn(cols, 16 - V.size(1) + 1, generator=torch.Generator().manual_seed(ia * 4 + ib))], 1)
            p, fp, geo, _, _ = _check(f"{ka} x {kb}", factors, x1, xb, V, backends, noise=0.1 if square else 0.0, dev=cuda_dev)
            assert geo["path"] == ("tc" if backends is TC2 else "simt")
            for q in (p, *fp):
                q.close()


def test_tensor_core_splits_ring_wrap_and_repeatability(cuda_dev):
    """More than one column split, more column tiles per split than ring stages (KP_a + KP_b = 80 + 16: five stages, nine or more tiles), the
    tensor-core and CUDA-core kernels against each other, and repeated products bit for bit."""
    n, d = 6000, 26
    x = ko.points(n, d, 5)
    factors = [("rbf", list(range(24)), 2.0, 1.1), ("matern12", [24, 25], 0.4, 0.9)]
    V = torch.randn(n, 11, generator=torch.Generator().manual_seed(6))
    p, fp, geo, out, _ = _check("splits tc", factors, x, None, V, TC2, noise=0.05, dev=cuda_dev)
    assert geo["path"] == "tc" and geo["nsplit"] > 1 and geo["T"] > po.ring_depth(geo["KP"]) and geo["KP"] == 96, geo
    assert torch.equal(out, p.kmv(V.to(cuda_dev), add_noise=True))
    ps, fs, geo_s, out_s, ref = _check("splits simt", factors, x, None, V, SIMT2, noise=0.05, dev=cuda_dev)
    assert geo_s["path"] == "simt" and geo_s["nsplit"] > 1
    assert torch.equal(out_s, ps.kmv(V.to(cuda_dev), add_noise=True))
    assert rel(out, out_s) < 1e-5
    # the widest tensor-core product: KP_a + KP_b = 128
    xw = ko.points(700, 40, 7)
    fw = [("matern52", list(range(20)), 2.5, 1.0), ("matern32", list(range(20, 40)), 2.0, 1.0)]
    _, _, geo_w, _, _ = _check("KP 128", fw, xw, ko.points(900, 40, 8), torch.randn(900, 16, generator=torch.Generator().manual_seed(9)),
                               TC2, dev=cuda_dev)
    assert geo_w["path"] == "tc" and geo_w["KP"] == 128
    # one more column than fits: AUTO takes the CUDA-core kernel
    fo = [("matern52", list(range(20)), 2.5, 1.0), ("rbf", list(range(19, 40)), 2.0, 1.0)]
    _, _, geo_o, _, _ = _check("KP 136", fo, xw, None, torch.randn(700, 3, generator=torch.Generator().manual_seed(10)), TC2, dev=cuda_dev)
    assert geo_o["path"] == "simt"


def test_three_and_four_factors_on_cuda_cores(cuda_dev):
    n, m, d = 500, 300, 6
    x1, x2 = ko.points(n, d, 11), ko.points(m, d, 12)
    f3 = [("rbf", [0, 1], 0.6, 1.2), ("matern12", [2], 0.5, 0.8), ("matern52", [1, 3, 4, 5], [0.9, 1.0, 1.1, 1.2], 1.5)]
    f4 = f3 + [("matern32", [0, 5], 0.8, 0.6)]
    for fs in (f3, f4):
        for xb in (None, x2):
            cols = n if xb is None else m
            V = torch.randn(cols, 5, generator=torch.Generator().manual_seed(len(fs)))
            _, _, geo, _, _ = _check(f"{len(fs)} factors", fs, x1, xb, V, ("auto",) * len(fs), dev=cuda_dev)
            assert geo["path"] == "simt"


def test_rows_diag_pivots_mll_and_lanczos_match_oracle(cuda_dev):
    n, d, rank = 3000, 4, 40
    x, y = om.synthetic_problem(n, d, 2, torch.float32)
    factors = [("rbf", [0, 1, 2], 0.6, 1.2), ("matern12", [3], 1.5, 0.7)]
    S = 1.2 * 0.7
    K = po.dense(po.f32_factors(factors), x)
    g = torch.Generator().manual_seed(5)
    for backends in (TC2, SIMT2):
        p, fp, geo = _plans(cuda_dev, factors, x, None, backends, noise=0.1)
        idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
        assert rel(p.rows(idx), K[idx]) < 2e-6
        assert rel(p.diag(), K.diagonal()) < 1e-6
        lt, piv, st = p.pivoted_cholesky(rank, 1e-3)
        L, piv_o = ol.pivoted_cholesky(torch.full((n,), float(bo.f32(S)), dtype=torch.float64), lambda i: K[i], rank)
        assert st == 0 and torch.equal(piv.cpu(), piv_o)
        assert rel(lt.t(), L) < 1e-3
        pn = om.make_probe_noise(n, rank, 10, 7)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, S, 0.1, tuple(a.double() for a in pn), precond_size=rank, K=K)
            o32 = om.mll_bbmm("rbf", x, y, 0.0, 1.0, S, 0.1, pn, precond_size=rank, K=K.float())
        res, sol = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000, want_solve=True)
        assert res.cg_iters == o64.iters and res.precond_rank == rank
        assert abs(res.inv_quad - o64.inv_quad) <= max(1e-4 * abs(o64.inv_quad), 3 * abs(o32.inv_quad - o64.inv_quad))
        assert abs(res.logdet - o64.logdet) <= max(1e-4 * abs(o64.logdet), 3 * abs(o32.logdet - o64.logdet))
        # the dense value: 10 probes estimate the log-determinant, so the tolerance is 2 % of the terms' size, not of their sum
        lp, sol_ref = po.mll_cholesky(K, y, 0.1)
        size = (abs(o64.inv_quad) + abs(o64.logdet)) / (2 * n)
        assert abs(res.mll - lp.item()) < 0.02 * size + 1e-3
        assert rel(sol, sol_ref) < 1e-2
        # without a preconditioner (fixed Rademacher probes)
        res0, _ = p.mll(y.to(cuda_dev), None, None, pn[2].to(cuda_dev), 10, 0, 2000)
        assert res0.precond_rank == 0 and abs(res0.mll - lp.item()) < 0.05 * size + 1e-3
        # re-packing a factor (new outputscale / lengthscale) is picked up by the next call on the product
        fp[1].set_hypers("matern12", 1.1, 2.0, 0.0)
        Kb = po.dense(po.f32_factors([factors[0], ("matern12", [3], 1.1, 2.0)]), x)
        v = torch.randn(n, 7, generator=g)
        assert rel(p.kmv(v.to(cuda_dev)), Kb @ v.double()) < 5e-6
        q, t = p.lanczos(torch.randn(n, generator=g).to(cuda_dev), 12)
        qd = q.double().cpu()
        assert rel(t, qd.t() @ (Kb + 0.1 * torch.eye(n, dtype=torch.float64)) @ qd) < 1e-3
        # cross plan: rows and the diagonal of K(x1, x2) with equal sizes
        x2 = ko.points(n, d, 77)
        pc, fc, _ = _plans(cuda_dev, factors, x, x2, backends)
        Kc = po.dense(po.f32_factors(factors), x, x2)
        assert rel(pc.rows(idx), Kc[idx]) < 2e-6 and rel(pc.diag(), Kc.diagonal()) < 2e-6
        for q_ in (p, pc, *fp, *fc):
            q_.close()


@pytest.mark.parametrize("backends", [TC2, SIMT2])
def test_bilinear_grad_matches_fp64_autograd(cuda_dev, backends):
    n, m, d, s = 700, 500, 5, 19
    x1, x2 = ko.points(n, d, 21), ko.points(m, d, 22)
    g = torch.Generator().manual_seed(23)
    cases = [([("rbf", [0, 1, 2], [0.5, 0.8, 1.1], 1.3), ("matern12", [3, 4], 0.6, 0.7)], None),
             ([("matern52", [0, 1], 0.9, 0.9), ("matern32", [1, 2, 3], [0.7, 1.0, 1.3], 1.6)], x2),
             ([("matern12", [0], 0.4, 1.1), ("rbf", [1, 2, 3, 4], 1.0, 0.8)], None)]
    for factors, xb in cases:
        cols = n if xb is None else m
        L, R = torch.randn(n, s, generator=g), torch.randn(cols, s, generator=g)
        p, fp, _ = _plans(cuda_dev, factors, x1, xb, backends)
        gl, go = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
        ref = po.bilinear_grads(factors, x1, xb, L, R)
        S = math.prod(float(bo.f32(f[3])) for f in factors)
        k = 0
        for f, (rl, rs) in zip(factors, ref):
            nl = rl.numel()
            scale = max(1.0, float(rl.abs().max()))
            assert torch.allclose(torch.tensor(gl[k:k + nl], dtype=torch.float64), rl.reshape(-1), rtol=2e-4, atol=2e-4 * scale), (f, gl, rl)
            assert go * S / float(bo.f32(f[3])) == pytest.approx(rs.item(), rel=2e-4, abs=2e-4), (f, go, rs)
            k += nl
        assert k == len(gl)
        for q in (p, *fp):
            q.close()


def test_refusals_and_nan(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import KronPlan, Plan

    x = torch.rand(500, 3, device=cuda_dev)
    pa = Plan(x[:, :2].contiguous()).set_hypers("rbf", 0.6, 1.0, 0.0)
    pb = Plan(x[:, 2:].contiguous()).set_hypers("matern12", 0.6, 1.0, 0.0)
    pshort = Plan(x[:400, 2:].contiguous()).set_hypers("rbf", 0.6, 1.0, 0.0)
    pp = Plan(x).set_product([pa, pb]).set_hypers("rbf", [1.0], 1.0, 0.1)
    before = pp.launches()
    lib = pp.lib

    def status(fn, *args):
        return fn(*args), _lib.last_error()

    import ctypes as C
    arr = (C.c_void_p * 2)(pp._h.value, pa._h.value)
    other = Plan(x).set_hypers("rbf", [1.0], 1.0, 0.1)
    for name, call in [
        ("gp_plan_set_sum", lambda: lib.gp_plan_set_sum(other._h, arr, 2)),
        ("gp_plan_set_product", lambda: lib.gp_plan_set_product(other._h, arr, 2)),
        ("gp_plan_set_kron", lambda: lib.gp_plan_set_kron(other._h, pp._h, 2)),
        ("gp_plan_set_deriv", lambda: lib.gp_plan_set_deriv(other._h, pp._h)),
        ("gp_plan_set_tasks", lambda: lib.gp_plan_set_tasks(pp._h, C.c_void_p(x.data_ptr()), None, 2)),
        ("gp_plan_set_lowrank", lambda: lib.gp_plan_set_lowrank(pp._h, C.c_void_p(x.data_ptr()), 3, 3)),
        ("gp_plan_set_ski", lambda: lib.gp_plan_set_ski(pp._h, (C.c_int * 3)(8, 8, 8), (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 1, 1), 3)),
        ("gp_plan_set_backend", lambda: lib.gp_plan_set_backend(pp._h, 2)),
        ("gp_kmv_input_grad", lambda: lib.gp_kmv_input_grad(pp._h, C.c_void_p(x.data_ptr()), 1, C.c_void_p(x.data_ptr()), 1, 1,
                                                            C.c_void_p(x.data_ptr()), 3, None, 3)),
        ("gp_kdense_input_grad", lambda: lib.gp_kdense_input_grad(pp._h, C.c_void_p(x.data_ptr()), 500, C.c_void_p(x.data_ptr()), 3, None, 3)),
    ]:
        st, msg = status(call)
        assert st == _lib.GP_E_STATE and ("product" in msg), (name, st, msg)
    assert pp.launches() == before
    with pytest.raises(RuntimeError, match="differs from the product"):
        Plan(x).set_hypers("rbf", [1.0], 1.0, 0.1).set_product([pa, pshort])
    with pytest.raises(RuntimeError, match="2 to 4 factors"):
        Plan(x).set_product([pa])
    sk = KronPlan(pa, 2).set_noise(0.0)
    with pytest.raises(RuntimeError, match="plain kernel plan"):
        Plan(x).set_hypers("rbf", [1.0], 1.0, 0.1).set_product([pa, sk])
    # a non-finite input in one factor: products, rows and gradients are NaN
    xn = x.clone()
    xn[7, 2] = float("nan")
    pn_ = Plan(xn[:, 2:].contiguous()).set_hypers("matern12", 0.6, 1.0, 0.0)
    pbad = Plan(xn).set_product([pa, pn_]).set_hypers("rbf", [1.0], 1.0, 0.1)
    v = torch.randn(500, 2, device=cuda_dev)
    assert bool(torch.isnan(pbad.kmv(v)).all())
    assert bool(torch.isnan(pbad.rows(torch.tensor([3]))).all())
    gl, go = pbad.bilinear_grad(v, v)
    assert all(math.isnan(t) for t in gl) and math.isnan(go)


def _space_time(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g)
    # smooth in (x0, x1), rough in x2: an Ornstein-Uhlenbeck-like path over a fine grid of x2 times a smooth envelope
    grid = torch.linspace(0, 1, 400)
    Kt = torch.exp(-(grid[:, None] - grid[None, :]).abs() / 0.15).double()
    path = (torch.linalg.cholesky(Kt + 1e-9 * torch.eye(400, dtype=torch.float64))
            @ torch.randn(400, generator=torch.Generator().manual_seed(99), dtype=torch.float64)).float()
    rough = path[(x[:, 2] * 399).round().long()]
    y = torch.sin(3 * x[:, 0]) * torch.cos(2 * x[:, 1]) * (1.0 + rough) + 0.05 * torch.randn(n, generator=g)
    return x, y


def _model(gp, xd, yd, lik, covar):
    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(xd, yd, lik)
            self.mean_module = gp.means.ZeroMean()
            self.covar_module = covar

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    return M().to(xd.device)


def test_api_product_kernel_mll_gradients_prediction_and_sampling(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import ProductKernelLinearOperator

    n = 2500
    x, y = _space_time(n, 1)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    lik = gp.likelihoods.GaussianLikelihood().to(cuda_dev)
    covar = gp.kernels.ScaleKernel(gp.kernels.ScaleKernel(gp.kernels.RBFKernel(active_dims=[0, 1]))
                                   * gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=0.5, active_dims=[2])))
    model = _model(gp, xd, yd, lik, covar)
    ka, kb = covar.base_kernel.kernels
    ka.base_kernel.lengthscale = 0.5; ka.outputscale = 0.9
    kb.base_kernel.lengthscale = 0.4; kb.outputscale = 0.6
    covar.outputscale = 1.7
    lik.noise = 0.2
    op = covar(xd)
    assert isinstance(op, ProductKernelLinearOperator) and len(op.ops) == 2
    fac = lambda l1, s1, l2, s2, so: [("rbf", [0, 1], l1, so * s1), ("matern12", [2], l2, s2)]  # noqa: E731
    K = po.dense(fac(0.5, 0.9, 0.4, 0.6, 1.7), x)
    assert rel(op.diagonal(), K.diagonal()) < 1e-6
    assert rel(op[:5].to_dense(), K[:5]) < 1e-5
    assert rel(covar(xd, diag=True), K.diagonal()) < 1e-6
    v = torch.randn(n, 3, device=cuda_dev)
    assert rel(op.matmul(v), K @ v.double().cpu()) < 2e-5
    mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
    model.train(); lik.train()
    with settings.max_preconditioner_size(50), settings.cg_tolerance(1e-3), settings.num_trace_samples(15), settings.probe_seed(3):
        loss = -mll(model(xd), yd)
        loss.backward()
    t = lambda v_: torch.tensor(v_, dtype=torch.float64, requires_grad=True)  # noqa: E731
    l1, s1, l2, s2, so, nz = t(0.5), t(0.9), t(0.4), t(0.6), t(1.7), t(0.2)
    Kd = po.dense(fac(l1, s1, l2, s2, so), x) + nz * torch.eye(n, dtype=torch.float64)
    Lc = torch.linalg.cholesky(Kd)
    r = y.double().unsqueeze(-1)
    ref = 0.5 * ((r * torch.cholesky_solve(r, Lc)).sum() + 2 * Lc.diagonal().log().sum() + n * math.log(2 * math.pi)) / n
    ref.backward()
    assert loss.item() == pytest.approx(ref.item(), rel=3e-2, abs=2e-3)

    def raw_grad(mod, name):   # chain rule through softplus: d raw = d value * sigmoid(raw)
        p = getattr(mod, name)
        return p.grad.item() / torch.sigmoid(p).item()

    # stochastic trace estimate with 15 probes: gradients agree to ~15 %
    for got, want in [(raw_grad(ka.base_kernel, "raw_lengthscale"), l1), (raw_grad(ka, "raw_outputscale"), s1),
                      (raw_grad(kb.base_kernel, "raw_lengthscale"), l2), (raw_grad(kb, "raw_outputscale"), s2),
                      (raw_grad(covar, "raw_outputscale"), so), (raw_grad(lik, "raw_noise"), nz)]:
        assert got == pytest.approx(want.grad.item(), rel=0.2, abs=3e-3)
    # the exact gradient path: K @ v through autograd against fp64 autograd through the dense product (rtol 2e-4)
    for p_ in model.parameters():
        p_.grad = None
    w = torch.randn(n, 3, device=cuda_dev)
    (w * covar(xd).matmul(v)).sum().backward()
    l1, s1, l2, s2, so = t(0.5), t(0.9), t(0.4), t(0.6), t(1.7)
    (w.double().cpu() * (po.dense(fac(l1, s1, l2, s2, so), x) @ v.double().cpu())).sum().backward()
    for got, want in [(raw_grad(ka.base_kernel, "raw_lengthscale"), l1), (raw_grad(ka, "raw_outputscale"), s1),
                      (raw_grad(kb.base_kernel, "raw_lengthscale"), l2), (raw_grad(kb, "raw_outputscale"), s2),
                      (raw_grad(covar, "raw_outputscale"), so)]:
        assert got == pytest.approx(want.grad.item(), rel=2e-4, abs=1e-3)
    # prediction: mean and variance (exact and fast_pred_var) against the dense fp64 posterior
    model.eval(); lik.eval()
    xt = torch.rand(40, 3, generator=torch.Generator().manual_seed(9))
    Kst = po.dense(fac(0.5, 0.9, 0.4, 0.6, 1.7), xt, x)
    Kss = po.dense(fac(0.5, 0.9, 0.4, 0.6, 1.7), xt)
    Ld = Lc.detach()
    mean_ref = Kst @ torch.cholesky_solve(r, Ld).squeeze(-1)
    var_ref = (Kss - Kst @ torch.cholesky_solve(Kst.t(), Ld)).diagonal()
    with torch.no_grad(), settings.eval_cg_tolerance(1e-4):
        pred = model(xt.to(cuda_dev))
        assert rel(pred.mean, mean_ref) < 2e-3
        assert rel(pred.variance, var_ref) < 2e-2
    model.train(); model.eval()
    with torch.no_grad(), settings.eval_cg_tolerance(1e-4), settings.fast_pred_var(True), settings.max_root_decomposition_size(200):
        predf = model(xt.to(cuda_dev))
        assert rel(predf.mean, mean_ref) < 2e-3
        # LOVE truncates the subtracted term to a rank-200 Lanczos root: within 2 % of the prior variance of the exact posterior
        assert float((predf.variance.double().cpu() - var_ref).abs().max()) < 0.02 * float(Kss.diagonal().max())
    # rsample with CIQ: |C_hat - K_hat|_F <= 3 sqrt((|K_hat|_F^2 + tr(K_hat)^2) / S) (Wishart variance), N = 64, S = 4096
    ns, S = 64, 4096
    small = _model(gp, xd[:ns], yd[:ns], lik, covar)
    small.train(); lik.train()
    with torch.no_grad(), settings.ciq_samples(True):
        torch.manual_seed(5)
        smp = lik(small(xd[:ns])).sample(torch.Size([S])).double().cpu()
    A = K[:ns, :ns] + 0.2 * torch.eye(ns, dtype=torch.float64)
    assert float((smp.t() @ smp / S - A).norm()) <= 3 * math.sqrt((float(A.norm()) ** 2 + float(A.trace()) ** 2) / S)


def test_api_training_beats_plain_rbf_and_fixed_noise(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n = 2000
    x, y = _space_time(n + 400, 2)
    xd, yd = x[:n].to(cuda_dev), y[:n].to(cuda_dev)
    xt, yt = x[n:].to(cuda_dev), y[n:]

    def fit(covar, lik):
        model = _model(gp, xd, yd, lik, covar)
        mll = gp.mlls.ExactMarginalLogLikelihood(lik, model)
        opt = torch.optim.Adam(list(model.parameters()) + [p for p in lik.parameters() if p.requires_grad], lr=0.1)
        model.train(); lik.train()
        losses = []
        with settings.max_preconditioner_size(30), settings.cg_tolerance(1e-2), settings.num_trace_samples(10), settings.probe_seed(1):
            for _ in range(25):
                opt.zero_grad()
                loss = -mll(model(xd), yd)
                loss.backward()
                opt.step()
                losses.append(loss.item())
        model.eval(); lik.eval()
        with torch.no_grad(), settings.eval_cg_tolerance(1e-3), settings.skip_posterior_variances(True):
            mae = (model(xt).mean.cpu() - yt).abs().mean().item()
        return losses, mae

    prod = gp.kernels.ScaleKernel(gp.kernels.RBFKernel(active_dims=[0, 1]) * gp.kernels.MaternKernel(nu=0.5, active_dims=[2]))
    lp, mae_p = fit(prod.to(cuda_dev), gp.likelihoods.GaussianLikelihood().to(cuda_dev))
    lr_, mae_r = fit(gp.kernels.ScaleKernel(gp.kernels.RBFKernel()).to(cuda_dev), gp.likelihoods.GaussianLikelihood().to(cuda_dev))
    assert lp[-1] < lp[0] - 0.05, lp
    assert mae_p < mae_r, (mae_p, mae_r)
    # FixedNoiseGaussianLikelihood: the per-row diagonal on a product plan
    noise = torch.full((n,), 0.05, device=cuda_dev) + 0.05 * torch.rand(n, device=cuda_dev)
    fl = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=noise).to(cuda_dev)
    covar = (gp.kernels.RBFKernel(active_dims=[0, 1]) * gp.kernels.MaternKernel(nu=0.5, active_dims=[2])).to(cuda_dev)
    model = _model(gp, xd, yd, fl, covar)
    model.train(); fl.train()
    with settings.max_preconditioner_size(30), settings.cg_tolerance(1e-3), settings.num_trace_samples(15), settings.probe_seed(2):
        out = gp.mlls.ExactMarginalLogLikelihood(fl, model)(model(xd), yd)
    ls = math.log(2.0)   # softplus(0)
    K = po.dense([("rbf", [0, 1], ls, 1.0), ("matern12", [2], ls, 1.0)], x[:n])
    Lc = torch.linalg.cholesky(K + torch.diag(noise.double().cpu()))
    r = y[:n].double().unsqueeze(-1)
    ref = -0.5 * ((r * torch.cholesky_solve(r, Lc)).sum() + 2 * Lc.diagonal().log().sum() + n * math.log(2 * math.pi)) / n
    assert out.item() == pytest.approx(ref.item(), rel=5e-2, abs=2e-3)   # 15 probes for the log-determinant
    # NaN in an input: NaN out (an error or a warning is fine), not a hang
    xb = xd.clone()
    xb[3, 2] = float("nan")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            res = covar(xb).matmul(torch.randn(n, 2, device=cuda_dev))
            assert bool(torch.isnan(res).all())
        except RuntimeError as e:
            assert "NaN" in str(e)
