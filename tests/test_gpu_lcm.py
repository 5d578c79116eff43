"""The Kronecker operator with several terms (LCMKernel, gp_plan_set_kron_terms) on the H100: products entry by entry within the
bounds of tests/lcm_oracle.py over Q, T, column counts, backends, kinds, active dimensions and cross plans; Q = 1 bit for bit
against gp_plan_set_kron; determinism; rows, diagonal and pivots; gradients per term; solves, the MLL, Lanczos and CIQ against
dense fp64; NaN propagation; the C refusals; and LCMKernel models end to end (the reference's LCM / ICM equivalence, a two-term
model's MLL gradients and posterior against fp64, CIQ samples)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import kmv_oracle as ko  # noqa: E402
import lcm_oracle as lo  # noqa: E402
import multitask_oracle as mo  # noqa: E402

RATIOS = {}
KINDS = ["rbf", "matern12", "matern52"]


def _within(key, got, ref, bnd):
    got = torch.as_tensor(got, dtype=torch.float64).cpu()
    ref, bnd = torch.as_tensor(ref, dtype=torch.float64).cpu(), torch.as_tensor(bnd, dtype=torch.float64).cpu()
    err = (got - ref).abs()
    frac = torch.where(bnd > 0, err / bnd, torch.where(err > 0, torch.inf, 0.0))
    w = int(frac.argmax())
    assert bool(torch.isfinite(got).all()) and float(frac.max()) <= 1.0, (key, w, float(err.reshape(-1)[w]), float(bnd.reshape(-1)[w]))
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(frac.max()))


def _build(dev, Q, T, backends, n=700, n2=None, d=4, seed=0, ard=False):
    """Q data plans (kind, lengthscale, outputscale, backend and active dimensions per term), the LcmPlan and the oracle terms."""
    from gpytorch_b200.engine import LcmPlan, Plan

    x = ko.points(n, d, seed)
    x2 = ko.points(n2, d, seed + 1) if n2 else None
    datas, terms = [], []
    for q in range(Q):
        dims = list(range(d)) if q == 0 else [c for c in range(d) if c != q % d]
        xq, x2q = x[:, dims].contiguous(), None if x2 is None else x2[:, dims].contiguous()
        kind, ls, os_ = KINDS[q % 3], (0.25 + 0.35 * q), 0.8 + 0.4 * q
        be = backends[q % len(backends)]
        lsv = [ls * (1 + 0.1 * c) for c in range(len(dims))] if ard else ls
        p = Plan(xq.to(dev), None if x2q is None else x2q.to(dev), backend=be).set_hypers(kind, lsv, os_, 0.0)
        assert p.info()["backend"] == be
        datas.append(p)
        terms.append(lo.term(kind, xq.to(dev), None if x2q is None else x2q.to(dev),
                             torch.tensor(lsv, dtype=torch.float64) if ard else ls, os_, mo.random_B(T, seed + 10 + q), be,
                             p.info()["n_sm"]))
    lp = LcmPlan(datas, T)
    lp.set_noise(0.0)
    lp.set_term_covars(torch.stack([tm["B"] for tm in terms]))
    return lp, datas, terms


@pytest.mark.parametrize("Q", [2, 3, 4])
@pytest.mark.parametrize("T", [1, 3, 8])
@pytest.mark.parametrize("cols", [16, 33, 512])
def test_products_within_bound(cuda_dev, Q, T, cols):
    t = max(1, cols // T) if cols != 512 else 16   # T t = 16, 33 (cross the chunk edge) and 512 columns of W
    t = {16: max(1, 16 // T), 33: max(1, -(-33 // T))}.get(cols, t)
    backends = [["tcgen05"], ["simt"], ["tcgen05", "simt"]][(Q + T) % 3]
    lp, _, terms = _build(cuda_dev, Q, T, backends, n=700 + 13 * Q)
    V = torch.randn(terms[0]["x1"].size(0) * T, t, generator=torch.Generator().manual_seed(Q * 100 + T))
    got = lp.kmv(V.to(cuda_dev))
    _within(("kmv", tuple(backends)), got, lo.exact(terms, V, T, t), lo.bound(terms, V, T, t))


@pytest.mark.parametrize("backends", [["tcgen05"], ["simt"], ["tcgen05", "simt"]])
def test_cross_products_and_ard_within_bound(cuda_dev, backends):
    T, t = 3, 5
    lp, _, terms = _build(cuda_dev, 2, T, backends, n=333, n2=517, ard=True)
    V = torch.randn(517 * T, t, generator=torch.Generator().manual_seed(4))
    _within(("kmv_cross", tuple(backends)), lp.kmv(V.to(cuda_dev)), lo.exact(terms, V, T, t), lo.bound(terms, V, T, t))


def test_one_term_is_bit_identical_to_gp_plan_set_kron_and_calls_repeat(cuda_dev):
    from gpytorch_b200.engine import KronPlan, LcmPlan, Plan

    T = 3
    x = ko.points(900, 3, 5).to(cuda_dev)
    data = Plan(x, backend="tcgen05").set_hypers("matern52", 0.4, 1.3, 0.0)
    B = mo.random_B(T, 6)
    kp = KronPlan(data, T).set_noise(0.1)
    kp.set_task_covar(B)
    lp = LcmPlan([data], T).set_noise(0.1)
    lp.set_term_covars(B[None])
    V = torch.randn(900 * T, 7, device=cuda_dev)
    assert torch.equal(kp.kmv(V, True), lp.kmv(V, True))
    gl, go = kp.bilinear_grad(V, V)
    tl, to, tdB = lp.terms_grad(V, V)
    assert tl[0] == gl and to[0] == go and torch.equal(tdB[0], kp.task_covar_grad(V, V))
    lp2, _, _ = _build(cuda_dev, 3, 4, ["tcgen05", "simt"])
    V2 = torch.randn(lp2.n2, 11, device=cuda_dev)
    a, b = lp2.kmv(V2), lp2.kmv(V2)
    assert torch.equal(a, b)
    g1, g2 = lp2.terms_grad(V2, V2), lp2.terms_grad(V2, V2)
    assert g1[0] == g2[0] and g1[1] == g2[1] and torch.equal(g1[2], g2[2])


def test_rows_diagonal_and_pivots(cuda_dev):
    T = 3
    lp, _, terms = _build(cuda_dev, 3, T, ["tcgen05", "simt"], n=300)
    A = lo.dense([dict(tm, x1=tm["x1"].cpu()) for tm in terms])
    idx = torch.tensor([0, 1, 2, 5, 299 * T + 2, 150 * T + 1])
    _within(("rows",), lp.rows(idx.to(cuda_dev)), A[idx], lo.rows_bound([dict(tm, x1=tm["x1"].cpu()) for tm in terms], idx))
    d = torch.diagonal(A)
    _within(("diag",), lp.diag(), d, (len(terms) + 1) * lo.U32 * d.abs() + lo.ROW_REL * sum(abs(tm["os"]) * torch.diagonal(
        tm["B"].double()).abs().repeat(300) for tm in terms))
    lt, piv, st = lp.pivoted_cholesky(12, 0.0)
    assert st == 0
    assert int(piv[0]) == int(torch.argmax(d))
    Lt = lt.double().cpu()
    # the factor reproduces its pivot rows of K (a greedy partial Cholesky interpolates its pivots' rows)
    P = piv.cpu()
    err = (Lt.t()[P] @ Lt - A[P]).abs().max()
    assert float(err) <= 1e-3 * float(A.abs().max()), float(err)


def test_gradients_per_term_within_bound(cuda_dev):
    T, t = 3, 4
    lp, _, terms = _build(cuda_dev, 3, T, ["tcgen05", "simt"], n=600)
    L = torch.randn(600 * T, t, generator=torch.Generator().manual_seed(11))
    R = torch.randn(600 * T, t, generator=torch.Generator().manual_seed(12))
    gl, go, dB = lp.terms_grad(L.to(cuda_dev), R.to(cuda_dev))
    for q, ((el, es, edB), (bl, bs, bdB)) in enumerate(zip(lo.grads(terms, L, R, T, t), lo.grads_bound(terms, L, R, T, t, lp.info()["n_sm"]))):
        _within(("grad_ls",), torch.tensor(gl[q]), torch.as_tensor(el).reshape(-1).cpu(), torch.as_tensor(bl).reshape(-1).cpu())
        _within(("grad_os",), torch.tensor([go[q]]), torch.tensor([float(es)]), torch.tensor([float(bs)]))
        _within(("dB",), dB[q], edB, bdB)


def test_solves_mll_lanczos_and_ciq_against_dense(cuda_dev):
    T, n, noise = 2, 400, 0.5   # a noise level at which 10 probes and 60 Lanczos steps estimate log det to a few percent
    lp, _, terms = _build(cuda_dev, 2, T, ["tcgen05", "simt"], n=n)
    lp.set_noise(noise)
    A = lo.dense([dict(tm, x1=tm["x1"].cpu()) for tm in terms]) + noise * torch.eye(n * T, dtype=torch.float64)
    y = torch.randn(n * T, generator=torch.Generator().manual_seed(2)).to(cuda_dev)
    want = torch.linalg.solve(A, y.double().cpu())
    for rank in (0, 10):
        w = None
        if rank:
            lt, _, _ = lp.pivoted_cholesky(rank)
            w, _, _ = lp.precond_build(lt)
        sol, _, info = lp.mbcg(y[:, None], tolerance=1e-5, max_iter=2000, precond_w=w)
        assert float((sol[:, 0].double().cpu() - want).abs().max()) <= 1e-3 * float(want.abs().max()), (rank, info)
    L = torch.linalg.cholesky(A)
    ld = 2 * torch.log(torch.diagonal(L)).sum()
    for rank in (0, 10):
        g = torch.Generator(device=cuda_dev).manual_seed(0)
        tp = 10
        rad = (torch.randint(0, 2, (n * T, tp), device=cuda_dev, generator=g).float() * 2 - 1)
        eps1 = torch.randn(rank or 1, tp, device=cuda_dev, generator=g)
        eps2 = torch.randn(n * T, tp, device=cuda_dev, generator=g)
        res, _ = lp.mll(y, eps1, eps2, rad, num_probes=tp, precond_rank=rank, min_precond_size=1 if rank else 10 ** 9, cg_tol=1e-5,
                        max_tridiag_iter=60)
        iq = float(y.double().cpu() @ want)
        assert abs(res.inv_quad - iq) <= 1e-3 * abs(iq)
        assert abs(res.logdet - float(ld)) <= 0.05 * abs(float(ld)) + 10.0, (rank, res.logdet, float(ld))
    q, tm = lp.lanczos(torch.ones(n * T, device=cuda_dev), 30)
    top = float(torch.linalg.eigvalsh(tm.double().cpu()).max())
    assert abs(top - float(torch.linalg.eigvalsh(A).max())) <= 1e-3 * top
    ev, U = torch.linalg.eigh(A)
    sq = U @ torch.diag(ev.sqrt()) @ U.t()
    from gpytorch_b200.sampling import contour_quadrature
    tau, wq = contour_quadrature(float(ev.min()), float(ev.max()) * 1.01, 15)
    b = torch.randn(n * T, 2, device=cuda_dev)
    out, _ = lp.ciq_sqrt_matmul(b, tau, wq, tol=1e-6, max_iter=2000)
    ref = sq @ b.double().cpu()
    assert float((out.double().cpu() - ref).abs().max()) <= 1e-2 * float(ref.abs().max())


def test_nan_from_one_term_or_one_B(cuda_dev):
    from gpytorch_b200.engine import LcmPlan, Plan

    T, n = 3, 200
    x = ko.points(n, 2, 1).to(cuda_dev)
    xb = x.clone()
    xb[17, 1] = float("nan")
    good = Plan(x, backend="simt").set_hypers("rbf", 0.5, 1.0, 0.0)
    bad = Plan(xb, backend="tcgen05").set_hypers("matern52", 0.5, 1.0, 0.0)
    lp = LcmPlan([good, bad], T).set_noise(0.1)
    Bs = torch.stack([mo.random_B(T, 1), mo.random_B(T, 2)])
    lp.set_term_covars(Bs)
    V = torch.randn(n * T, 3, device=cuda_dev)
    assert bool(torch.isnan(lp.kmv(V)).all())
    lp2 = LcmPlan([good, Plan(x, backend="tcgen05").set_hypers("matern12", 0.3, 1.0, 0.0)], T).set_noise(0.1)
    lp2.set_term_covars(Bs)
    assert bool(torch.isfinite(lp2.kmv(V)).all())
    Bs2 = Bs.clone()
    Bs2[1, 0, 2] = float("inf")
    lp2.set_term_covars(Bs2)
    assert bool(torch.isnan(lp2.kmv(V)).all())


def test_c_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    lib = _lib.load()
    T = 2
    x = ko.points(100, 2, 3).to(cuda_dev)
    d1 = Plan(x, backend="simt").set_hypers("rbf", 0.5, 1.0, 0.0)
    d2 = Plan(x, backend="tcgen05").set_hypers("matern32", 0.5, 1.0, 0.0)
    p = Plan(x, backend="simt").set_hypers("rbf", 0.5, 1.0, 0.1)
    parent = C.c_void_p()
    stream = torch.cuda.current_stream(cuda_dev).cuda_stream
    assert lib.gp_plan_create(C.byref(parent), cuda_dev.index or 0, C.c_void_p(stream)) == 0
    arr = lambda ps: (C.c_void_p * len(ps))(*[q._h.value for q in ps])
    assert lib.gp_plan_set_kron_terms(parent, arr([d1] * 5), 5, T) == _lib.GP_E_SHAPE
    assert lib.gp_plan_set_kron_terms(parent, arr([d1, d2]), 0, T) == _lib.GP_E_SHAPE
    assert lib.gp_plan_set_kron_terms(parent, arr([d1, d2]), 2, 33) == _lib.GP_E_SHAPE
    other = Plan(ko.points(101, 2, 4).to(cuda_dev), backend="simt").set_hypers("rbf", 0.5, 1.0, 0.0)
    assert lib.gp_plan_set_kron_terms(parent, arr([d1, other]), 2, T) == _lib.GP_E_SHAPE
    rq = Plan(x, backend="simt").set_hypers_rq(0.5, 1.0, 1.0, 0.0)
    assert lib.gp_plan_set_kron_terms(parent, arr([d1, rq]), 2, T) == _lib.GP_E_STATE
    assert lib.gp_plan_set_kron_terms(parent, arr([d1, d2]), 2, T) == 0
    assert lib.gp_plan_set_hypers(parent, _lib.KIND["rbf"], (C.c_float * 1)(1.0), 1, 1.0, 0.1) == 0
    one = (C.c_float * (T * T))(*([1.0] * (T * T)))
    two = (C.c_float * (2 * T * T))(*([1.0, 0.2, 0.2, 1.0] * 2))
    assert lib.gp_plan_set_task_covar(parent, one, T) == _lib.GP_E_STATE
    assert b"gp_plan_set_kron_term_covars" in lib.gp_last_error()
    assert lib.gp_plan_set_kron_term_covars(parent, two, 3, T) == _lib.GP_E_SHAPE
    assert lib.gp_plan_set_kron_term_covars(parent, two, 2, T) == 0
    z = torch.zeros(100 * T, 1, device=cuda_dev)
    g = (C.c_double * 4)()
    pz = C.c_void_p(z.data_ptr())
    assert lib.gp_bilinear_grad(parent, pz, 1, pz, 1, 1, g, g) == _lib.GP_E_STATE
    assert b"gp_kron_terms_grad" in lib.gp_last_error()
    assert lib.gp_task_covar_grad(parent, pz, 1, pz, 1, 1, g) == _lib.GP_E_STATE
    assert lib.gp_plan_set_kron_observed(parent, None, 0, None, 0) == _lib.GP_E_STATE
    assert lib.gp_plan_set_kron_terms(parent, None, 0, 0) == 0
    lib.gp_plan_destroy(parent)


# ---- LCMKernel models ------------------------------------------------------------------------------------------------------------
def _model(gp, train_x, train_y, T, covar):
    class M(gp.models.ExactGP):
        def __init__(self):
            lik = gp.likelihoods.MultitaskGaussianLikelihood(num_tasks=T)
            super().__init__(train_x, train_y, lik)
            self.mean_module = gp.means.MultitaskMean(gp.means.ConstantMean(), num_tasks=T)
            self.covar_module = covar

        def forward(self, x):
            return gp.distributions.MultitaskMultivariateNormal(self.mean_module(x), self.covar_module(x))

    return M()


def test_lcm_icm_equivalence(cuda_dev):
    import gpytorch_b200 as gp

    torch.manual_seed(0)
    train_x = torch.linspace(0, 1, 100, device=cuda_dev)
    y1 = torch.sin(train_x * (2 * math.pi)) + torch.randn(train_x.size(), device=cuda_dev) * 0.2
    y2 = torch.cos(train_x * (2 * math.pi)) + torch.randn(train_x.size(), device=cuda_dev) * 0.2
    train_y = torch.stack([y1, y2], -1)
    means = []
    for covar in (lambda: gp.kernels.LCMKernel([gp.kernels.RBFKernel()], num_tasks=2, rank=1),
                  lambda: gp.kernels.MultitaskKernel(gp.kernels.RBFKernel(), num_tasks=2, rank=1)):
        torch.manual_seed(1)
        model = _model(gp, train_x, train_y, 2, covar()).to(cuda_dev)
        opt = torch.optim.Adam(model.parameters(), lr=0.1)
        model.train()
        mll = gp.mlls.ExactMarginalLogLikelihood(model.likelihood, model)
        for _ in range(50):
            opt.zero_grad()
            loss = -mll(model(train_x), train_y)
            loss.backward()
            opt.step()
        model.eval()
        with torch.no_grad():
            means.append(model.likelihood(model(torch.linspace(0, 1, 51, device=cuda_dev))).mean)
    assert float((means[0] - means[1]).pow(2).mean()) < 1e-2


def _two_term(gp, cuda_dev, n=300, T=4):
    torch.manual_seed(3)
    x = torch.rand(n, 1, device=cuda_dev)
    y = torch.stack([torch.sin(6 * x[:, 0] + a) + 0.3 * torch.cos(x[:, 0] * (a + 1)) for a in range(T)], -1)
    y = y + 0.1 * torch.randn(n, T, device=cuda_dev)
    short = gp.kernels.RBFKernel()
    long_ = gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))
    covar = gp.kernels.LCMKernel([short, long_], num_tasks=T, rank=[1, 2])
    model = _model(gp, x, y, T, covar).to(cuda_dev)
    short.lengthscale = 0.1
    long_.base_kernel.lengthscale = 1.5
    long_.outputscale = 0.7
    model.likelihood.noise = 0.05
    return model, x, y


def _dense_mll(model, x, y, T):
    """fp64 dense ExactMarginalLogLikelihood of the two-term model, differentiable in every parameter."""
    terms = []
    for m in model.covar_module.covar_module_list:
        dm = m.data_covar_module
        base = getattr(dm, "base_kernel", dm)
        os_ = dm.outputscale.double() if hasattr(dm, "base_kernel") else 1.0
        kind = "rbf" if base.kind == "rbf" else base.kind
        terms.append(dict(kind=kind, x1=x.double(), x2=None, ls=base.lengthscale.double().reshape(()), os=os_,
                          B=m.task_covar_module.covar_matrix.double()))
    K = lo.dense([dict(tm, x1=tm["x1"]) for tm in terms])
    lik = model.likelihood
    n = x.size(0)
    tn = lik.task_noises.double() if hasattr(lik, "task_noises") and lik.task_noises is not None else torch.zeros(T, dtype=torch.float64, device=x.device)
    A = K + torch.diag((tn + lik.noise.double().reshape(-1)[:1]).repeat(n))
    mean = torch.stack([mm.constant.double().reshape(()) for mm in model.mean_module.base_means]) if hasattr(model.mean_module, "base_means") else 0.0
    r = (y.double() - mean).reshape(-1, 1)
    L = torch.linalg.cholesky(A)
    a = torch.cholesky_solve(r, L)
    N = r.numel()
    return -0.5 * ((r * a).sum() + 2 * torch.log(torch.diagonal(L)).sum() + N * math.log(2 * math.pi)) / N


def test_two_term_mll_gradients_against_dense_fp64(cuda_dev):
    import gpytorch_b200 as gp

    T = 4
    model, x, y = _two_term(gp, cuda_dev, T=T)
    model.train()
    mll = gp.mlls.ExactMarginalLogLikelihood(model.likelihood, model)
    seeds = 4   # the stochastic log det gradient, averaged over four probe sets
    got = {}
    for seed in range(seeds):
        model.zero_grad()
        with gp.settings.max_cholesky_size(0), gp.settings.cg_tolerance(1e-4), gp.settings.num_trace_samples(15), \
                gp.settings.probe_seed(seed):
            loss = -mll(model(x), y)
            loss.backward()
        for n, p in model.named_parameters():
            got[n] = got.get(n, 0.0) + p.grad.detach().clone() / seeds
    model.zero_grad()
    (-_dense_mll(model, x, y, T)).backward()
    for n, p in model.named_parameters():
        ref = p.grad.double()
        assert got[n] is not None, n
        # stochastic trace estimate (4 x 15 probes) against the exact log det gradient
        tol = 0.15 * float(ref.abs().max()) + 3e-3
        assert float((got[n].double() - ref).abs().max()) <= tol, (n, got[n], ref)
    assert any(n.startswith("covar_module.covar_module_list.1") for n in got)


@pytest.mark.parametrize("fast", [False, True])
def test_two_term_posterior_against_fp64(cuda_dev, fast):
    import gpytorch_b200 as gp

    T = 4
    model, x, y = _two_term(gp, cuda_dev, T=T)
    model.eval()
    xs = torch.rand(20, 1, device=cuda_dev)
    with torch.no_grad(), gp.settings.fast_pred_var(fast), gp.settings.max_cholesky_size(0), gp.settings.eval_cg_tolerance(1e-6):
        pred = model(xs)
        mu, cov = pred.mean, pred.covariance_matrix
    terms_tr, terms_x = [], []
    for m in model.covar_module.covar_module_list:
        dm = m.data_covar_module
        base = getattr(dm, "base_kernel", dm)
        os_ = float(dm.outputscale.detach()) if hasattr(dm, "base_kernel") else 1.0
        B = m.task_covar_module.covar_matrix.detach().double().cpu()
        ls = float(base.lengthscale.detach())
        terms_tr.append(dict(kind=base.kind, x1=x.double().cpu(), x2=None, ls=ls, os=os_, B=B))
        terms_x.append(dict(kind=base.kind, x1=torch.cat([x, xs]).double().cpu(), x2=None, ls=ls, os=os_, B=B))
    n = x.size(0)
    lik = model.likelihood
    noise = float(lik.noise) + (lik.task_noises.detach().double().cpu() if getattr(lik, "task_noises", None) is not None else torch.zeros(T, dtype=torch.float64))
    A = lo.dense(terms_tr) + torch.diag(torch.as_tensor(noise, dtype=torch.float64).expand(T).repeat(n))
    J = lo.dense(terms_x)
    Ksx, Kss = J[n * T:, :n * T], J[n * T:, n * T:]
    mean_tr = model.mean_module(x).detach().double().cpu()
    mean_s = model.mean_module(xs).detach().double().cpu()
    alpha = torch.linalg.solve(A, (y.double().cpu() - mean_tr).reshape(-1))
    mu_ref = (Ksx @ alpha).reshape(-1, T) + mean_s
    cov_ref = Kss - Ksx @ torch.linalg.solve(A, Ksx.t())
    assert float((mu.double().cpu() - mu_ref).abs().max()) <= 1e-3 * float(mu_ref.abs().max()) + 1e-4
    tol = (3e-2 if fast else 1e-3) * float(Kss.diagonal().max())
    assert float((cov.double().cpu() - cov_ref).abs().max()) <= tol


def test_two_term_ciq_rsample(cuda_dev):
    import gpytorch_b200 as gp

    model, x, y = _two_term(gp, cuda_dev, T=2)
    model.train()
    with torch.no_grad(), gp.settings.ciq_samples(True), gp.settings.max_cholesky_size(0):
        prior = model.likelihood(model(x))   # K + noise, as the Kronecker model's CIQ test samples it
        s = prior.rsample(torch.Size([64]))
    assert tuple(s.shape) == (64, x.size(0), 2) and bool(torch.isfinite(s).all())
    # the sample covariance of 64 draws is within a few standard errors of the prior diagonal
    var = s.reshape(64, -1).var(0).mean()
    d = prior.lazy_covariance_matrix.diagonal().mean()
    assert 0.5 * float(d) < float(var) < 1.6 * float(d)


def test_zz_report_fraction_of_bound(cuda_dev):
    print("\nlargest |engine - fp64| / bound (LCM):")
    for k, v in sorted(RATIOS.items(), key=str):
        print(f"  {k}: {v:.3g}")
