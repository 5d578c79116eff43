"""Additive GPs on the device (run with -m gpu): sums of D one-dimensional RBF / Matern components and their interaction terms up
to degree M as ONE engine operator (gp_plan_set_additive, csrc/additive.cu).  Every comparison is against the fp64 oracle of
tests/additive_oracle.py: K.V entry by entry within its derived bound, rows, diagonal, pivots, the MLL, the hyper-parameter
gradients, NaN inputs, and the public API (.sum(dim=-3), sum_interaction_terms, training, prediction, sampling)."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

import additive_oracle as ao  # noqa: E402
from oracle import linalg as ol, mll as om  # noqa: E402
import pivchol_oracle as po  # noqa: E402

KINDS = ["rbf", "matern12", "matern32", "matern52"]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _points(n, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, D, generator=g) * 4 - 2


def _hyp(D, seed, shared):
    g = torch.Generator().manual_seed(seed)
    ls = (torch.rand(D, generator=g) * 1.2 + 0.4).tolist()
    sc = (torch.rand(D, generator=g) * 1.0 + 0.3).tolist()
    if shared:   # an unbatched kernel: one value broadcast to every component
        ls, sc = [ls[0]] * D, [sc[0]] * D
    return ls, sc


def _plan(dev, kind, X1, X2, ls, sc, M, noise=0.0):
    from gpytorch_b200.engine import Plan

    return Plan(X1.to(dev), None if X2 is None else X2.to(dev)).set_additive(M, sc).set_hypers(kind, ls, 1.0, noise)


CASES = [  # kind, D, M, n1, n2 (None: square), t, shared
    ("rbf", 1, 1, 63, None, 1, False),
    ("matern12", 2, 2, 129, 63, 11, True),
    ("matern32", 7, 3, 4099, None, 16, False),
    ("matern52", 7, 8, 129, 1, 11, False),
    ("rbf", 32, 8, 1, 129, 16, True),
    ("matern52", 32, 2, 4099, 129, 1, False),
    ("rbf", 7, 1, 4099, 4099, 11, True),
    ("matern12", 32, 3, 129, None, 11, False),
    ("matern32", 2, 8, 63, 4099, 16, False),
    ("rbf", 2, 3, 129, None, 16, False),
    ("matern32", 1, 8, 4099, None, 11, True),
    ("matern52", 7, 4, 4099, None, 11, False),
    ("rbf", 32, 4, 129, 63, 16, True),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-D{c[1]}-M{c[2]}-n{c[3]}x{c[4]}-t{c[5]}-{'shared' if c[6] else 'per'}" for c in CASES])
def test_kmv_within_bound(cuda_dev, case):
    kind, D, M, n1, n2, t, shared = case
    X1 = _points(n1, D, 11 + D)
    X2 = None if n2 is None else _points(n2, D, 13 + D)
    ls, sc = _hyp(D, 3 + D, shared)
    p = _plan(cuda_dev, kind, X1, X2, ls, sc, M)
    assert p.info()["backend"] == "simt"
    Xb = X1 if X2 is None else X2
    V = torch.randn(Xb.size(0), t, generator=torch.Generator().manual_seed(5))
    out = p.kmv(V.to(cuda_dev)).double().cpu()
    X1d, Xbd = X1.double().to(cuda_dev), Xb.double().to(cuda_dev)
    exact = (ao.additive_dense(kind, X1d, Xbd, ls, sc, M) @ V.double().to(cuda_dev)).cpu()
    bound = ao.kmv_bound(kind, X1d, Xbd, ls, sc, M, V.to(cuda_dev)).cpu()
    err = (out - exact).abs()
    assert bool((err <= bound).all()), f"max err/bound {(err / bound).max().item():.3g}"
    p.close()


def test_d1_matches_plain_plan_and_m1_matches_kernel_sum(cuda_dev):
    from gpytorch_b200.engine import Plan
    from gpytorch_b200.operators import KernelLinearOperator, SumKernelLinearOperator

    n = 2000
    X = _points(n, 4, 7).to(cuda_dev)
    V = torch.randn(n, 11, device=cuda_dev)
    p1 = _plan(cuda_dev, "matern52", X[:, :1].contiguous(), None, [0.7], [1.3], 1)
    q1 = Plan(X[:, :1].contiguous(), backend="simt").set_hypers("matern52", [0.7], 1.3, 0.0)
    assert rel(p1.kmv(V), q1.kmv(V)) < 1e-6
    ls, sc = [0.5, 0.8, 1.1, 0.9], [1.2, 0.6, 0.9, 1.4]
    cols = [X[:, i:i + 1].contiguous() for i in range(4)]
    terms = [KernelLinearOperator(cols[i], None, "rbf", torch.tensor(ls[i], device=cuda_dev), torch.tensor(sc[i], device=cuda_dev))
             for i in range(4)]
    s4 = SumKernelLinearOperator(terms)
    pa = _plan(cuda_dev, "rbf", X, None, ls, sc, 1)
    assert rel(pa.kmv(V), s4.matmul(V)) < 2e-6


U32 = 2.0 ** -24


@pytest.mark.parametrize("kind", KINDS)
def test_pivots_match_fp64_oracle(cuda_dev, kind):
    """PC_KIND_ADDITIVE entries: the same pivot sequence as the fp64 greedy pivoting of the dense operator.  Step 0 is a tie of the
    constant diagonal, broken to the lowest index on both sides; from step 1 on the inputs are chosen so that no two candidates
    lie within the fp32 error of the residual diagonal (asserted, not assumed)."""
    n, D, M, rank = 600, 5, 2, 20
    x = _points(n, D, 102)
    ls, sc = _hyp(D, 9, False)
    K = ao.additive_dense(kind, x.double(), x.double(), ls, sc, M)
    kd = ao.esym_sum([torch.tensor(s, dtype=torch.float64) for s in sc], M).item()
    diag32 = torch.full((n,), float(torch.tensor(kd, dtype=torch.float32)), dtype=torch.float64)
    L, piv_o = ol.pivoted_cholesky(diag32, lambda i: K[i], rank)
    gaps = po.pivot_gaps(diag32, L, piv_o)
    assert gaps[0] == 0.0 and min(gaps[1:]) > 2 ** 4 * (rank + 1) * U32 * kd
    p = _plan(cuda_dev, kind, x, None, ls, sc, M, noise=0.1)
    lt, piv, st = p.pivoted_cholesky(rank, 1e-3)
    assert st == 0 and lt.size(0) == L.size(1) == rank
    assert torch.equal(piv.cpu(), piv_o)
    ltd, Lt64 = lt.double().cpu(), L.t()
    for m in range(rank):
        pm = int(piv_o[m])
        assert float((ltd[m] - Lt64[m]).abs().max()) <= 2 ** 8 * (m + 1) * U32 * kd / float(Lt64[m, pm])
    p.close()


# |MLL(fp32 oracle) - MLL(fp64 oracle)| with these probes and preconditioner: rbf 6.2e-5, matern12 1.41e-3, matern32 3.6e-5,
# matern52 6.0e-6.  The smooth kinds are held to 1e-4; the rough Matern-1/2 sum, whose Krylov quantities move by 1.4e-3 under fp32
# rounding in the oracle itself, to three times that distance.
@pytest.mark.parametrize("kind", KINDS)
def test_rows_diag_and_mll(cuda_dev, kind):
    n, D, M, rank = 2500, 5, 2, 30
    x, y = om.synthetic_problem(n, D, 4, torch.float32)
    ls, sc = _hyp(D, 9, False)
    K = ao.additive_dense(kind, x.double(), x.double(), ls, sc, M)
    p = _plan(cuda_dev, kind, x, None, ls, sc, M, noise=0.1)
    idx = torch.tensor([0, 1, 63, 64, n - 1, 17])
    assert rel(p.rows(idx), K[idx]) < 2e-6
    kd = ao.esym_sum([torch.tensor(s, dtype=torch.float64) for s in sc], M).item()
    assert torch.allclose(p.diag().double().cpu(), torch.full((n,), kd, dtype=torch.float64), rtol=1e-6)
    pn = om.make_probe_noise(n, rank, 10, 7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o64 = om.mll_bbmm("rbf", x.double(), y.double(), 0.0, 1.0, kd, 0.1, tuple(a.double() for a in pn), precond_size=rank, K=K)
        o32 = om.mll_bbmm("rbf", x, y, 0.0, 1.0, kd, 0.1, pn, precond_size=rank, K=K.float())
    res, sol = p.mll(y.to(cuda_dev), pn[0].to(cuda_dev), pn[1].to(cuda_dev), pn[2].to(cuda_dev), 10, rank, 2000, want_solve=True)
    assert res.precond_rank == rank and res.cg_iters == o64.iters
    tol = 3 * abs(o32.mll - o64.mll) if kind == "matern12" else 1e-4 * max(1.0, abs(o64.mll))
    assert abs(res.mll - o64.mll) <= tol
    Kh = K + 0.1 * torch.eye(n, dtype=torch.float64)
    Lc = torch.linalg.cholesky(Kh)
    yd = y.double()
    alpha = torch.cholesky_solve(yd.reshape(-1, 1), Lc).reshape(-1)
    lp = -0.5 * (yd @ alpha + 2 * Lc.diagonal().log().sum() + n * math.log(2 * math.pi)) / n
    assert abs(res.mll - lp.item()) < 0.02 * max(1.0, abs(lp.item()))
    # cross plan: rows and the diagonal of K(x1, x2) with equal sizes
    x2 = _points(n, D, 77)
    pc = _plan(cuda_dev, kind, x, x2, ls, sc, M)
    Kc = ao.additive_dense(kind, x.double(), x2.double(), ls, sc, M)
    assert rel(pc.rows(idx), Kc[idx]) < 2e-6 and rel(pc.diag(), Kc.diagonal()) < 2e-6
    p.close(), pc.close()


@pytest.mark.parametrize("kind,D,M", [("rbf", 3, 1), ("matern52", 5, 2), ("matern12", 10, 3), ("matern32", 9, 8), ("rbf", 20, 4)])
def test_bilinear_grad_matches_fp64_autograd(cuda_dev, kind, D, M):
    n, m, s = 600, 450, 13
    x1, x2 = _points(n, D, 21), _points(m, D, 22)
    ls, sc = _hyp(D, 23, False)
    g = torch.Generator().manual_seed(24)
    L, R = torch.randn(n, s, generator=g), torch.randn(m, s, generator=g)
    p = _plan(cuda_dev, kind, x1, x2, ls, sc, M)
    gl, gs = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    lt = torch.tensor(ls, dtype=torch.float64, requires_grad=True)
    st = torch.tensor(sc, dtype=torch.float64, requires_grad=True)
    cs = []
    for i in range(D):
        r = (x1[:, i].double().reshape(-1, 1) - x2[:, i].double().reshape(1, -1)).abs() / lt[i]
        if kind == "rbf":
            k = torch.exp(-0.5 * r * r)
        else:
            nu = ao.NU[kind]
            dd = math.sqrt(2 * nu) * r
            k = torch.exp(-dd) * (1 if nu == 0.5 else (1 + dd if nu == 1.5 else 1 + dd + dd * dd / 3))
        cs.append(st[i] * k)
    F = (L.double() * (ao.esym_sum(cs, M) @ R.double())).sum()
    F.backward()
    assert torch.allclose(torch.tensor(gl, dtype=torch.float64), lt.grad, rtol=2e-4, atol=2e-4 * lt.grad.abs().max().item())
    assert torch.allclose(torch.tensor(gs, dtype=torch.float64), st.grad, rtol=2e-4, atol=2e-4 * st.grad.abs().max().item())
    p.close()


def test_nan_inputs_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan

    n, D = 300, 3
    x = _points(n, D, 31)
    x[5, 1] = float("nan")
    p = _plan(cuda_dev, "rbf", x, None, [0.5] * D, [1.0] * D, 2)
    V = torch.randn(n, 3, device=cuda_dev)
    assert bool(p.kmv(V).isnan().all())
    assert bool(p.rows(torch.tensor([0, 1])).isnan().all()) and bool(p.diag().isnan().all())
    gl, gs = p.bilinear_grad(V, V)
    assert all(math.isnan(v) for v in gl + gs)
    q = _plan(cuda_dev, "rbf", _points(n, D, 32), None, [0.5] * D, [1.0] * D, 2)
    with pytest.raises(RuntimeError, match="gp_plan_set_backend is not available on an additive plan"):
        _lib.check(q.lib.gp_plan_set_backend(q._h, 2))
    with pytest.raises(RuntimeError, match="gp_kmv_input_grad is not available on an additive plan"):
        q.kmv_input_grad(V, V)
    other = Plan(_points(n, D, 33).to(cuda_dev)).set_hypers("rbf", [0.5], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="an additive plan as a term is not available"):
        other.set_sum([q])
    with pytest.raises(RuntimeError, match="an additive plan as a factor is not available"):
        other.set_product([q, q])
    for r in (p, q, other):
        r.close()


def _additive_model(train_x, train_y, M, kind="rbf"):
    import gpytorch_b200 as gp
    from gpytorch_b200 import kernels, likelihoods, means, models
    from gpytorch_b200.utils import sum_interaction_terms

    d = train_x.size(-1)

    class AdditiveGP(models.ExactGP):
        def __init__(self):
            super().__init__(train_x, train_y, likelihoods.GaussianLikelihood())
            self.mean_module = means.ConstantMean()
            base = kernels.RBFKernel(batch_shape=torch.Size([d]), ard_num_dims=1) if kind == "rbf" else \
                kernels.MaternKernel(nu=2.5, batch_shape=torch.Size([d]), ard_num_dims=1)
            self.covar_module = kernels.ScaleKernel(base)

        def forward(self, X):
            mean = self.mean_module(X)
            batched = self.covar_module(X.mT.unsqueeze(-1))
            covar = batched.sum(dim=-3) if M == 1 else sum_interaction_terms(batched, max_degree=M, dim=-3)
            return gp.distributions.MultivariateNormal(mean, covar)

    return AdditiveGP().to(train_x.device)


def _dense_posterior(model, train_x, train_y, test_x, M):
    """fp64 posterior mean / variance of the model's current hyper-parameters (the dense oracle)."""
    ck = model.covar_module
    ls = ck.base_kernel.lengthscale.detach().reshape(-1).double().cpu().tolist()
    sc = ck.outputscale.detach().reshape(-1).double().cpu().tolist()
    kind = getattr(ck.base_kernel, "kind")
    noise = float(model.likelihood.noise.detach().reshape(-1)[0])
    mu = float(model.mean_module.constant.detach().reshape(-1)[0])
    xt, xs = train_x.double().cpu(), test_x.double().cpu()
    Kxx = ao.additive_dense(kind, xt, xt, ls, sc, M) + noise * torch.eye(xt.size(0), dtype=torch.float64)
    Ksx = ao.additive_dense(kind, xs, xt, ls, sc, M)
    kss = ao.esym_sum([torch.tensor(s, dtype=torch.float64) for s in sc], M)
    sol = torch.linalg.solve(Kxx, torch.cat([(train_y.double().cpu() - mu).reshape(-1, 1), Ksx.t()], 1))
    mean = mu + Ksx @ sol[:, 0]
    var = kss - (Ksx * sol[:, 1:].t()).sum(1)
    return mean, var


@pytest.mark.parametrize("M", [1, 2])
def test_tutorial_models_train_predict_and_sample(cuda_dev, M):
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    torch.manual_seed(0)
    n, d = 600, 6
    train_x = torch.rand(n, d, device=cuda_dev)
    train_y = (torch.sin(3 * train_x[:, 0]) + train_x[:, 1] * train_x[:, 2] + 0.05 * torch.randn(n, device=cuda_dev)).contiguous()
    model = _additive_model(train_x, train_y, M)
    model.train()
    mll = gp.ExactMarginalLogLikelihood(model.likelihood, model)
    opt = torch.optim.Adam(model.parameters(), lr=0.1)
    losses = []
    with settings.max_cholesky_size(0):
        for _ in range(8):
            opt.zero_grad()
            loss = -mll(model(train_x), train_y)
            loss.backward()
            losses.append(loss.item())
            opt.step()
        assert losses[-1] < losses[0]
        assert model.covar_module.base_kernel.raw_lengthscale.grad is not None
        model.eval()
        test_x = torch.rand(50, d, device=cuda_dev)
        mean_o, var_o = _dense_posterior(model, train_x, train_y, test_x, M)
        with torch.no_grad(), settings.eval_cg_tolerance(1e-6):   # the posterior solves to well below the checked tolerance
            f = model(test_x)
            # fp32 solves of K + sigma^2 I: 2e-3 relative (the M = 2 model measured 1.2e-3 against the fp64 posterior)
            assert rel(f.mean, mean_o) < 2e-3
            assert rel(f.variance, var_o) < 2e-2
            with settings.fast_pred_var():
                f2 = model(test_x)
                assert rel(f2.mean, mean_o) < 2e-3
                assert rel(f2.variance.clamp_min(0), var_o) < 5e-2
            with settings.ciq_samples(True):
                s1 = model(test_x).rsample(torch.Size([3]))
                assert s1.shape == (3, 50) and bool(torch.isfinite(s1).all())
            with settings.fast_pred_var(), settings.fast_pred_samples():
                s2 = model(test_x).rsample(torch.Size([4]))
                assert s2.shape == (4, 50) and bool(torch.isfinite(s2).all())
