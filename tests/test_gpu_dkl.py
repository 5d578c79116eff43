"""Deep kernel learning on the GPU: gp_ski_input_grad against the fp64 closed form (tests/dkl_oracle.py), and MLL gradients
reaching a feature extractor through exact, kernel-sum and KISS-GP operators via the public API.

Bounds, derived, not tuned (u = 2^-24):
  * gp_ski_input_grad.  Every term of the closed form is a product of fp32 factors summed in fp32: the scatter W^T R (<= n terms per
    node), d 3xTF32 mode products (G_i terms each, 2^-22 per product), the outputscale, 4^d interpolation terms, t columns and two
    sides.  First order, worst case with one sign: |engine - fp64| <= k u * mag with k = n + sum_i 4 G_i + 2 4^d + 2 t + 16, mag the
    same formula with every factor replaced by its absolute value (dkl_oracle.ski_input_grad).  The weights come from t = (x - lo)
    / step in fp32, off by 2 u G in the cell fraction; the Keys kernel is C^1 with |w''| <= 5, so that adds 20 G u of mag.  Points
    within 1e-4 of the two nodes where the one-hot cells begin are kept out (there the derivative jumps).
  * API, Cholesky branch.  The engine and the fp64 reference differ by the fp32 Cholesky of K_hat, kappa(K_hat) u with
    kappa <= 1 + n s / sigma^2 = 1 + 150 * 1.5 / 0.5 = 451 (Higham, Thm 10.3): 3e-5 of the gradient's scale; plus the input-gradient
    primitive, (n + 40) u of the magnitudes (1e-5).  1e-4 of max |gradient| per parameter.
  * API, CG branch.  With fixed probes the estimator's fp64 value is the gradient of a surrogate with the solves held fixed; the
    engine solves by CG to 1e-6 (relative residual), so its solves agree to kappa 1e-6 = 5e-4 of their scale: 2e-3 of max |gradient|.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from dkl_oracle import dense_ski, ski_input_grad  # noqa: E402
from oracle import kernels as ok  # noqa: E402

GP_E_SHAPE, GP_E_STATE = 1, 7
U = 2.0 ** -24
SIZES = {1: [37], 2: [23, 17], 3: [12, 9, 14], 4: [6, 7, 5, 8]}


def _grid(sizes):
    step = [1.0 / (g - 2) for g in sizes]
    lo = [-s for s in step]
    lo32 = [float(torch.tensor(v, dtype=torch.float32)) for v in lo]
    st32 = [float(torch.tensor(v, dtype=torch.float32)) for v in step]
    axes = [torch.tensor(a, dtype=torch.float64) + torch.tensor(s, dtype=torch.float64) * torch.arange(g, dtype=torch.float64)
            for a, s, g in zip(lo32, st32, sizes)]
    return lo32, st32, axes


def _points(n, sizes, g):
    lo, step, axes = _grid(sizes)
    x = torch.rand(n, len(sizes), generator=g) * 0.98 + 0.01
    for i, (a, s) in enumerate(zip(lo, step)):
        x[0, i] = a + 0.5 * s                            # first cell (one-hot)
        x[1, i] = axes[i][-2] + 0.5 * s                  # last cell (one-hot)
        x[2, i] = axes[i][3]                             # on an interior node
    for i, ax in enumerate(axes):                        # away from the two edges of the one-hot cells
        for e in (float(ax[1]), float(ax[-2])):
            x[:, i] = torch.where((x[:, i] - e).abs() < 1e-4, x[:, i] + 3e-4, x[:, i])
    return x


def _ski_plan(dev, x, sizes, kind, ls, s):
    from gpytorch_b200.engine import Plan

    lo, step, _ = _grid(sizes)
    return Plan(x.to(dev)).set_ski(sizes, lo, step).set_hypers(kind, ls, s, 0.0)


@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("t", [1, 11, 40])
def test_ski_input_grad_matches_fp64(cuda_dev, d, t):
    g = torch.Generator().manual_seed(100 * d + t)
    sizes, n = SIZES[d], 700
    x = _points(n, sizes, g)
    L, R = torch.randn(n, t, generator=g), torch.randn(n, t, generator=g)
    ls, s = [0.25 + 0.1 * i for i in range(d)], 1.3
    plan = _ski_plan(cuda_dev, x, sizes, "rbf" if d != 3 else "matern52", ls, s)
    got = plan.ski_input_grad(L.to(cuda_dev), R.to(cuda_dev)).double().cpu()
    ref, mag = ski_input_grad("rbf" if d != 3 else "matern52", x.double(), _grid(sizes)[2], ls, s, L.double(), R.double())
    k = n + 4 * sum(sizes) + 2 * 4 ** d + 2 * t + 16 + 20 * max(sizes)
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= k * U * mag + 1e-30).all(), float((err / (k * U * mag + 1e-30)).max())
    assert torch.all(got[:2] == 0)                       # both coordinates in a one-hot cell: exactly zero


def test_ski_input_grad_is_deterministic_and_stride_free(cuda_dev):
    g = torch.Generator().manual_seed(5)
    sizes, n, t = SIZES[2], 3000, 11
    x = _points(n, sizes, g)
    plan = _ski_plan(cuda_dev, x, sizes, "rbf", [0.3, 0.4], 1.1)
    wide = torch.randn(n, 2 * t + 7, generator=g).to(cuda_dev)
    L, R = wide[:, 3:3 + t], wide[:, 5 + t:5 + 2 * t]
    a = plan.ski_input_grad(L.contiguous(), R.contiguous())
    b = plan.ski_input_grad(L, R)
    # the gradient pass itself has no atomics; its grid blocks come from the SKI scatter, whose per-tile red.add order varies,
    # so two calls agree to fp32 rounding of those sums (n u of the magnitudes), not bit for bit
    assert L.stride(0) == 2 * t + 7
    torch.testing.assert_close(a, b, rtol=0, atol=1e-5 * float(a.abs().max()))


def test_ski_input_grad_refusals_and_nan(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan, _ptr

    g = torch.Generator().manual_seed(6)
    sizes, n, t = SIZES[2], 200, 3
    x = _points(n, sizes, g)
    plan = _ski_plan(cuda_dev, x, sizes, "rbf", [0.3, 0.4], 1.1)
    L, R = torch.randn(n, t, generator=g).to(cuda_dev), torch.randn(n, t, generator=g).to(cuda_dev)
    out = torch.empty(n, 2, device=cuda_dev)

    def call(p, ldl=t, ldr=t, tt=t, ldo=2):
        return p.lib.gp_ski_input_grad(p._h, _ptr(L), ldl, _ptr(R), ldr, tt, _ptr(out), ldo)

    assert call(plan) == _lib.GP_OK
    assert call(plan, tt=0) == GP_E_SHAPE and call(plan, ldl=t - 1) == GP_E_SHAPE and call(plan, ldr=t - 1) == GP_E_SHAPE
    assert call(plan, ldo=1) == GP_E_SHAPE
    exact = Plan(x.to(cuda_dev)).set_hypers("rbf", 0.3, 1.0, 0.0)
    assert call(exact) == GP_E_STATE
    plan.set_lowrank(torch.randn(n, 2, device=cuda_dev))
    assert call(plan) == GP_E_STATE
    plan.set_lowrank(None)
    L[7, 1] = float("nan")
    dx = plan.ski_input_grad(L, R)
    assert torch.isnan(dx[7]).all()


# ---- through the API ------------------------------------------------------------------------------------------------------------
def _mlp(din, dout, seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(din, 8), torch.nn.Tanh(), torch.nn.Linear(8, dout))


def _exact_model(gp, case, x, y, net, dev):
    n = x.size(0)
    if case == "fixed":
        fixed = (0.4 + 0.2 * torch.rand(n, generator=torch.Generator().manual_seed(1))).to(dev)
        lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=fixed)
    else:
        lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.net = net
            self.mean_module = gp.means.ConstantMean()
            if case == "sum":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel()) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=1.5))
            elif case == "ard":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel(ard_num_dims=2, active_dims=[0, 2]))
            elif case == "matern":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=2.5))
            else:
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            z = self.net(xx)
            return gp.distributions.MultivariateNormal(self.mean_module(z), self.covar_module(z))

    model = M().to(dev)
    lik = lik.to(dev)
    if case == "sum":
        a, b = model.covar_module.kernels
        a.base_kernel.lengthscale = 0.7; a.outputscale = 1.0
        b.base_kernel.lengthscale = 1.1; b.outputscale = 0.5
        terms = [("rbf", [0, 1, 2], 0.7, 1.0), ("matern32", [0, 1, 2], 1.1, 0.5)]
    elif case == "ard":
        model.covar_module.base_kernel.lengthscale = torch.tensor([[0.6, 0.9]])
        model.covar_module.outputscale = 1.5
        terms = [("rbf", [0, 2], torch.tensor([0.6, 0.9], dtype=torch.float64), 1.5)]
    else:
        kind = "matern52" if case == "matern" else "rbf"
        model.covar_module.base_kernel.lengthscale = 0.8
        model.covar_module.outputscale = 1.5
        terms = [(kind, [0, 1, 2], 0.8, 1.5)]
    if case != "fixed":
        lik.noise = 0.5
    model.mean_module.constant = 0.2
    noise = fixed.double().cpu() if case == "fixed" else torch.full((n,), 0.5, dtype=torch.float64)
    return model, lik, terms, noise


def _dense_mll(net64, x64, y64, terms, noise, c=0.2):
    z = net64(x64)
    K = sum(ok.kernel_matrix(k, z[:, dims], z[:, dims], ls, s, True) for k, dims, ls, s in terms)
    Kh = K + torch.diag(noise)
    Lc = torch.linalg.cholesky(Kh)
    r = (y64 - c).unsqueeze(-1)
    iq = (r * torch.cholesky_solve(r, Lc)).sum()
    n = x64.size(0)
    return -0.5 * (iq + 2 * Lc.diagonal().log().sum() + n * torch.log(torch.tensor(2 * torch.pi, dtype=torch.float64))) / n


@pytest.mark.parametrize("case", ["rbf", "matern", "sum", "ard", "fixed"])
def test_exact_dkl_cholesky_gradients_match_fp64(cuda_dev, case):
    import copy

    import gpytorch_b200 as gp

    n = 150
    g = torch.Generator().manual_seed(11)
    x = torch.rand(n, 4, generator=g)
    y = torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(n, generator=g)
    net = _mlp(4, 3, 0)
    net64 = copy.deepcopy(net).double()
    model, lik, terms, noise = _exact_model(gp, case, x.to(cuda_dev), y.to(cuda_dev), net, cuda_dev)
    model.train(); lik.train()
    mll = gp.ExactMarginalLogLikelihood(lik, model)
    loss = -mll(model(x.to(cuda_dev)), y.to(cuda_dev))
    loss.backward()
    ref = -_dense_mll(net64, x.double(), y.double(), terms, noise)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-4 * max(1.0, abs(ref.item()))
    for (name, p), p64 in zip(model.net.named_parameters(), net64.parameters()):
        assert p.grad is not None, name
        err = (p.grad.double().cpu() - p64.grad).abs().max().item()
        assert err <= 1e-4 * p64.grad.abs().max().item() + 1e-7, (name, err)


def test_exact_dkl_cg_branch_matches_its_estimator(cuda_dev):
    import copy

    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n, tp = 300, 8
    g = torch.Generator().manual_seed(12)
    x = torch.rand(n, 4, generator=g)
    y = torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(n, generator=g)
    net = _mlp(4, 3, 1)
    net64 = copy.deepcopy(net).double()
    model, lik, terms, noise = _exact_model(gp, "rbf", x.to(cuda_dev), y.to(cuda_dev), net, cuda_dev)
    model.train(); lik.train()
    seed = 1234
    with settings.max_cholesky_size(0), settings.cg_tolerance(1e-6), settings.num_trace_samples(tp), settings.probe_seed(seed), \
            settings.max_lanczos_quadrature_iterations(50):
        out = model(x.to(cuda_dev))
        loss = -gp.ExactMarginalLogLikelihood(lik, model)(out, y.to(cuda_dev))
        loss.backward()
        # the same probes as the engine drew (no preconditioner below min_preconditioning_size: Rademacher columns)
        gen = torch.Generator(device=cuda_dev).manual_seed(seed)
        z = (torch.randint(0, 2, (n, tp), device=cuda_dev, generator=gen).to(torch.float32) * 2 - 1).double().cpu()
    zz = net64(x.double())
    kind, _, ls, s = terms[0]
    Kh = ok.kernel_matrix(kind, zz, zz, ls, s, True).detach() + torch.diag(noise)
    r = (y.double() - 0.2).unsqueeze(-1)
    alpha = torch.linalg.solve(Kh, r)
    u = torch.linalg.solve(Kh, z)
    K = ok.kernel_matrix(kind, zz, zz, ls, s, True)
    # d mll = -1/(2n) [ -alpha^T dK alpha + (1/tp) sum_i u_i^T dK z_i ]  (solves held fixed)
    surrogate = 0.5 / n * (-(alpha * (K @ alpha)).sum() + (u * (K @ z)).sum() / tp)
    surrogate.backward()
    scale = max(p64.grad.abs().max().item() for p64 in net64.parameters())   # the last bias has gradient 0 (a shift of stationary features)
    for (name, p), p64 in zip(model.net.named_parameters(), net64.parameters()):
        err = (p.grad.double().cpu() - p64.grad).abs().max().item()
        assert err <= 2e-3 * scale, (name, err, scale)


def test_exact_dkl_cg_inverse_quadratic_matches_dense(cuda_dev):
    import copy

    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n = 300
    g = torch.Generator().manual_seed(13)
    x = torch.rand(n, 4, generator=g)
    y = torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(n, generator=g)
    net = _mlp(4, 3, 2)
    net64 = copy.deepcopy(net).double()
    model, lik, terms, noise = _exact_model(gp, "rbf", x.to(cuda_dev), y.to(cuda_dev), net, cuda_dev)
    model.train(); lik.train()
    with settings.max_cholesky_size(0), settings.cg_tolerance(1e-6):
        out = lik(model(x.to(cuda_dev)))
        r = y.to(cuda_dev) - out.mean
        out.lazy_covariance_matrix.inv_quad(r.detach()).backward()
    zz = net64(x.double())
    kind, _, ls, s = terms[0]
    Kh = ok.kernel_matrix(kind, zz, zz, ls, s, True) + torch.diag(noise)
    r64 = (y.double() - 0.2).unsqueeze(-1)
    (r64 * torch.linalg.solve(Kh, r64)).sum().backward()
    scale = max(p64.grad.abs().max().item() for p64 in net64.parameters())   # the last bias has gradient 0 (a shift of stationary features)
    for (name, p), p64 in zip(model.net.named_parameters(), net64.parameters()):
        err = (p.grad.double().cpu() - p64.grad).abs().max().item()
        assert err <= 2e-3 * scale, (name, err, scale)


class _KissDKL:
    """The reference's KISS-GP DKL example: MLP (2 outputs) -> ScaleToBounds(-1, 1) -> ScaleKernel(GridInterpolationKernel(
    RBFKernel(ard_num_dims=2), grid_size, num_dims=2))."""

    @staticmethod
    def build(gp, x, y, grid_size, dev, seed=0):
        from gpytorch_b200.utils.grid import ScaleToBounds

        lik = gp.likelihoods.GaussianLikelihood()

        class M(gp.models.ExactGP):
            def __init__(self):
                super().__init__(x, y, lik)
                self.feature_extractor = _mlp(x.size(1), 2, seed)
                self.scale_to_bounds = ScaleToBounds(-1.0, 1.0)
                self.mean_module = gp.means.ConstantMean()
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.GridInterpolationKernel(
                    gp.kernels.RBFKernel(ard_num_dims=2), grid_size=grid_size, num_dims=2, grid_bounds=[(-1.0, 1.0), (-1.0, 1.0)]))

            def forward(self, xx):
                z = self.scale_to_bounds(self.feature_extractor(xx))
                return gp.distributions.MultivariateNormal(self.mean_module(z), self.covar_module(z))

        model = M().to(dev)
        return model, lik.to(dev)


def test_kiss_gp_dkl_gradients_match_the_ski_oracle_and_adam_trains(cuda_dev):
    import copy

    import gpytorch_b200 as gp
    from gpytorch_b200.utils.grid import ScaleToBounds

    n, G = 200, 100
    g = torch.Generator().manual_seed(21)
    x = torch.rand(n, 3, generator=g)
    y = torch.sin(4 * x[:, 0]) * x[:, 1] + 0.05 * torch.randn(n, generator=g)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model, lik = _KissDKL.build(gp, xd, yd, G, cuda_dev)
    model.covar_module.base_kernel.base_kernel.lengthscale = torch.tensor([[0.3, 0.4]])
    model.covar_module.outputscale = 1.2
    lik.noise = 0.3
    model.mean_module.constant = 0.1
    net64 = copy.deepcopy(model.feature_extractor).cpu().double()
    model.train(); lik.train()
    mll = gp.ExactMarginalLogLikelihood(lik, model)
    loss = -mll(model(xd), yd)
    loss.backward()
    lo, step = model.covar_module.base_kernel._grid()
    axes = [torch.tensor(a, dtype=torch.float64) + torch.tensor(s, dtype=torch.float64) * torch.arange(G, dtype=torch.float64)
            for a, s in zip(lo, step)]
    z = ScaleToBounds(-1.0, 1.0).double()(net64(x.double()))
    Kh = dense_ski("rbf", z, axes, [0.3, 0.4], 1.2) + 0.3 * torch.eye(n, dtype=torch.float64)
    Lc = torch.linalg.cholesky(Kh)
    r = (y.double() - 0.1).unsqueeze(-1)
    ref = 0.5 / n * ((r * torch.cholesky_solve(r, Lc)).sum() + 2 * Lc.diagonal().log().sum() + n * torch.log(torch.tensor(2 * torch.pi, dtype=torch.float64)))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-3 * max(1.0, abs(ref.item()))
    for (name, p), p64 in zip(model.feature_extractor.named_parameters(), net64.parameters()):
        assert p.grad is not None, name
        err = (p.grad.double().cpu() - p64.grad).abs().max().item()
        assert err <= 1e-3 * p64.grad.abs().max().item() + 1e-6, (name, err)
    # 30 Adam steps on everything, as the reference example trains
    opt = torch.optim.Adam(list(model.parameters()) + list(lik.parameters()), lr=0.01)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = -mll(model(xd), yd)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0] - 0.05, losses


def test_training_loop_keeps_plans_and_memory_flat_and_reused_plans_exact(cuda_dev):
    import gpytorch_b200 as gp
    from gpytorch_b200 import operators
    from gpytorch_b200.engine import Plan

    operators.clear_plan_cache()
    n, G = 3000, 40
    g = torch.Generator().manual_seed(22)
    x = torch.rand(n, 3, generator=g)
    y = torch.sin(4 * x[:, 0]) + 0.05 * torch.randn(n, generator=g)
    xd, yd = x.to(cuda_dev), y.to(cuda_dev)
    model, lik = _KissDKL.build(gp, xd, yd, G, cuda_dev)
    model.train(); lik.train()
    mll = gp.ExactMarginalLogLikelihood(lik, model)
    opt = torch.optim.Adam(list(model.parameters()) + list(lik.parameters()), lr=0.01)
    counts, mem, seen = [], [], set()
    for step in range(50):
        opt.zero_grad()
        loss = -mll(model(xd), yd)
        loss.backward()
        opt.step()
        counts.append(len(operators._PLAN_CACHE) + len(operators._SUM_PLANS))
        seen.update(id(p) for p in operators._PLAN_CACHE.values())
        torch.cuda.synchronize()
        mem.append(torch.cuda.memory_allocated(cuda_dev))
        if step == 4:
            torch.cuda.reset_peak_memory_stats(cuda_dev)
    peak = torch.cuda.max_memory_allocated(cuda_dev)
    assert max(counts[5:]) == counts[5] and counts[5] <= 3, counts
    assert len(seen) <= 3, len(seen)
    assert mem[-1] <= mem[5] + (1 << 20) and peak <= mem[5] + (512 << 20), (mem[5], mem[-1], peak)
    # a re-pointed plan computes what a fresh plan over the same inputs computes, bit for bit
    model.eval()
    with torch.no_grad():
        z = model.scale_to_bounds(model.feature_extractor(xd)).contiguous()
    op = model.covar_module(z)
    reused = op.plan()
    assert id(reused) in seen
    lo, step = model.covar_module.base_kernel._grid()
    ls = model.covar_module.base_kernel.base_kernel.lengthscale.detach().reshape(-1).tolist()
    fresh = Plan(z).set_ski([G, G], lo, step).set_hypers("rbf", ls, float(model.covar_module.outputscale), 0.0)
    # the re-packed interpolation data and grid factors: diagonal and interpolation are atomic-free passes over them
    assert torch.equal(reused.diag(), fresh.diag())
    c = torch.randn(G * G, 5, device=cuda_dev)
    assert torch.equal(reused.ski_interp_matmul(c), fresh.ski_interp_matmul(c))
    v = torch.randn(n, 5, device=cuda_dev)
    torch.testing.assert_close(reused.kmv(v), fresh.kmv(v), rtol=0, atol=1e-5 * float(fresh.kmv(v).abs().max()))
