"""gp_bilinear_grad (the lengthscale / outputscale gradient of sum(L * (K @ R))) against the fp64 closed form of
tests/bilinear_oracle.py, within its derived worst-case fp32 bound, on the tensor-core scalar path, the SIMT scalar path and the
SIMT ARD path; refusals, determinism and non-finite inputs; and the hyper-parameter gradients of the MLL and of a
cross-covariance product through the public API against fp64 dense autograd.

API tolerances: on the Cholesky branch the engine and the fp64 reference differ by the fp32 Cholesky of K_hat, kappa(K_hat) u
with kappa <= 1 + n s / sigma^2 = 1 + 300 * 1.5 / 0.5 = 901 (Higham, Thm 10.3): 5.4e-5 of the gradient's scale, plus the
primitive (its bound, below 1e-5 of the scale here).  1e-4 of the gradient scale, the 2-norm over all raw hyper-parameters.
"""
import ctypes as C
import math
import re
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu

import bilinear_oracle as bo  # noqa: E402
from oracle import kernels as ok  # noqa: E402

GP_E_SHAPE = 1
KINDS = list(bo.KINDS)
RATIOS = {}   # (path, kind) -> largest |engine - fp64| / bound seen


def _check(tag, path, kind, engine, ref, bnd):
    (gl, go), (rl, ro), (bl, bob) = engine, ref, bnd
    errs = [abs(a - b) for a, b in zip(gl, rl.tolist())] + [abs(go - ro)]
    bounds = bl.tolist() + [bob]
    for e, b in zip(errs, bounds):
        assert math.isfinite(e) and e <= b, (tag, errs, bounds, gl, rl.tolist(), go, ro)
    key = (path, kind)
    RATIOS[key] = max([RATIOS.get(key, 0.0)] + [e / b for e, b in zip(errs, bounds) if b > 0])


def _run(dev, kind, x1, x2, ls, os_, L, R, backend, same, row_begin=0, row_count=0, n_sm=None):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if same else x2.to(dev), backend=backend, row_begin=row_begin, row_count=row_count)
    p.set_hypers(kind, ls if isinstance(ls, float) else list(ls), os_, 0.1)
    ard = not isinstance(ls, float)
    path = "tc" if (p.info()["backend"] == "tcgen05" and not ard) else "simt"
    out = p.bilinear_grad(L.float().to(dev), R.float().to(dev))
    n_sm = p.info()["n_sm"]
    args = (kind, x1.to(dev), None if same else x2.to(dev), ls, os_, L.double().to(dev), R.double().to(dev))
    ref = bo.closed_form(*args, same=same, row_begin=row_begin)
    bnd = bo.bound(*args, path, same=same, row_begin=row_begin, n_sm=n_sm)
    return p, path, out, ref, bnd


def _factors(n1, n2, s, g, positive=False):
    if positive:
        return 0.1 + torch.rand(n1, s, generator=g), 0.1 + torch.rand(n2, s, generator=g)
    return torch.randn(n1, s, generator=g), torch.randn(n2, s, generator=g)


def _ard(d):
    return [float(v) for v in torch.linspace(0.5, 1.5, d)]


# ---- paths x kinds, operand widths ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", ["tc", "simt", "ard_tc", "ard_simt"])
def test_paths_and_kinds_within_bound(cuda_dev, kind, variant):
    g = torch.Generator().manual_seed(1 + KINDS.index(kind))
    n, d, s = 257, 5, 17
    x = torch.rand(n, d, generator=g)
    L, R = _factors(n, n, s, g)
    ls = _ard(d) if variant.startswith("ard") else 0.8
    backend = "simt" if variant.endswith("simt") else "tcgen05"
    p, path, out, ref, bnd = _run(cuda_dev, kind, x, None, ls, 1.3, L, R, backend, True)
    assert path == ("tc" if variant == "tc" else "simt")
    _check(variant, path, kind, out, ref, bnd)


@pytest.mark.parametrize("d", [1, 4, 5, 8, 12, 17, 24, 32, 41, 42, 64])
@pytest.mark.parametrize("ard", [False, True])
def test_operand_widths_within_bound(cuda_dev, d, ard):
    kind = KINDS[d % 4]
    g = torch.Generator().manual_seed(100 + d)
    n1, n2, s = 129, 200, 16
    x1, x2 = torch.rand(n1, d, generator=g), torch.rand(n2, d, generator=g)
    L, R = _factors(n1, n2, s, g)
    ls = _ard(d) if ard else 0.4 * math.sqrt(d)
    p, path, out, ref, bnd = _run(cuda_dev, kind, x1, x2, ls, 0.7, L, R, "auto", False)
    assert p.info()["backend"] == ("tcgen05" if d <= 41 else "simt")
    _check(f"d={d}", path, kind, out, ref, bnd)
    if not ard and d <= 41:   # the same plan on the SIMT kernel
        p, path, out, ref, bnd = _run(cuda_dev, kind, x1, x2, ls, 0.7, L, R, "simt", False)
        _check(f"d={d} simt", path, kind, out, ref, bnd)


# ---- shapes and column counts ---------------------------------------------------------------------------------------------------
SHAPES = [(1, 1, 1), (63, 63, 15), (64, 64, 16), (65, 65, 17), (127, 127, 33), (128, 128, 1), (129, 129, 301),
          (257, 257, 15), (1000, 1000, 17), (1, 257, 16), (129, 1, 33), (63, 1000, 17), (1000, 65, 301), (128, 127, 16)]


@pytest.mark.parametrize("n1,n2,s", SHAPES)
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_shapes_within_bound(cuda_dev, n1, n2, s, backend):
    g = torch.Generator().manual_seed(n1 * 7 + n2 + s)
    same = n1 == n2
    kind = KINDS[(n1 + s) % 4]
    x1 = torch.rand(n1, 3, generator=g)
    x2 = None if same else torch.rand(n2, 3, generator=g)
    L, R = _factors(n1, n2, s, g)
    ls = 0.6 if backend == "tcgen05" or s != 17 else [0.5, 0.7, 0.9]
    p, path, out, ref, bnd = _run(cuda_dev, kind, x1, x2, ls, 1.1, L, R, backend, same)
    _check(f"{n1}x{n2} s={s}", path, kind, out, ref, bnd)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_cross_plan_of_coinciding_points_within_bound(cuda_dev, kind, backend):
    """x2 a copy of x1: a cross plan (no diagonal mask), every diagonal pair at distance 0."""
    g = torch.Generator().manual_seed(31 + KINDS.index(kind))
    x = torch.rand(300, 4, generator=g)
    L, R = _factors(300, 300, 17, g, positive=True)
    p, path, out, ref, bnd = _run(cuda_dev, kind, x, x.clone(), 0.7, 1.0, L, R, backend, False)
    _check("copy", path, kind, out, ref, bnd)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_small_square_psd_weights_within_bound(cuda_dev, kind, backend):
    """L = R > 0: every diagonal weight is positive, so an unmasked diagonal could not cancel (test_bilinear_host.py)."""
    g = torch.Generator().manual_seed(61)
    x = torch.rand(64, 4, generator=g)
    L = 0.1 + torch.rand(64, 16, generator=g)
    p, path, out, ref, bnd = _run(cuda_dev, kind, x, None, 0.6, 1.2, L, L, backend, True)
    _check("psd", path, kind, out, ref, bnd)


@pytest.mark.parametrize("points", ["repeat4", "grid", "near"])
@pytest.mark.parametrize("kind", KINDS)
def test_duplicate_and_grid_points_within_bound(cuda_dev, points, kind):
    g = torch.Generator().manual_seed(41 + KINDS.index(kind))
    l = 0.5
    if points == "repeat4":
        x = torch.rand(100, 3, generator=g).repeat(4, 1)
    elif points == "grid":
        x = (torch.rand(400, 3, generator=g) * 8).round() / 8
    else:
        x = torch.rand(400, 3, generator=g)
        x[1] = x[0] + torch.tensor([1e-4 * l, 0.0, 0.0])
    L, R = _factors(400, 400, 17, g)
    for backend, ls in (("tcgen05", l), ("simt", l), ("simt", [l, 0.8 * l, 1.2 * l])):
        p, path, out, ref, bnd = _run(cuda_dev, kind, x, None, ls, 1.2, L, R, backend, True)
        _check(points, path, kind, out, ref, bnd)


# ---- row shards -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend,ard", [("tcgen05", False), ("simt", False), ("simt", True)])
def test_row_shards_within_bound_and_sum_to_the_full_gradient(cuda_dev, backend, ard):
    g = torch.Generator().manual_seed(5)
    n, d, s = 1000, 4, 17
    x = torch.rand(n, d, generator=g)
    L, R = _factors(n, n, s, g, positive=True)
    ls = _ard(d) if ard else 0.6
    full = bo.closed_form("matern12", x.to(cuda_dev), None, ls, 1.4, L.double().to(cuda_dev), R.double().to(cuda_dev), same=True)
    tot_l, tot_o, bsum_l, bsum_o = 0.0, 0.0, 0.0, 0.0
    for b, c in [(0, 129), (129, 200), (329, 371), (700, 300)]:
        p, path, out, ref, bnd = _run(cuda_dev, "matern12", x, None, ls, 1.4, L[b:b + c], R, backend, True, b, c)
        _check(f"shard {b}+{c}", path, "matern12", out, ref, bnd)
        tot_l, tot_o = tot_l + torch.tensor(out[0], dtype=torch.float64), tot_o + out[1]
        bsum_l, bsum_o = bsum_l + bnd[0], bsum_o + bnd[1]
    assert ((tot_l - full[0]).abs() <= bsum_l).all() and abs(tot_o - full[1]) <= bsum_o


# ---- C ABI: strides, refusals ---------------------------------------------------------------------------------------------------
def test_strided_factors_one_row_and_refusals(cuda_dev):
    from gpytorch_b200 import _lib
    from gpytorch_b200.engine import Plan, _ptr

    g = torch.Generator().manual_seed(9)
    n, s = 200, 17
    x = torch.rand(n, 3, generator=g)
    L, R = _factors(n, n, s, g)
    p = Plan(x.to(cuda_dev), backend="tcgen05").set_hypers("matern32", 0.6, 1.2, 0.1)
    base = p.bilinear_grad(L.to(cuda_dev), R.to(cuda_dev))
    Lp = torch.zeros(n, s + 5, device=cuda_dev); Lp[:, :s] = L.to(cuda_dev)
    Rp = torch.zeros(n, s + 11, device=cuda_dev); Rp[:, :s] = R.to(cuda_dev)
    gl, go = (C.c_double * 1)(), C.c_double()
    assert p.lib.gp_bilinear_grad(p._h, _ptr(Lp), s + 5, _ptr(Rp), s + 11, s, gl, C.byref(go)) == 0
    assert (gl[0], go.value) == (base[0][0], base[1])   # ldl, ldr > s: the same columns, bit for bit
    # ldl < s is refused before any launch
    l0 = p.launches()
    assert p.lib.gp_bilinear_grad(p._h, _ptr(Lp), s - 1, _ptr(Rp), s + 11, s, gl, C.byref(go)) == GP_E_SHAPE
    assert p.lib.gp_bilinear_grad(p._h, _ptr(Lp), s + 5, _ptr(Rp), 3, s, gl, C.byref(go)) == GP_E_SHAPE
    assert p.launches() == l0
    # one test point: a one-row L with row stride 0 (an expanded row), against a contiguous copy and the bound
    xs = torch.rand(1, 3, generator=g)
    pc = Plan(xs.to(cuda_dev), x.to(cuda_dev), backend="tcgen05").set_hypers("rbf", 0.6, 1.2, 0.1)
    row = torch.randn(1, s, generator=g).to(cuda_dev)
    assert pc.lib.gp_bilinear_grad(pc._h, _ptr(row), 0, _ptr(R.to(cuda_dev)), s, s, gl, C.byref(go)) == 0
    assert (gl[0], go.value) == tuple(v[0] if isinstance(v, list) else v for v in pc.bilinear_grad(row, R.to(cuda_dev)))
    assert pc.bilinear_grad(row.as_strided((1, s), (0, 1)), R.to(cuda_dev)) == pc.bilinear_grad(row, R.to(cuda_dev))
    # d = 65: refused with its message before the two to_v16 launches
    wide = Plan(torch.rand(50, 65, device=cuda_dev)).set_hypers("rbf", 3.0, 1.0, 0.0)
    Lw = torch.randn(50, 2, device=cuda_dev)
    l0 = wide.launches()
    assert wide.lib.gp_bilinear_grad(wide._h, _ptr(Lw), 2, _ptr(Lw), 2, 2, gl, C.byref(go)) == GP_E_SHAPE
    assert "d <= 64" in _lib.last_error() and wide.launches() == l0
    # the Python seam checks shapes, dtype and device
    for bad in (L.to(cuda_dev)[:, :3], L.to(cuda_dev)[:-1], L.double().to(cuda_dev), L):
        with pytest.raises(RuntimeError):
            p.bilinear_grad(bad, R.to(cuda_dev))


def test_api_model_with_d_over_64_raises_from_backward(cuda_dev):
    import gpytorch_b200 as gp
    x = torch.rand(1000, 100, device=cuda_dev)
    y = torch.randn(1000, device=cuda_dev)
    lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(cuda_dev)
    model.train(); lik.train()
    loss = -gp.ExactMarginalLogLikelihood(lik, model)(model(x), y)
    with pytest.raises(RuntimeError, match="d <= 64"):
        loss.backward()


# ---- the reference's own numbers, determinism, non-finite inputs ----------------------------------------------------------------
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_reference_goldens_through_the_engine(cuda_dev, golden, backend):
    names = {"rbf": "rbf", "matern12": "mat12", "matern32": "mat32", "matern52": "mat52"}
    for tag in "abcd":
        x1 = torch.from_numpy(golden[f"{tag}_f32_x1"]); x2 = torch.from_numpy(golden[f"{tag}_f32_x2"])
        same = bool(golden[f"{tag}_f32_same"])
        ls = float(golden[f"{tag}_f32_ls"])
        W = torch.from_numpy(golden[f"{tag}_f32_rbf_W"])
        I = torch.eye(x2.size(0))
        for kind, nk in names.items():
            p, path, out, ref, bnd = _run(cuda_dev, kind, x1, x2, ls, 1.0, W, I, backend, same)
            gold = float(golden[f"{tag}_f32_{nk}_dls"].reshape(-1)[0])
            # the golden is the reference's own fp32 backward: allow its rounding (n1 n2 u of the magnitudes) on top
            tol = bnd[0][0].item() + 2e-5 * abs(ref[0][0].item()) + 1e-6
            assert abs(out[0][0] - gold) <= tol, (tag, kind, out[0][0], gold, ref[0][0].item())
            _check(f"golden {tag}", path, kind, out, ref, bnd)


@pytest.mark.parametrize("backend,ls", [("tcgen05", 0.7), ("simt", 0.7), ("simt", [0.6, 0.9, 1.1])])
def test_repeated_calls_are_bit_identical(cuda_dev, backend, ls):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(3)
    x = torch.rand(700, 3, generator=g).to(cuda_dev)
    L, R = (t.to(cuda_dev) for t in _factors(700, 700, 33, g))
    p = Plan(x, backend=backend).set_hypers("matern52", ls, 1.0, 0.1)
    first = p.bilinear_grad(L, R)
    for _ in range(3):
        assert p.bilinear_grad(L, R) == first


@pytest.mark.parametrize("where", ["x1", "x2"])
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
@pytest.mark.parametrize("backend,ls", [("tcgen05", 0.7), ("simt", 0.7), ("simt", [0.6, 0.9, 1.1])])
@pytest.mark.parametrize("kind", ["rbf", "matern12"])
def test_non_finite_inputs_give_nan_gradients_and_rows(cuda_dev, where, bad, backend, ls, kind):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(4)
    x1, x2 = torch.rand(150, 3, generator=g), torch.rand(90, 3, generator=g)
    (x1 if where == "x1" else x2)[17, 1] = bad
    p = Plan(x1.to(cuda_dev), x2.to(cuda_dev), backend=backend).set_hypers(kind, ls, 1.0, 0.1)
    gl, go = p.bilinear_grad(torch.randn(150, 5, device=cuda_dev), torch.randn(90, 5, device=cuda_dev))
    assert all(math.isnan(v) for v in gl) and math.isnan(go), (gl, go)
    assert torch.isnan(p.rows(torch.arange(150, device=cuda_dev))).all()
    sq = Plan(x1.to(cuda_dev), backend=backend).set_hypers(kind, ls, 1.0, 0.1)
    if where == "x1":
        gl, go = sq.bilinear_grad(torch.randn(150, 17, device=cuda_dev), torch.randn(150, 17, device=cuda_dev))
        assert all(math.isnan(v) for v in gl) and math.isnan(go), (gl, go)
        assert torch.isnan(sq.rows(torch.tensor([0, 17, 149], device=cuda_dev))).all()


# ---- long accumulation: C2 size -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend,ls,kind", [("tcgen05", 1.0, "rbf"), ("simt", [float(v) for v in torch.linspace(0.7, 1.6, 10)], "matern32")])
def test_long_accumulation_at_n_50000(cuda_dev, backend, ls, kind):
    from oracle import mll as om

    n = 50000
    x, _ = om.synthetic_problem(n, 10, 0, torch.float32)
    g = torch.Generator().manual_seed(8)
    L, R = _factors(n, n, 2, g)
    p, path, out, ref, bnd = _run(cuda_dev, kind, x, None, ls, 1.0, L, R, backend, True)
    _check("n=50000", path, kind, out, ref, bnd)


# ---- SKI: its own 16-column chunk loop ------------------------------------------------------------------------------------------
def test_ski_strided_33_columns_match_unstrided_chunks(cuda_dev):
    from gpytorch_b200.engine import Plan

    g = torch.Generator().manual_seed(21)
    n, s = 500, 33
    x = (torch.rand(n, 2, generator=g) * 0.8 + 0.1).to(cuda_dev)
    L, R = (t.to(cuda_dev) for t in _factors(n, n, s, g))
    p = Plan(x).set_ski([30, 30], [0.0, 0.0], [1.0 / 29, 1.0 / 29]).set_hypers("rbf", 0.3, 1.2, 0.1)
    Lp = torch.zeros(n, s + 7, device=cuda_dev); Lp[:, :s] = L
    Rp = torch.zeros(n, s + 3, device=cuda_dev); Rp[:, :s] = R
    full = p.bilinear_grad(Lp[:, :s], Rp[:, :s])
    parts = [p.bilinear_grad(L[:, c:c + 16].contiguous(), R[:, c:c + 16].contiguous()) for c in (0, 16, 32)]
    tl, to = sum(q[0][0] for q in parts), sum(q[1] for q in parts)
    # the chunk sums of one call are the per-chunk calls added in double; the scatter's atomics reorder fp32 adds
    assert full[0][0] == pytest.approx(tl, rel=1e-5, abs=1e-5) and full[1] == pytest.approx(to, rel=1e-5, abs=1e-5)


# ---- through the API ------------------------------------------------------------------------------------------------------------
def _softplus(raw, lb=0.0):
    return torch.nn.functional.softplus(raw) + lb


def _api_case(gp, case, x, y, dev):
    n = x.size(0)
    fixed = None
    if case == "fixed":
        fixed = (0.4 + 0.2 * torch.rand(n, generator=torch.Generator().manual_seed(1))).to(dev)
        lik = gp.likelihoods.FixedNoiseGaussianLikelihood(noise=fixed)
    else:
        lik = gp.likelihoods.GaussianLikelihood()

    class M(gp.models.ExactGP):
        def __init__(self):
            super().__init__(x, y, lik)
            self.mean_module = gp.means.ConstantMean()
            if case == "sum":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel()) + gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=0.5))
            elif case == "ard":
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu=1.5, ard_num_dims=2, active_dims=[0, 2]))
            elif case in ("rbf", "fixed"):
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.RBFKernel())
            else:
                self.covar_module = gp.kernels.ScaleKernel(gp.kernels.MaternKernel(nu={"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}[case]))

        def forward(self, xx):
            return gp.distributions.MultivariateNormal(self.mean_module(xx), self.covar_module(xx))

    model = M().to(dev)
    lik = lik.to(dev)
    scales = model.covar_module.kernels if case == "sum" else [model.covar_module]
    for i, sk in enumerate(scales):
        sk.base_kernel.lengthscale = torch.tensor([[0.6, 0.9]]) if case == "ard" else 0.5 + 0.3 * i
        sk.outputscale = 1.5 - 0.5 * i
    if case != "fixed":
        lik.noise = 0.5
    model.mean_module.constant = 0.2
    return model, lik, scales, fixed


def _api_k64(case, x, scales, lik, fixed):
    """K_hat in fp64 from fp64 copies of the raw parameters, through the same softplus transforms: (K_hat, [(param, raw64)])."""
    kinds = {"sum": ["rbf", "matern12"], "ard": ["matern32"], "fixed": ["rbf"], "rbf": ["rbf"]}.get(case, [case])
    raws, K = [], 0.0
    x64 = x.double().cpu()
    for kind, sk in zip(kinds, scales):
        rl = sk.base_kernel.raw_lengthscale.detach().double().cpu().requires_grad_()
        ro = sk.raw_outputscale.detach().double().cpu().requires_grad_()
        raws += [(sk.base_kernel.raw_lengthscale, rl), (sk.raw_outputscale, ro)]
        ls = _softplus(rl).reshape(-1)
        xs = x64[:, [0, 2]] if case == "ard" else x64
        K = K + ok.kernel_matrix(kind, xs, xs, ls if ls.numel() > 1 else ls[0], _softplus(ro), True)
    n = x64.size(0)
    if fixed is not None:
        noise = fixed.double().cpu()
    else:
        rn = lik.noise_covar.raw_noise.detach().double().cpu().requires_grad_()
        raws.append((lik.noise_covar.raw_noise, rn))
        noise = (_softplus(rn, 1e-4)).expand(n)
    return K + torch.diag(noise), raws


def _compare_hyper_grads(tag, raws, rel):
    """Every raw hyper-parameter gradient within rel of the model's gradient scale (the 2-norm over all of them)."""
    got = torch.cat([p.grad.double().cpu().reshape(-1) for p, _ in raws])
    want = torch.cat([r.grad.reshape(-1) for _, r in raws])
    scale = want.norm().item()
    err = (got - want).abs().max().item()
    print(f"{tag}: max |engine - fp64| = {err:.3e} = {err / scale:.3e} of the gradient scale {scale:.3e}")
    assert err <= rel * scale, (tag, got, want)


@pytest.mark.parametrize("case", ["rbf", "matern12", "matern32", "matern52", "ard", "sum", "fixed"])
def test_api_cholesky_branch_hyper_gradients_match_fp64(cuda_dev, case):
    import gpytorch_b200 as gp

    n = 300
    g = torch.Generator().manual_seed(13)
    x = torch.rand(n, 3, generator=g)
    y = torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(n, generator=g)
    model, lik, scales, fixed = _api_case(gp, case, x.to(cuda_dev), y.to(cuda_dev), cuda_dev)
    model.train(); lik.train()
    loss = -gp.ExactMarginalLogLikelihood(lik, model)(model(x.to(cuda_dev)), y.to(cuda_dev))
    loss.backward()
    Kh, raws = _api_k64(case, x, scales, lik, fixed)
    Lc = torch.linalg.cholesky(Kh)
    r = (y.double() - 0.2).unsqueeze(-1)
    iq = (r * torch.cholesky_solve(r, Lc)).sum()
    (0.5 * (iq + 2 * Lc.diagonal().log().sum() + n * math.log(2 * math.pi)) / n).backward()
    _compare_hyper_grads(f"cholesky {case}", raws, 1e-4)


@pytest.mark.parametrize("case", ["rbf", "matern12", "ard"])
def test_api_cg_branch_hyper_gradients_match_the_fp64_estimator(cuda_dev, case):
    """With fixed probes z the engine's gradient estimates d(-MLL) = (1/2n) [-alpha^T dK_hat alpha + (1/t) sum_i u_i^T dK_hat z_i]
    with alpha = K_hat^-1 r and u_i = K_hat^-1 z_i from CG: the fp64 gradient of that surrogate with the solves held fixed.  CG
    stops at a relative residual of 1e-6, so the solves agree to kappa 1e-6 <= 901e-6 of their scale: 2e-3 of the gradient scale."""
    import gpytorch_b200 as gp
    from gpytorch_b200 import settings

    n, tp, seed = 300, 8, 1234
    g = torch.Generator().manual_seed(14)
    x = torch.rand(n, 3, generator=g)
    y = torch.sin(3 * x[:, 0]) + 0.1 * torch.randn(n, generator=g)
    model, lik, scales, fixed = _api_case(gp, case, x.to(cuda_dev), y.to(cuda_dev), cuda_dev)
    model.train(); lik.train()
    with settings.max_cholesky_size(0), settings.cg_tolerance(1e-6), settings.num_trace_samples(tp), settings.probe_seed(seed), \
            settings.max_lanczos_quadrature_iterations(50):
        loss = -gp.ExactMarginalLogLikelihood(lik, model)(model(x.to(cuda_dev)), y.to(cuda_dev))
        loss.backward()
        # the probes the engine drew: Rademacher columns (no preconditioner below min_preconditioning_size)
        gen = torch.Generator(device=cuda_dev).manual_seed(seed)
        z = (torch.randint(0, 2, (n, tp), device=cuda_dev, generator=gen).to(torch.float32) * 2 - 1).double().cpu()
    Kh, raws = _api_k64(case, x, scales, lik, fixed)
    r = (y.double() - 0.2).unsqueeze(-1)
    alpha = torch.linalg.solve(Kh.detach(), r)
    u = torch.linalg.solve(Kh.detach(), z)
    (0.5 / n * (-(alpha * (Kh @ alpha)).sum() + (u * (Kh @ z)).sum() / tp)).backward()
    _compare_hyper_grads(f"cg {case}", raws, 2e-3)


def test_api_expanded_rhs_hyper_gradients(cuda_dev):
    """A right-hand side with row stride 0 (expand) reaches gp_bilinear_grad as a copy: the gradients match fp64 autograd."""
    from gpytorch_b200.operators import KernelLinearOperator

    g = torch.Generator().manual_seed(15)
    n, t = 400, 3
    X = torch.rand(n, 4, generator=g)
    w = torch.randn(n, t, generator=g)
    row = torch.randn(1, t, generator=g)
    for rhs, wt in ((row.to(cuda_dev).expand(n, t), w), (torch.tensor(0.7, device=cuda_dev).expand(n), w[:, 0])):
        assert rhs.stride(0) == 0
        ls = torch.tensor(0.6, device=cuda_dev, requires_grad=True)
        os_ = torch.tensor(1.3, device=cuda_dev, requires_grad=True)
        op = KernelLinearOperator(X.to(cuda_dev), None, "matern32", ls, os_)
        (wt.to(cuda_dev) * (op @ rhs)).sum().backward()
        assert op.plan().info()["backend"] == "tcgen05"
        ls64 = torch.tensor(0.6, dtype=torch.float32).double().requires_grad_()
        os64 = torch.tensor(1.3, dtype=torch.float32).double().requires_grad_()
        K = ok.kernel_matrix("matern32", X.double(), X.double(), ls64, os64, True)
        (wt.double() * (K @ rhs.double().cpu())).sum().backward()
        L2 = wt.double().reshape(n, -1).to(cuda_dev)
        R2 = rhs.double().reshape(n, -1).contiguous().to(cuda_dev)
        bl, bs = bo.bound("matern32", X.to(cuda_dev), None, 0.6, 1.3, L2, R2, "tc", same=True)
        assert abs(ls.grad.item() - ls64.grad.item()) <= bl.item() and abs(os_.grad.item() - os64.grad.item()) <= bs


@pytest.mark.parametrize("m", [1, 7, 300])
@pytest.mark.parametrize("kind", ["rbf", "matern12"])
def test_api_cross_covariance_product_hyper_gradients(cuda_dev, m, kind):
    from gpytorch_b200.operators import KernelLinearOperator

    g = torch.Generator().manual_seed(m)
    n, t = 500, 3
    X, xs = torch.rand(n, 4, generator=g), torch.rand(m, 4, generator=g)
    v, w = torch.randn(n, t, generator=g), torch.randn(m, t, generator=g)
    ls = torch.tensor(0.6, device=cuda_dev, requires_grad=True)
    os_ = torch.tensor(1.3, device=cuda_dev, requires_grad=True)
    op = KernelLinearOperator(xs.to(cuda_dev), X.to(cuda_dev), kind, ls, os_)
    (w.to(cuda_dev) * (op @ v.to(cuda_dev))).sum().backward()
    assert op.plan().info()["backend"] == "tcgen05"   # the bound below is the tensor-core path's
    ls64 = torch.tensor(0.6, dtype=torch.float32).double().requires_grad_()
    os64 = torch.tensor(1.3, dtype=torch.float32).double().requires_grad_()
    (w.double() * (ok.kernel_matrix(kind, xs.double(), X.double(), ls64, os64, False) @ v.double())).sum().backward()
    bl, bs = bo.bound(kind, xs.to(cuda_dev), X.to(cuda_dev), 0.6, 1.3, w.double().to(cuda_dev), v.double().to(cuda_dev), "tc")
    assert abs(ls.grad.item() - ls64.grad.item()) <= bl.item() and abs(os_.grad.item() - os64.grad.item()) <= bs


def test_api_nan_training_input_never_gives_a_finite_loss(cuda_dev):
    import gpytorch_b200 as gp

    n = 200
    x = torch.rand(n, 3, device=cuda_dev)
    x[5, 0] = float("nan")
    y = torch.randn(n, device=cuda_dev)
    model, lik, _, _ = _api_case(gp, "rbf", x, y, cuda_dev)
    model.train(); lik.train()
    try:
        loss = -gp.ExactMarginalLogLikelihood(lik, model)(model(x), y)
    except RuntimeError as e:   # the dense branch's Cholesky of a NaN matrix (torch's LinAlgError, NotPSDError) or NanError
        assert re.search(r"positive.definite|nan", str(e), re.IGNORECASE), e
        return
    assert not math.isfinite(loss.item())


def test_zz_report_error_fraction_of_bound(cuda_dev):
    """Largest observed |engine - fp64| / bound per path and kind over this module's cases (printed with -s)."""
    name = torch.cuda.get_device_name(0)
    smi = shutil.which("nvidia-smi")
    q = subprocess.run([smi, "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True) if smi else None
    name += f", power limit {(q.stdout.strip() if q else '') or 'unknown'}"
    for (path, kind), r in sorted(RATIOS.items()):
        print(f"[{name}] bilinear {path:4s} {kind:9s} max err / bound = {r:.3e}")
    assert all(r <= 1.0 for r in RATIOS.values())
