"""CPU checks of the piecewise polynomial kernel: the reference's golden covariances and gradients against the fp64 oracle, the
module's q = 2 coefficient against R&W's, the host restatement of the compact-support schedule (every pair with r < 1 lies in a
listed tile pair) on random, clustered, collinear and duplicate points and on a dense schedule, mutants that fall outside the K.V
bound, the class surface and its refusals, and the compiled kernels (no local memory, no shared fp32 atomics)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import ppoly_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
GOLD = os.path.join(ROOT, "tests", "golden", "ppoly_golden.npz")


def test_golden_against_the_oracle():
    g = np.load(GOLD)
    assert int(g["ncases"]) == 32
    seen = set()
    zeros = inside = 0
    for ci in range(int(g["ncases"])):
        q, D, ard, n1, n2 = (int(v) for v in g[f"c{ci}_meta"])
        seen.add((q, D, ard))
        x1, x2, W = (torch.from_numpy(g[f"c{ci}_{k}"]) for k in ("x1", "x2", "W"))
        ls = g[f"c{ci}_ls"].reshape(-1)
        K = po.kernel(x1, x2, ls, q)
        assert torch.allclose(K, torch.from_numpy(g[f"c{ci}_K"]), rtol=1e-12, atol=1e-12)
        Kxx = po.kernel(x1, x1, ls, q)
        assert torch.allclose(Kxx, torch.from_numpy(g[f"c{ci}_Kxx"]), rtol=1e-12, atol=1e-12)
        assert torch.allclose(torch.diagonal(Kxx), torch.from_numpy(g[f"c{ci}_diag"]), rtol=1e-12, atol=1e-12)
        # sum(W * K) = sum(L * (K R)) with L = W, R = I
        gl, _ = po.grads(x1, x2, ls, q, 1.0, W, torch.eye(n2, dtype=torch.float64))
        ref = g[f"c{ci}_gls"].reshape(-1)
        assert np.allclose(gl, ref, rtol=1e-10, atol=1e-12), (ci, gl, ref)
        zeros += int((K == 0).sum())
        inside += int((K > 0).sum())
    assert zeros > 100 and inside > 100   # the cases cross the support boundary
    assert seen == {(q, D, a) for q in range(4) for D in (1, 2, 3, 5) for a in (0, 1)}


def test_q2_coefficient_is_the_modules_not_the_textbooks():
    """The reference module writes (j + 4*j + 3) / 3 where R&W eq. 4.21 (and the reference's own test) has (j^2 + 4 j + 3) / 3.
    The engine follows the module, which the golden pins; a fix in the reference would show up as a golden regeneration."""
    for D in (1, 2, 3, 5, 16):
        _, mod = po.coeffs(2, D)
        _, rw = po.coeffs(2, D, textbook=True)
        j = D // 2 + 3
        assert mod[1] == (5 * j + 3) / 3.0 and rw[1] == (j * j + 4 * j + 3) / 3.0 and mod[1] != rw[1]
    src = open(os.path.join(ROOT, "gpytorch_b200", "csrc", "compact.cu")).read()
    assert "(J + 4.0 * J + 3.0) / 3.0" in src


def _clustered(gen, n, d):
    c = torch.rand(8, d, generator=gen, dtype=torch.float64)
    return (c[torch.randint(0, 8, (n,), generator=gen)] + 0.01 * torch.randn(n, d, generator=gen, dtype=torch.float64)).float()


@pytest.mark.parametrize("layout", ["random", "clustered", "collinear", "duplicates", "dense"])
@pytest.mark.parametrize("d", [1, 2, 3, 5])
def test_schedule_covers_every_pair_within_reach(layout, d):
    gen = torch.Generator().manual_seed(11 + d)
    n1, n2 = 700, 450
    x = torch.rand(n1, d, generator=gen)
    y = torch.rand(n2, d, generator=gen)
    ls = [0.05 * (1 + c) for c in range(d)]
    if layout == "clustered":
        x, y = _clustered(gen, n1, d), _clustered(gen, n2, d)
    elif layout == "collinear":
        t = torch.rand(n1, 1, generator=gen)
        x = t * torch.linspace(1.0, 2.0, d)[None, :]
        y = x[:n2] + 1e-3
    elif layout == "duplicates":
        x = x[torch.randint(0, 60, (n1,), generator=gen)]
        y = x[:n2]
    elif layout == "dense":
        ls = [10.0] * d
    X1, X2 = x.numpy(), y.numpy()
    for other in (None, X2):
        assert po.uncovered_pairs(X1, other, ls) == 0
    _, _, R = po.schedule(X1, None, ls)
    if layout == "dense":
        assert R.all()


def test_schedule_is_lengthscale_free_in_its_order_and_stable_on_ties():
    gen = torch.Generator().manual_seed(5)
    x = torch.rand(300, 2, generator=gen).numpy()
    x[100:150] = x[100]   # ties keep their input order
    p = po.morton_perm(x)
    tied = p[np.isin(p, np.arange(100, 150))]
    assert (np.diff(tied) > 0).all()
    x[7, 0] = np.nan   # a NaN key sorts as cell 0 and does not disturb the rest
    q = po.morton_perm(x)
    assert sorted(q.tolist()) == list(range(300))


def test_mutants_fall_outside_the_bound():
    gen = torch.Generator().manual_seed(3)
    n, d, q = 400, 2, 2
    x = torch.rand(n, d, generator=gen)
    ls = [0.15, 0.2]
    V = torch.randn(n, 4, generator=gen)
    K = po.kernel(x, x, ls, q)
    ref = K @ V.double()
    bnd = po.kmv_bound(x, x, ls, q, 1.0, V)
    assert bool(((K @ V.double() - ref).abs() <= bnd).all())
    e, c = po.coeffs(q, d)
    dd = (x[:, None, :].double() - x[None, :, :].double()) / torch.tensor(ls, dtype=torch.float64)
    r = torch.sqrt((dd * dd).sum(-1))
    m = torch.clamp(1 - r, min=0)
    rw = m ** e * (1 + c[0] * r + po.coeffs(q, d, textbook=True)[1][1] * r * r)
    # a tile pair dropped: the columns of one 64-column tile zeroed for the rows of one 128-row tile
    perm = po.morton_perm(x.numpy())
    drop = K.clone()
    rows, cols = perm[:128], perm[64:128]
    drop[np.ix_(rows, cols)] = 0.0
    mutants = {"R&W coefficient": rw, "exponent j": m ** (e - q) * (1 + c[0] * r + c[1] * r * r), "l not applied": po.kernel(x, x, 1.0, q),
               "dropped tile pair": drop}
    for name, Km in mutants.items():
        assert bool(((Km @ V.double() - ref).abs() > bnd).any()), name


def test_class_surface_and_refusals():
    import gpytorch_b200 as gp
    from gpytorch_b200.operators import PiecewisePolynomialKernelLinearOperator

    k = gp.kernels.PiecewisePolynomialKernel()
    assert k.q == 2 and tuple(k.raw_lengthscale.shape) == (1, 1) and type(k.raw_lengthscale_constraint).__name__ == "Positive"
    assert sorted(k.state_dict().keys()) == ["raw_lengthscale", "raw_lengthscale_constraint.lower_bound",
                                             "raw_lengthscale_constraint.upper_bound"]
    ka = gp.kernels.PiecewisePolynomialKernel(q=0, ard_num_dims=3)
    assert tuple(ka.raw_lengthscale.shape) == (1, 3)
    sk = gp.kernels.ScaleKernel(gp.kernels.PiecewisePolynomialKernel(q=1, ard_num_dims=2))
    assert {"base_kernel.raw_lengthscale", "raw_outputscale"} <= set(sk.state_dict().keys())
    for bad in (4, -1, 1.5, None):
        with pytest.raises(ValueError, match="q expected to be 0, 1, 2 or 3"):
            gp.kernels.PiecewisePolynomialKernel(q=bad)
    with pytest.raises(NotImplementedError):
        gp.kernels.PiecewisePolynomialKernel(lengthscale_prior=object())
    with pytest.raises(NotImplementedError):
        gp.kernels.PiecewisePolynomialKernel(batch_shape=torch.Size([2, 2]))
    assert tuple(gp.kernels.PiecewisePolynomialKernel(batch_shape=torch.Size([2])).raw_lengthscale.shape) == (2, 1, 1)
    x = torch.randn(6, 3)
    k.lengthscale = 0.7
    op = gp.kernels.ScaleKernel(gp.kernels.ScaleKernel(k))(x)
    assert isinstance(op, PiecewisePolynomialKernelLinearOperator) and op.q == 2 and abs(float(op.lengthscale) - 0.7) < 1e-6
    for o in (op.detach(), op._transpose_nonbatch(), op[1:4, :], gp.operators.with_outputscale(op, torch.tensor(2.0))):
        assert isinstance(o, PiecewisePolynomialKernelLinearOperator) and o.q == 2
    assert gp.kernels.PiecewisePolynomialKernel(active_dims=[0, 2])(x).x1.shape[1] == 2
    assert gp.operators.LowRankUpdatedKernelLinearOperator.supports(op)
    rbf = gp.operators.KernelLinearOperator(x, None, "rbf", torch.tensor(1.0))
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        k.forward(x, x, last_dim_is_batch=True)
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        op.mul(rbf)
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        rbf.mul(op)
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        rbf + op
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        op + rbf
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        gp.kernels.PiecewisePolynomialKernel() + gp.kernels.RBFKernel()
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        gp.kernels.ProductKernel(gp.kernels.PiecewisePolynomialKernel(), gp.kernels.RBFKernel())
    with pytest.raises(NotImplementedError, match="PiecewisePolynomialKernel"):
        gp.kernels.GridInterpolationKernel(gp.kernels.PiecewisePolynomialKernel(), grid_size=16, num_dims=1)
    with pytest.raises(NotImplementedError):
        gp.kernels.MultitaskKernel(gp.kernels.PiecewisePolynomialKernel(), num_tasks=2)(x)
    with pytest.raises(NotImplementedError, match="row-sharded"):
        PiecewisePolynomialKernelLinearOperator(x, None, 2, torch.tensor(1.0), comm=object())
    with pytest.raises(NotImplementedError, match="inputs"):
        k(x.clone().requires_grad_(True))
    with pytest.raises(NotImplementedError, match="inputs"):
        op._input_grad_list(None, None, [True])
    assert op._dense_input_grad_list(None, [False]) == [None]


def test_header_and_bindings_document_the_calls():
    h = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert "GP_PPOLY = 6" in h and "GP_BACKEND_COMPACT = 8" in h
    assert re.search(r"int gp_plan_set_hypers_pp\(gp_plan\* plan, int q, const float\* lengthscale, int n_ls, float outputscale, "
                     r"float noise\);", h)
    assert "int gp_plan_tile_pairs(gp_plan* plan, int64_t* evaluated, int64_t* total);" in h
    from gpytorch_b200 import _lib
    assert _lib.GP_PPOLY == 6 and _lib.GP_BACKEND_COMPACT == 8
    assert "gp_plan_set_hypers_pp" in _lib.PROTOTYPES and "gp_plan_tile_pairs" in _lib.PROTOTYPES
    api = open(os.path.join(ROOT, "gpytorch_b200", "csrc", "api.cu")).read()
    assert "call gp_plan_set_hypers_pp" in api
    assert "compact.cu" in open(os.path.join(ROOT, "gpytorch_b200", "build.py")).read()


def _tool(name):
    t = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return t if os.path.exists(t) else None


def test_new_kernels_have_no_local_memory_and_no_shared_float_atomics():
    tool = _tool("cuobjdump")
    if not tool or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function" in line and re.search(r"_ZN2gp\d+pp_\w+kernel", line):
            seen += 1
            assert int(re.search(r"LOCAL:(\d+)", lines[i + 1]).group(1)) == 0, line
            assert int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1)) == 0, line
    assert seen == 4 + 8 + 6, seen   # K.V (4 widths), gradient (4 widths x ARD), and the six schedule kernels
    obj = os.path.join(ROOT, "gpytorch_b200", "build", "compact.o")   # the object build() links: a much smaller dump than the library
    sass = subprocess.run([tool, "-sass", obj if os.path.exists(obj) else LIB], capture_output=True, text=True, timeout=900).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    pp = [f for f in funcs if re.match(r"_ZN2gp\d+pp_", f)]
    assert len(pp) == seen
    for f in pp:
        assert not re.search(r"\b(ATOMS|ATOM|RED)\.[A-Z.]*F32", f), f.splitlines()[0]
        assert not re.search(r"\b(LDL|STL)\b", f), f.splitlines()[0]
