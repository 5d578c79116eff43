"""Missing observations without a GPU: the masked Kronecker oracle of tests/kron_mask_oracle.py against a dense fp64
P (K (x) B) P^T and against the Hadamard oracle on the observed (point, task) pairs, mutants of the masked mix, scatter, row map and
gradient expansion that must leave the derived bound, settings.observation_nan_policy, MaskedLinearOperator's dispatch, shapes and
refusals, and the resource usage of the new kernels."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import hadamard_oracle as ho
import kmv_oracle as kmo
import kron_mask_oracle as km
import multitask_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LS, OS = 0.5, 1.3


def _case(T=3, n=40, t=4, pat="frac50", seed=0):
    x = kmo.points(n, 3, seed).double()
    B = mo.random_B(T, seed + 1).double()
    rows = km.pattern(pat, n, T, seed + 2)
    V = torch.randn(rows.numel(), t, generator=torch.Generator().manual_seed(seed + 3), dtype=torch.float64)
    return x, B, rows, V


@pytest.mark.parametrize("pat", ["one", "frac50", "point", "task", "straddle"])
def test_oracle_matches_dense_and_hadamard(pat):
    T, t = 3, 4
    x, B, rows, V = _case(T, 40, t, pat)
    dense = km.mask_matrix("rbf", x, None, LS, OS, B, rows, rows) @ V
    got = km.mask_exact("rbf", x, None, B, LS, OS, V, T, t, rows, rows)
    assert torch.allclose(got, dense, rtol=1e-6, atol=1e-6)
    xr, tr = x[rows // T], rows % T
    H = ho.hadamard_matrix("rbf", xr, xr, tr, tr, LS, OS, B, True)
    assert torch.allclose(got, H @ V, rtol=1e-6, atol=1e-6)
    # cross: observed columns of another point set
    x2 = kmo.points(30, 3, 9).double()
    cols = km.pattern(pat, 30, T, 10)
    V2 = torch.randn(cols.numel(), t, dtype=torch.float64)
    dense = km.mask_matrix("rbf", x, x2, LS, OS, B, rows, cols) @ V2
    assert torch.allclose(km.mask_exact("rbf", x, x2, B, LS, OS, V2, T, t, rows, cols), dense, rtol=1e-6, atol=1e-6)


def test_gradients_match_dense():
    T, t = 3, 2
    x, B, rows, _ = _case(T, 30, t)
    g = torch.Generator().manual_seed(5)
    L, R = torch.randn(rows.numel(), t, generator=g, dtype=torch.float64), torch.randn(rows.numel(), t, generator=g, dtype=torch.float64)
    Bv = B.clone().requires_grad_(True)
    ls = torch.tensor(LS, dtype=torch.float64, requires_grad=True)
    os_ = torch.tensor(OS, dtype=torch.float64, requires_grad=True)
    import kron_oracle as ko
    from oracle import kernels as ok
    K = ok.kernel_matrix("rbf", x, x, ls, os_, True)
    F = (L * (torch.kron(K, Bv)[rows][:, rows] @ R)).sum()
    F.backward()
    dB = km.mask_dB("rbf", x, None, LS, OS, L, R, T, t, rows, rows)
    assert torch.allclose(dB, Bv.grad, rtol=1e-6, atol=1e-6)
    gl, gs = km.mask_grad("rbf", x, None, B, LS, OS, L, R, T, t, rows, rows)
    assert torch.allclose(gl.reshape(-1), ls.grad.reshape(-1), rtol=1e-6) and abs(float(gs) - float(os_.grad)) < 1e-6 * abs(float(os_.grad))


@pytest.mark.parametrize("mutant", ["mix_neighbour", "scatter_shift", "rowmap_task"])
def test_product_mutants_leave_the_bound(mutant):
    T, t = 3, 4
    x, B, rows, V = _case(T, 300, t, "frac50", 20)
    geo = kmo.geometry(300, 300, 3, "tcgen05", 132)
    ref = km.mask_exact("matern52", x, None, B, LS, OS, V, T, t, rows, rows)
    bnd = km.mask_bound("matern52", x, None, B, LS, OS, V, T, t, rows, rows, geo)
    assert bool(((ref - km.mask_exact("matern52", x, None, B, LS, OS, V, T, t, rows, rows)).abs() <= bnd).all())
    bad = km.mask_exact("matern52", x, None, B, LS, OS, V, T, t, rows, rows, mutant=mutant)
    assert bool(((bad - ref).abs() > bnd).any()), mutant


def test_dB_drop_expand_row_leaves_the_bound():
    T, t = 3, 4
    x, B, rows, _ = _case(T, 300, t, "frac10", 30)
    g = torch.Generator().manual_seed(31)
    L, R = torch.randn(rows.numel(), t, generator=g, dtype=torch.float64), torch.randn(rows.numel(), t, generator=g, dtype=torch.float64)
    geo = kmo.geometry(300, 300, 3, "simt", 132)
    ref = km.mask_dB("rbf", x, None, LS, OS, L, R, T, t, rows, rows)
    bnd = km.mask_dB_bound("rbf", x, None, LS, OS, L, R, T, t, rows, rows, geo)
    bad = km.mask_dB("rbf", x, None, LS, OS, L, R, T, t, rows, rows, mutant="drop_expand", mutant_arg=7)
    assert bool(((bad - ref).abs() > bnd).any())


def test_nan_policy_knob():
    from gpytorch_b200 import settings

    assert settings.observation_nan_policy.value() == "ignore"
    assert settings.observation_nan_policy._fill_value == -999.0
    with pytest.raises(ValueError):
        settings.observation_nan_policy("drop")
    with settings.observation_nan_policy("mask"):
        assert settings.observation_nan_policy.value() == "mask"
        snap = settings.snapshot()
    assert settings.observation_nan_policy.value() == "ignore"
    with settings.restore(snap):
        assert settings.observation_nan_policy.value() == "mask"
    y = torch.tensor([[[1.0, float("nan")], [2.0, 3.0]], [[1.0, 2.0], [float("nan"), 3.0]]])   # batch 2, event (2, 2)
    obs = settings.observation_nan_policy._get_observed(y, torch.Size([2, 2]))
    assert torch.equal(obs, torch.tensor([[True, False], [False, True]]))
    assert torch.equal(settings.observation_nan_policy._fill_tensor(y)[0, 0], torch.tensor([1.0, -999.0]))


def test_mll_refuses_fill():
    from gpytorch_b200 import likelihoods, settings
    from gpytorch_b200.distributions import MultivariateNormal
    from gpytorch_b200.mlls import ExactMarginalLogLikelihood

    mll = ExactMarginalLogLikelihood(likelihoods.GaussianLikelihood(), None)
    with settings.observation_nan_policy("fill"), pytest.raises(ValueError, match="fill"):
        mll(MultivariateNormal(torch.zeros(3), torch.eye(3)), torch.zeros(3))


def test_masked_operator_dispatch_shapes_and_refusals():
    from gpytorch_b200 import operators as ops

    x = torch.rand(10, 2)
    ls = torch.tensor(0.5)
    mask = torch.tensor([True, False] * 5)
    plain = ops.KernelLinearOperator(x, None, "rbf", ls)
    m = ops.MaskedLinearOperator(plain, mask, mask)
    assert type(m) is ops.KernelLinearOperator and m.same and m.shape == (5, 5) and torch.equal(m.x1, x[mask])
    c = ops.MaskedLinearOperator(plain, None, mask)
    assert not c.same and c.shape == (10, 5)
    # a sum's terms share one indexed tensor: the sum stays square
    s = ops.MaskedLinearOperator(plain + ops.KernelLinearOperator(x, None, "matern52", ls), mask, mask)
    assert s.same and all(o.x1 is s.ops[0].x1 for o in s.ops)
    h = ops.HadamardKernelLinearOperator(x, None, "rbf", ls, torch.tensor(1.0), torch.arange(10) % 3, None, torch.eye(3))
    hm = ops.MaskedLinearOperator(h, mask, mask)
    assert hm.same and torch.equal(hm.t1, (torch.arange(10) % 3)[mask])
    d = ops.AddedDiagLinearOperator(plain, ops.DiagLinearOperator(torch.arange(10.0)))
    dm = ops.MaskedLinearOperator(d, mask, mask)
    assert dm.shape == (5, 5) and torch.equal(dm.diag.diag_vec, torch.arange(10.0)[mask])
    k = ops.KroneckerKernelLinearOperator(x, None, "rbf", ls, torch.tensor(1.0), torch.eye(2))
    km_ = ops.MaskedLinearOperator(k, torch.arange(20) % 3 != 0, torch.arange(20) % 3 != 0)
    assert km_.shape == (13, 13) and km_.same and torch.equal(km_.rows, (torch.arange(20) % 3 != 0).nonzero().reshape(-1))
    with pytest.raises(NotImplementedError, match="equal row and column"):
        ops.MaskedLinearOperator(k, mask.repeat(2), ~mask.repeat(2))
    with pytest.raises(NotImplementedError, match="no slices"):
        km_[0:2, 0:2]
    with pytest.raises(NotImplementedError, match="DerivKernelLinearOperator"):
        ops.MaskedLinearOperator(ops.DerivKernelLinearOperator(x, None, ls), None, torch.ones(30, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="boolean"):
        ops.MaskedLinearOperator(plain, torch.arange(10), None)


def test_new_kron_kernels_have_no_local_memory():
    """cuobjdump resource usage of the masked-Kronecker kernels and the PC_KIND_KRON_OBS pivoted Cholesky: no stack, no local memory."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
    if not os.path.exists(tool) or not os.path.exists(lib):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    want = {"kron_mix_kernelILb1E", "kron_scatter_kernelILb1E", "masked_kron_gather_kernel", "masked_kron_idx_kernel", "masked_kron_expand_kernel",
            "pc_persistent1_kernelILi72E", "pc_init_kron_obs_kernel"}
    seen = set()
    for i, line in enumerate(lines):
        for w in want:
            if re.search(r"Function \S*" + w, line):
                use = lines[i + 1]
                assert int(re.search(r"STACK:(\d+)", use).group(1)) == 0, line
                assert int(re.search(r"LOCAL:(\d+)", use).group(1)) == 0, line
                seen.add(w)
    assert seen == want, want - seen
