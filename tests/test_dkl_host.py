"""Host checks of deep kernel learning: the SKI weight derivatives of the fp64 oracle against the reference's own autograd
(tests/golden/dkl_golden.npz, generator tests/golden/make_golden_dkl.py); the fp64 closed form of the SKI input gradient
(tests/dkl_oracle.py) against autograd through a dense W K_uu W^T; the solve-side autograd plumbing of operators.py on fake
plans; the new kernel's local memory; ScaleToBounds against the reference module."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from dkl_oracle import dense_ski, interp_with_derivatives, ski_input_grad
from oracle import ski

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "dkl_golden.npz"))


@pytest.mark.parametrize("tag,d", [("d1", 1), ("d2", 2), ("d3", 3)])
def test_weight_derivatives_match_reference_autograd(tag, d):
    x = torch.from_numpy(GOLD[f"{tag}_x"])
    axes = [torch.from_numpy(GOLD[f"{tag}_grid{i}"]) for i in range(d)]
    ref_idx, ref_dval = torch.from_numpy(GOLD[f"{tag}_idx"]), torch.from_numpy(GOLD[f"{tag}_dval"])
    # the oracle through autograd: row i of W depends on x_i only, so d(sum_i val[i, q]) / dx = d val[:, q] / dx row by row
    xr = x.clone().requires_grad_(True)
    idx, val = ski.interpolate(axes, xr)
    assert torch.equal(idx, ref_idx)
    auto = torch.zeros_like(ref_dval)
    for q in range(val.size(1)):
        (gq,) = torch.autograd.grad(val[:, q].sum(), xr, retain_graph=True)
        auto[:, :, q] = gq.t()
    torch.testing.assert_close(auto, ref_dval, rtol=1e-12, atol=1e-12)
    # the closed form the GPU tests use, including the exact zeros of the one-hot first / last cells (rows 0 and 1)
    cidx, cval, dval = interp_with_derivatives(axes, x)
    assert torch.equal(cidx, ref_idx)
    torch.testing.assert_close(cval, torch.from_numpy(GOLD[f"{tag}_val"]), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(dval, ref_dval, rtol=1e-12, atol=1e-12)
    assert torch.all(dval[:, :2] == 0) and torch.all(ref_dval[:, :2] == 0)


@pytest.mark.parametrize("kind,sizes", [("rbf", [11]), ("matern52", [9, 12]), ("rbf", [6, 7, 8])])
def test_closed_form_matches_autograd_through_dense_ski(kind, sizes):
    g = torch.Generator().manual_seed(len(sizes) + 3)
    d, n, t = len(sizes), 25, 3
    axes = ski.create_grid(sizes, [(0.0, 1.0)] * d, dtype=torch.float64)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    x[0] = torch.stack([a[0] + 0.5 * (a[1] - a[0]) for a in axes])      # first cell
    L = torch.randn(n, t, generator=g, dtype=torch.float64)
    R = torch.randn(n, t, generator=g, dtype=torch.float64)
    ls = [0.3 + 0.1 * i for i in range(d)]
    xr = x.clone().requires_grad_(True)
    (ref,) = torch.autograd.grad((L * (dense_ski(kind, xr, axes, ls, 1.7) @ R)).sum(), xr)
    got, mag = ski_input_grad(kind, x, axes, ls, 1.7, L, R)
    torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-10)
    assert torch.all(got[0] == 0) and torch.all(mag >= got.abs() - 1e-12)


# ---- autograd plumbing on fake plans ---------------------------------------------------------------------------------------------
class _FakePlan:
    """Stands in for engine.Plan: solves are rhs / 2 (K_hat = 2 I), K is zero, and every gradient entry point records its factors."""

    def __init__(self, n, d):
        self.n1 = self.n2 = self.row_count = n
        self.d, self.same, self.noise = d, True, 0.0
        self.calls = []
        self._hyp_key = None

    def set_hypers(self, kind, ls, os_=1.0, noise=0.0):
        self.noise = noise
        return self

    def kmv(self, v, add_noise=False):
        return torch.zeros_like(v)

    def rows(self, idx):
        return torch.zeros(idx.numel(), self.n2)

    def mbcg(self, rhs, n_tridiag, *a):
        info = type("I", (), {"iters": 3})()
        return rhs / 2, torch.eye(3).expand(max(n_tridiag, 1), 3, 3).clone(), info

    def slq_logdet(self, tmat, n):
        return 0.0

    def bilinear_grad(self, left, right):
        self.calls.append(("bilinear", left.clone(), right.clone()))
        return [0.0], 0.0

    def kmv_input_grad(self, g, v, dx1=True, dx2=True):
        self.calls.append(("kmv", g.clone(), v.clone()))
        return torch.full((self.n1, self.d), 2.0), None

    def dense_input_grad(self, w, dx1=True, dx2=True):
        self.calls.append(("dense", w.clone()))
        return torch.full((self.n1, self.d), 3.0), None

    def ski_input_grad(self, left, right):
        self.calls.append(("ski", left.clone(), right.clone()))
        return torch.full((self.n1, self.d), 4.0)


def _model(n=6, d=2, ski_op=False, x_grad=True, hyp_grad=True):
    from gpytorch_b200.operators import ConstantDiagLinearOperator, KernelLinearOperator, SKIKernelLinearOperator

    x = torch.rand(n, d).requires_grad_(x_grad)
    ls = torch.tensor(0.5).requires_grad_(hyp_grad)
    plan = _FakePlan(n, d)
    if ski_op:
        op = SKIKernelLinearOperator(x, "rbf", ls, torch.tensor(1.0), [8] * d, [0.0] * d, [0.2] * d)
        op._plan = plan
    else:
        op = KernelLinearOperator(x, None, "rbf", ls, torch.tensor(1.0), plan=plan)
    return op + ConstantDiagLinearOperator(torch.tensor(2.0), n), x, plan


def test_cg_branch_passes_the_hyperparameter_factors():
    from gpytorch_b200 import settings

    khat, x, plan = _model()
    y = torch.rand(6)
    with settings.max_cholesky_size(0), settings.num_trace_samples(4):
        iq, ld = khat.inv_quad_logdet(y, logdet=True)
        (iq + ld).backward()
    kinds = [c[0] for c in plan.calls]
    assert kinds == ["bilinear", "kmv"]
    torch.testing.assert_close(plan.calls[1][1], plan.calls[0][1], rtol=0, atol=0)
    torch.testing.assert_close(plan.calls[1][2], plan.calls[0][2], rtol=0, atol=0)
    assert plan.calls[1][1].shape == (6, 5) and torch.equal(x.grad, torch.full((6, 2), 2.0))
    # the solve: factors (-K_hat^-1 g, K_hat^-1 rhs), as for the hyper-parameters
    plan.calls.clear()
    x.grad = None
    rhs = torch.rand(6, 2)
    with settings.max_cholesky_size(0):
        khat.solve(rhs).sum().backward()
    assert [c[0] for c in plan.calls] == ["bilinear", "kmv"]
    torch.testing.assert_close(plan.calls[1][1], -torch.ones(6, 2) / 2)
    torch.testing.assert_close(plan.calls[1][2], rhs / 2)


def test_cholesky_branch_uses_the_dense_weight():
    khat, x, plan = _model(hyp_grad=False)
    y = torch.rand(6, 1)
    iq, ld = khat.inv_quad_logdet(y, logdet=True, reduce_inv_quad=False)
    (3.0 * iq.sum() + 0.5 * ld).backward()
    assert [c[0] for c in plan.calls] == ["dense"]
    sol = y / 2                                               # K_hat = 2 I on the fake plan
    w = -3.0 * sol @ sol.t() + 0.5 * torch.eye(6) / 2
    torch.testing.assert_close(plan.calls[0][1], w)
    assert torch.equal(x.grad, torch.full((6, 2), 3.0))


def test_kernel_sum_calls_every_term_and_ski_goes_to_its_entry():
    from gpytorch_b200 import settings
    from gpytorch_b200.operators import ConstantDiagLinearOperator, SumKernelLinearOperator

    a, xa, pa = _model()
    b, xb, pb = _model()
    s = SumKernelLinearOperator([a.kernel_op, b.kernel_op])
    for o, p in zip(s.ops, (pa, pb)):
        o._plan = p
    s.plan = lambda noise=0.0: pa
    khat = s + ConstantDiagLinearOperator(torch.tensor(2.0), 6)
    with settings.max_cholesky_size(0):
        khat.inv_quad(torch.rand(6)).backward()
    assert [c[0] for c in pa.calls] == ["bilinear", "kmv"] and [c[0] for c in pb.calls] == ["bilinear", "kmv"]
    assert torch.equal(xa.grad, torch.full((6, 2), 2.0)) and torch.equal(xb.grad, torch.full((6, 2), 2.0))
    pa.calls.clear(); pb.calls.clear()
    khat.inv_quad(torch.rand(6)).backward()                    # Cholesky branch: one dense call per term
    assert [c[0] for c in pa.calls] == ["bilinear", "dense"] and [c[0] for c in pb.calls] == ["bilinear", "dense"]

    k, x, plan = _model(ski_op=True)
    assert k.kernel_op.input_tensors() == [] and k.kernel_op.solve_input_tensors() == [k.kernel_op.x1]
    with settings.max_cholesky_size(0):
        k.inv_quad(torch.rand(6)).backward()
    assert [c[0] for c in plan.calls] == ["bilinear", "ski"] and torch.equal(x.grad, torch.full((6, 2), 4.0))
    plan.calls.clear()
    k.inv_quad(torch.rand(6)).backward()                       # Cholesky branch: the product form with the identity
    assert [c[0] for c in plan.calls] == ["bilinear", "ski"] and torch.equal(plan.calls[1][2], torch.eye(6))


def test_hyperparameter_only_training_makes_no_input_gradient_call():
    from gpytorch_b200 import settings

    for chol in (True, False):
        khat, x, plan = _model(x_grad=False)
        with settings.max_cholesky_size(800 if chol else 0):
            iq, ld = khat.inv_quad_logdet(torch.rand(6), logdet=True)
            (iq + ld).backward()
        assert all(c[0] == "bilinear" for c in plan.calls) and x.grad is None
        assert khat.kernel_op.lengthscale.grad is not None


def test_ski_input_grad_kernel_has_no_local_memory():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
    if not os.path.exists(tool) or not os.path.exists(lib):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = set()
    for i, line in enumerate(lines):
        m = re.search(r"ski_input_grad_tiled_kernelILi(\d)E", line)
        if "Function" in line and m:
            assert int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1)) == 0, line
            assert int(re.search(r"LOCAL:(\d+)", lines[i + 1]).group(1)) == 0, line
            seen.add(int(m.group(1)))
    assert seen == {1, 2, 3, 4}


def test_scale_to_bounds_matches_reference_module():
    from gpytorch_b200.utils.grid import ScaleToBounds

    m = ScaleToBounds(-1.0, 1.0).double()
    x = torch.from_numpy(GOLD["stb_x"]).clone().requires_grad_(True)
    y = m(x)
    torch.testing.assert_close(y, torch.from_numpy(GOLD["stb_train"]), rtol=1e-14, atol=1e-14)
    (g,) = torch.autograd.grad((y * torch.from_numpy(GOLD["stb_w"])).sum(), x)
    torch.testing.assert_close(g, torch.from_numpy(GOLD["stb_grad"]), rtol=1e-13, atol=1e-14)
    m.eval()
    torch.testing.assert_close(m(torch.from_numpy(GOLD["stb_xe"])), torch.from_numpy(GOLD["stb_eval"]), rtol=1e-14, atol=1e-14)
