"""Host checks of the kernel input gradient: the fp64 closed form (tests/xgrad_oracle.py) against fp64 autograd through
oracle.kernels and against the reference's own code (tests/golden/xgrad_golden.npz); the autograd plumbing of operators.py
asks the engine only for the inputs that need a gradient; the new kernel keeps its registers at d <= 20."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import kernels as ok
from xgrad_oracle import input_grad

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["rbf", "matern12", "matern32", "matern52"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ard", [False, True])
def test_closed_form_matches_fp64_autograd(kind, ard):
    g = torch.Generator().manual_seed(7 + KINDS.index(kind) + 10 * ard)
    n1, n2, d = 9, 14, 4
    x1 = torch.rand(n1, d, generator=g, dtype=torch.float64)
    x2 = torch.rand(n2, d, generator=g, dtype=torch.float64)
    ls = torch.linspace(0.3, 0.9, d, dtype=torch.float64) if ard else 0.55
    s = 1.3
    W = torch.randn(n1, n2, generator=g, dtype=torch.float64)
    a1, a2 = x1.clone().requires_grad_(), x2.clone().requires_grad_()
    F = (W * ok.kernel_matrix(kind, a1, a2, ls, s, x1_eq_x2=False)).sum()
    r1, r2 = torch.autograd.grad(F, (a1, a2))
    c1, c2 = input_grad(kind, x1, x2, ls, s, W)
    torch.testing.assert_close(c1, r1, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(c2, r2, rtol=1e-10, atol=1e-12)
    # square: both arguments are the same points; the diagonal has zero input gradient
    Ws = torch.randn(n1, n1, generator=g, dtype=torch.float64)
    a = x1.clone().requires_grad_()
    (rs,) = torch.autograd.grad((Ws * ok.kernel_matrix(kind, a, a, ls, s, x1_eq_x2=True)).sum(), (a,))
    torch.testing.assert_close(input_grad(kind, x1, x1, ls, s, Ws, same=True), rs, rtol=1e-9, atol=1e-11)


def test_closed_form_matches_reference_goldens():
    gd = np.load(os.path.join(ROOT, "tests", "golden", "xgrad_golden.npz"))
    tags = sorted({k.split("_")[0] for k in gd.files})
    assert tags == ["a", "b", "c"]
    for tag in tags:
        f = {k: torch.from_numpy(np.asarray(gd[f"{tag}_{k}"])) for k in ("x1", "x2", "ls", "W", "Wsq", "dx1", "dx2", "dxsq")}
        s = float(gd[f"{tag}_os"])
        d1, d2 = input_grad("rbf", f["x1"], f["x2"], f["ls"], s, f["W"])
        torch.testing.assert_close(d1, f["dx1"], rtol=1e-9, atol=1e-11)
        torch.testing.assert_close(d2, f["dx2"], rtol=1e-9, atol=1e-11)
        ds = input_grad("rbf", f["x1"], f["x1"], f["ls"], s, f["Wsq"], same=True)
        torch.testing.assert_close(ds, f["dxsq"], rtol=1e-9, atol=1e-11)


class _FakePlan:
    """Stands in for engine.Plan on the CPU: records which input gradients the autograd functions ask for."""

    def __init__(self, n1, n2, d, same):
        self.n1, self.n2, self.d, self.same, self.row_count = n1, n2, d, same, n1
        self.calls = []
        self._hyp_key = None

    def set_hypers(self, *a):
        return self

    def kmv(self, v, add_noise=False):
        return torch.zeros(self.n1 if v.size(0) == self.n2 else self.n2, *v.shape[1:])

    def rows(self, idx):
        return torch.zeros(idx.numel(), self.n2)

    def _out(self, dx1, dx2):
        return (torch.full((self.n1, self.d), 2.0) if dx1 else None,
                torch.full((self.n2, self.d), 3.0) if (dx2 and not self.same) else None)

    def kmv_input_grad(self, g, v, dx1=True, dx2=True):
        self.calls.append(("kmv", dx1, dx2, tuple(g.shape), tuple(v.shape)))
        return self._out(dx1, dx2)

    def dense_input_grad(self, w, dx1=True, dx2=True):
        self.calls.append(("dense", dx1, dx2, tuple(w.shape)))
        return self._out(dx1, dx2)


def _op(n1, n2, d, x1_grad, x2_grad, same=False):
    from gpytorch_b200.operators import KernelLinearOperator

    x1 = torch.rand(n1, d).requires_grad_(x1_grad)
    x2 = None if same else torch.rand(n2, d).requires_grad_(x2_grad)
    plan = _FakePlan(n1, n1 if same else n2, d, same)
    op = KernelLinearOperator(x1, x2, "rbf", torch.tensor(0.5), torch.tensor(1.0), plan=plan)
    return op, plan


@pytest.mark.parametrize("x1_grad,x2_grad", [(True, False), (False, True), (True, True), (False, False)])
def test_kernel_matmul_asks_only_for_needed_inputs(x1_grad, x2_grad):
    op, plan = _op(5, 8, 3, x1_grad, x2_grad)
    op._transpose_nonbatch = lambda: op        # K^T g for the right-hand side's gradient, on the same fake plan
    rhs = torch.rand(8, 2, requires_grad=True)
    op.matmul(rhs).sum().backward()
    if x1_grad or x2_grad:
        assert plan.calls == [("kmv", x1_grad, x2_grad, (5, 2), (8, 2))]
    else:
        assert plan.calls == []
    assert (op.x1.grad is not None) == x1_grad and (op.x2.grad is not None) == x2_grad
    if x1_grad:
        assert torch.equal(op.x1.grad, torch.full((5, 3), 2.0))
    if x2_grad:
        assert torch.equal(op.x2.grad, torch.full((8, 3), 3.0))


def test_kernel_dense_asks_only_for_needed_inputs_and_square_gets_one_total():
    op, plan = _op(5, 8, 3, False, True)
    op.to_dense().sum().backward()
    assert plan.calls == [("dense", False, True, (5, 8))] and op.x1.grad is None
    sq, psq = _op(6, 6, 2, True, False, same=True)
    assert sq.input_tensors() == [sq.x1]
    (sq.to_dense() * 2).sum().backward()
    assert psq.calls == [("dense", True, False, (6, 6))] and torch.equal(sq.x1.grad, torch.full((6, 2), 2.0))
    # hyper-parameters only: the input-gradient entry points are not called (training behaves as before)
    op2, p2 = _op(5, 8, 3, False, False)
    op2.lengthscale.requires_grad_(True)
    op2.to_dense().sum()
    assert p2.calls == []


def test_kernel_sum_calls_every_term():
    from gpytorch_b200.operators import SumKernelLinearOperator

    a, pa = _op(4, 6, 2, True, False)
    b, pb = _op(4, 6, 2, True, False)
    s = SumKernelLinearOperator([a, b])
    for o, p in zip(s.ops, (pa, pb)):
        o._plan = p
    s.plan = lambda noise=0.0: pa
    assert s.input_tensors() == [a.x1, a.x2, b.x1, b.x2]
    s.matmul(torch.rand(6, 3)).sum().backward()
    assert pa.calls == [("kmv", True, False, (4, 3), (6, 3))] and pb.calls == pa.calls
    assert torch.equal(a.x1.grad, torch.full((4, 2), 2.0))


def test_ski_and_detached_operators_carry_no_input_gradient():
    from gpytorch_b200.operators import SKIKernelLinearOperator

    x = torch.rand(10, 2, requires_grad=True)
    ski = SKIKernelLinearOperator(x, "rbf", torch.tensor(0.5), torch.tensor(1.0), [8, 8], [0.0, 0.0], [0.2, 0.2])
    assert ski.input_tensors() == []
    op, _ = _op(5, 8, 3, True, True)
    det = op.detach()
    assert not any(t.requires_grad for t in det.input_tensors())


def test_input_grad_kernel_has_no_local_memory_at_small_d():
    """cuobjdump resource usage of xgrad_kernel<KIND, DP, TW>: no stack / spills for the instantiations used at d <= 20."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
    if not os.path.exists(tool) or not os.path.exists(lib):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        m = re.search(r"xgrad_kernelILi(\d)ELi(\d+)ELi(\d+)E", line)
        if "Function" not in line or not m:
            continue
        kind, dp, tw = (int(v) for v in m.groups())
        if dp <= 24:
            stack = int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1))
            assert stack == 0, f"xgrad_kernel<{kind}, {dp}, {tw}>: {stack} bytes of local memory"
            seen += 1
    assert seen == 4 * 5 * 3, seen   # 4 kinds x DP in {4, 8, 12, 16, 24} x TW in {0 (dense), 8, 32}
