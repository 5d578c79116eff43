"""Periodic kernels without a GPU: the fp64 oracle against the reference's own PeriodicKernel (tests/golden/periodic_golden.npz), the
bound's independence of |x|, the kernel's parameters, constraints, setters and refusals, operator construction and slots, the C
ABI and the gradient kernel's ptxas report."""
import os
import re

import numpy as np
import pytest
import torch

import periodic_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "periodic_golden.npz"))


def _cases():
    return range(int(GOLD["ncases"]))


@pytest.mark.parametrize("c", list(_cases()))
def test_oracle_matches_reference_golden(c):
    d, ard, n1, n2, B = (int(v) for v in GOLD[f"c{c}_meta"])
    for b in range(max(B, 1)):
        sl = (lambda a: a[b]) if B else (lambda a: a)
        x1, x2 = torch.tensor(sl(GOLD[f"c{c}_x1"])), torch.tensor(sl(GOLD[f"c{c}_x2"]))
        ls, per = torch.tensor(sl(GOLD[f"c{c}_ls"])).reshape(-1), torch.tensor(sl(GOLD[f"c{c}_per"])).reshape(-1)
        assert torch.allclose(po.kernel(x1, x2, ls, per), torch.tensor(sl(GOLD[f"c{c}_K"])), rtol=0, atol=1e-12)
        assert torch.allclose(po.kernel(x1, x1, ls, per), torch.tensor(sl(GOLD[f"c{c}_Kxx"])), rtol=0, atol=1e-12)
        assert torch.allclose(torch.ones(n1, dtype=torch.float64), torch.tensor(sl(GOLD[f"c{c}_diag"])), atol=1e-12)
        gl, gp_, _ = po.grads(x1, x2, ls, per, torch.tensor(sl(GOLD[f"c{c}_W"])))
        assert torch.allclose(gl, torch.tensor(sl(GOLD[f"c{c}_gls"])).reshape(-1), rtol=1e-10, atol=1e-10)
        assert torch.allclose(gp_, torch.tensor(sl(GOLD[f"c{c}_gper"])).reshape(-1), rtol=1e-10, atol=1e-10)


def test_bound_does_not_grow_with_x():
    x = torch.rand(200, 1) * 10
    V = torch.randn(200, 3)
    ls, per = torch.tensor([0.7]), torch.tensor([1.3])
    b0 = po.kmv_bound(x, x, ls, per, V, 1.0, "tc", 1, 4, same=True)
    b1 = po.kmv_bound(x + 1.3 * 70000, x + 1.3 * 70000, ls, per, V, 1.0, "tc", 1, 4, same=True)
    # the shifted fp32 inputs are other points, so compare the bound's scale, not entry by entry
    assert float(b1.max()) <= 1.1 * float(b0.max()) and float(b0.max()) <= 1.1 * float(b1.max())


def test_embedding_identity():
    x1, x2 = torch.randn(30, 3) * 50, torch.randn(20, 3) * 50
    ls, per = torch.tensor([0.5, 1.0, 2.0]), torch.tensor([1.1, 0.7, 3.0])
    u1, u2 = po.embed(x1, ls, per), po.embed(x2, ls, per)
    K = torch.exp(-0.5 * torch.cdist(u1, u2) ** 2)
    assert torch.allclose(K, po.kernel(x1, x2, ls, per), atol=1e-12)


def test_kernel_parameters_setters_and_refusals():
    from gpytorch_b200 import constraints, kernels

    k = kernels.PeriodicKernel()
    assert k.raw_period_length.shape == (1, 1) and k.raw_lengthscale.shape == (1, 1)
    k.period_length = 2.5
    k.lengthscale = 0.3
    assert torch.allclose(k.period_length, torch.tensor([[2.5]])) and torch.allclose(k.lengthscale, torch.tensor([[0.3]]))
    ka = kernels.PeriodicKernel(ard_num_dims=3, batch_shape=torch.Size([2]))
    assert ka.raw_period_length.shape == (2, 1, 3) and ka.raw_lengthscale.shape == (2, 1, 3)
    kc = kernels.PeriodicKernel(period_length_constraint=constraints.Positive())
    assert isinstance(kc.raw_period_length_constraint, constraints.Positive)
    with pytest.raises(NotImplementedError, match="priors are not available"):
        kernels.PeriodicKernel(period_length_prior=object())
    with pytest.raises(NotImplementedError, match="products with a PeriodicKernel factor"):
        kernels.PeriodicKernel() * kernels.RBFKernel()
    with pytest.raises(NotImplementedError, match="products with a PeriodicKernel factor"):
        kernels.ScaleKernel(kernels.PeriodicKernel()) * kernels.RBFKernel()
    with pytest.raises(NotImplementedError, match="PeriodicKernel base kernel of a GridInterpolationKernel"):
        kernels.GridInterpolationKernel(kernels.PeriodicKernel(), 16, num_dims=1)
    mk = kernels.MultitaskKernel(kernels.ScaleKernel(kernels.PeriodicKernel()), num_tasks=2)
    with pytest.raises(NotImplementedError, match="PeriodicKernel data kernel of a MultitaskKernel"):
        mk.forward(torch.zeros(4, 1), torch.zeros(4, 1))


def test_operator_dispatch_refusals_and_slot_keys():
    from gpytorch_b200 import kernels, operators as ops

    x = torch.randn(10, 2)
    k = kernels.ScaleKernel(kernels.PeriodicKernel(ard_num_dims=2, active_dims=[0, 2]))
    op = k(torch.randn(10, 3))
    assert isinstance(op, ops.PeriodicKernelLinearOperator) and op.x1.shape == (10, 2)
    assert op.period.shape == (2,) and op.outputscale is not None and len(op.hyper_tensors()) == 3
    op2 = kernels.PeriodicKernel()(x)
    assert isinstance(op2, ops.PeriodicKernelLinearOperator) and op2.period.dim() == 0
    cross = kernels.PeriodicKernel()(x, torch.randn(7, 2))
    for o in (cross._transpose_nonbatch(), cross.detach(), cross[2:5, 1:4]):
        assert isinstance(o, ops.PeriodicKernelLinearOperator) and o.period is not None
    s = kernels.ScaleKernel(kernels.PeriodicKernel()) + kernels.ScaleKernel(kernels.RBFKernel())
    so = s(x)
    assert isinstance(so, ops.SumKernelLinearOperator)
    assert isinstance(so.ops[0], ops.PeriodicKernelLinearOperator) and type(so.ops[1]) is ops.KernelLinearOperator
    assert so.ops[0]._plan_slot == ops._slot("periodic", "sum_term", 0) and so.ops[1]._plan_slot == ops._slot("plain", "sum_term", 1)
    sc = kernels.ScaleKernel(kernels.PeriodicKernel() + kernels.RBFKernel())(x)
    assert isinstance(sc.ops[0], ops.PeriodicKernelLinearOperator) and sc.ops[0].period is not None
    b = kernels.ScaleKernel(kernels.PeriodicKernel(batch_shape=torch.Size([3])))(torch.randn(3, 10, 1))
    assert all(isinstance(o, ops.PeriodicKernelLinearOperator) for o in b.ops)
    with pytest.raises(NotImplementedError, match="inputs of a periodic operator"):
        kernels.PeriodicKernel()(x.clone().requires_grad_(True))
    with pytest.raises(NotImplementedError, match="1 <= d <= 16"):
        kernels.PeriodicKernel()(torch.randn(5, 17))
    with pytest.raises(NotImplementedError, match="products that contain a periodic operator"):
        op2.mul(op2)


def test_gradients_split_onto_parameter_shapes():
    from gpytorch_b200 import operators as ops

    class _P:
        def bilinear_grad(self, left, right):
            return [1.0, 2.0, 3.0, 4.0], 6.0

    op = ops.PeriodicKernelLinearOperator(torch.zeros(4, 2), None, torch.ones(2), torch.ones(2) * 2, torch.tensor(1.5))
    op.plan = lambda noise=0.0: _P()
    g = op._bilinear_derivative_list(None, None)
    assert g[0].tolist() == [1.0, 2.0] and g[1].tolist() == [3.0, 4.0] and float(g[2]) == 6.0


def test_plan_slot_keys_are_disjoint():
    from gpytorch_b200 import operators as ops

    others = ("plain", "rq", "poly", "task", "spectral", "kron", "deriv", "additive", "lcm", "ppoly", "sum", "product")
    used = {ops._slot(f, r, i) for f in others for r in ops._SLOT_ROLES for i in range(4)}
    mine = {ops._slot("periodic", "own"), ops._slot("periodic", "lowrank"), *(ops._slot("periodic", "sum_term", i) for i in range(4))}
    assert len(mine) == 6 and not (mine & used)
    op = ops.PeriodicKernelLinearOperator(torch.zeros(4, 1), None, torch.tensor(1.0), torch.tensor(2.0))
    assert op._plan_slot == ops._slot("periodic", "own")
    assert ops.LowRankUpdatedKernelLinearOperator(op, torch.ones(4, 1)).base._plan_slot == ops._slot("periodic", "lowrank")


def test_c_abi_declares_periodic():
    h = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert "int gp_plan_set_periodic(gp_plan* plan, const float* period, int n_period, int d);" in h
    from gpytorch_b200 import _lib

    assert "gp_plan_set_periodic" in _lib.PROTOTYPES


def test_ptxas_reports_no_spills_in_periodic_kernels():
    log = os.path.join(ROOT, "gpytorch_b200", "build", "periodic.o.log")
    if not os.path.exists(log):
        pytest.skip("not built")
    txt = open(log).read()
    props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", txt)
    names = [p[0] for p in props if "periodic" in p[0]]
    assert sum("periodic_bilinear_kernel" in n for n in names) == 16
    for name, st, ss, sl in props:
        assert (st, ss, sl) == ("0", "0", "0"), name
