"""Periodic plans keep a consistent state on the device (run with -m gpu): a refused gp_plan_set_periodic or gp_plan_set_hypers
leaves the plan as it was, so the gradient output the host sizes always matches what the engine writes; and nested ScaleKernels
around a PeriodicKernel compute the scaled periodic covariance, not an RBF one."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import periodic_oracle as po  # noqa: E402


def _points(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g) * 8 - 4


def test_refused_calls_leave_the_plan_unchanged(cuda_dev):
    from gpytorch_b200.engine import Plan

    n, d = 300, 2
    x = _points(n, d, 1).to(cuda_dev)
    V = torch.randn(n, 3, device=cuda_dev)
    m = Plan(x).set_hypers("matern52", [0.7, 1.1], 1.0, 0.0)
    ref_m = m.kmv(V)
    with pytest.raises(RuntimeError, match="gp_plan_set_periodic needs the kind GP_RBF"):
        m.set_periodic([1.3, 0.9])
    assert getattr(m, "_periodic", None) is None and torch.equal(m.kmv(V), ref_m)
    m.set_hypers("rbf", [0.7, 1.1], 1.0, 0.0)   # still a plain plan: two lengthscale gradients
    gl, _ = m.bilinear_grad(V, V)
    assert len(gl) == 2
    p = Plan(x).set_periodic([1.3, 0.9]).set_hypers("rbf", [0.7], 1.0, 0.0)
    ref_p = p.kmv(V)
    gl0, gs0 = p.bilinear_grad(V, V)
    with pytest.raises(RuntimeError, match="takes the kind GP_RBF"):
        p.set_hypers("matern52", [0.4, 0.5, 0.6][:d], 2.0, 0.0)
    assert p.lengthscale == [0.7] and torch.equal(p.kmv(V), ref_p)
    assert p.bilinear_grad(V, V) == (gl0, gs0) and len(gl0) == 1 + 2
    with pytest.raises(RuntimeError, match="1 or d"):
        p.set_periodic([1.0, 2.0, 3.0])
    assert torch.equal(p.kmv(V), ref_p)
    m.close(), p.close()


def test_nested_scale_kernels_on_the_device(cuda_dev):
    from gpytorch_b200 import kernels

    inner = kernels.ScaleKernel(kernels.PeriodicKernel())
    k = kernels.ScaleKernel(inner)
    k.outputscale, inner.outputscale = 2.0, 0.5
    inner.base_kernel.period_length, inner.base_kernel.lengthscale = 1.3, 0.8
    k = k.to(cuda_dev)
    x = _points(500, 1, 2)
    V = torch.randn(500, 4)
    out = (k(x.to(cuda_dev)) @ V.to(cuda_dev)).detach().double().cpu()
    ref = po.kernel(x, x, torch.tensor([0.8]), torch.tensor([1.3]), 1.0) @ V.double()
    assert ((out - ref).norm() / ref.norm()).item() < 1e-5
