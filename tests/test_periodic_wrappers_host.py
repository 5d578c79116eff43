"""Periodic kernels under every wrapper, without a GPU: each composition either builds a periodic operator that keeps the period
(with every outputscale folded in) or refuses; none silently rebuilds a plain RBF operator over the raw inputs.  Also: a periodic
operator re-sends its period and hyper-parameters to a cached plan only when their host values change."""
import pytest
import torch


def _periodic_terms(op):
    from gpytorch_b200 import operators as ops

    return [o for o in (op.ops if isinstance(op, ops.SumKernelLinearOperator) else [op]) if isinstance(o, ops.PeriodicKernelLinearOperator)]


def test_nested_scale_kernels_keep_the_period_and_both_scales():
    from gpytorch_b200 import kernels, operators as ops

    inner = kernels.ScaleKernel(kernels.PeriodicKernel())
    k = kernels.ScaleKernel(inner)
    k.outputscale, inner.outputscale = 2.0, 3.0
    inner.base_kernel.period_length = 1.7
    op = k(torch.randn(10, 1))
    assert isinstance(op, ops.PeriodicKernelLinearOperator)
    assert torch.allclose(op.period, torch.tensor(1.7)) and torch.allclose(op.outputscale, torch.tensor(6.0))
    op.outputscale.backward()
    assert k.raw_outputscale.grad is not None and inner.raw_outputscale.grad is not None
    op3 = kernels.ScaleKernel(kernels.ScaleKernel(kernels.ScaleKernel(kernels.PeriodicKernel())))(torch.randn(6, 2))
    assert isinstance(op3, ops.PeriodicKernelLinearOperator)
    b = kernels.ScaleKernel(kernels.ScaleKernel(kernels.PeriodicKernel(batch_shape=torch.Size([2]))))(torch.randn(2, 8, 1))
    assert all(isinstance(o, ops.PeriodicKernelLinearOperator) for o in b.ops)


WRAPPERS = {
    "periodic": lambda P: P(),
    "scale": lambda P: __import__("gpytorch_b200.kernels", fromlist=["x"]).ScaleKernel(P()),
    "scale_scale": lambda P: _k().ScaleKernel(_k().ScaleKernel(P())),
    "sum": lambda P: P() + _k().RBFKernel(),
    "sum_of_nested_scale": lambda P: _k().ScaleKernel(_k().ScaleKernel(P())) + _k().ScaleKernel(_k().RBFKernel()),
    "scale_of_sum": lambda P: _k().ScaleKernel(P() + _k().RBFKernel()),
    "scale_scale_of_sum": lambda P: _k().ScaleKernel(_k().ScaleKernel(_k().ScaleKernel(P()) + _k().RBFKernel())),
    "product": lambda P: P() * _k().RBFKernel(),
    "product_of_nested_scale": lambda P: _k().ProductKernel(_k().ScaleKernel(_k().ScaleKernel(P())), _k().RBFKernel()),
    "grid": lambda P: _k().GridInterpolationKernel(P(), 16, num_dims=1),
    "grid_of_scale": lambda P: _k().GridInterpolationKernel(_k().ScaleKernel(P()), 16, num_dims=1),
    "multitask": lambda P: _k().MultitaskKernel(_k().ScaleKernel(_k().ScaleKernel(P())), num_tasks=2),
}


# products, SKI and multitask models do not take a periodic kernel; every other wrapper keeps it
REFUSED = {"product", "product_of_nested_scale", "grid", "grid_of_scale", "multitask"}


def _k():
    from gpytorch_b200 import kernels

    return kernels


@pytest.mark.parametrize("name", sorted(WRAPPERS))
def test_every_wrapper_keeps_the_period_or_refuses(name):
    from gpytorch_b200 import operators as ops

    def P():
        k = _k().PeriodicKernel()
        k.period_length = 1.25
        return k

    x = torch.randn(12, 1)
    if name in REFUSED:
        with pytest.raises((NotImplementedError, RuntimeError)):
            k = WRAPPERS[name](P)
            k.forward(x, x) if isinstance(k, _k().MultitaskKernel) else k(x)
        return
    k = WRAPPERS[name](P)
    op = k(x)
    terms = _periodic_terms(op)
    assert terms, f"{name}: no periodic operator in {type(op).__name__}"
    for t in terms:
        assert torch.allclose(t.period, torch.tensor(1.25))
    if isinstance(op, ops.SumKernelLinearOperator):
        assert all(type(o) in (ops.KernelLinearOperator, ops.PeriodicKernelLinearOperator) for o in op.ops)


class _FakePlan:
    def __init__(self):
        self.calls = []

    def set_periodic(self, per):
        self.calls.append(("periodic", tuple(per)))

    def set_hypers(self, kind, ls, os_, nz):
        self.calls.append(("hypers", tuple(ls), os_, nz))


def test_period_and_hypers_resent_only_when_their_values_change(monkeypatch):
    from gpytorch_b200 import operators as ops

    fake = _FakePlan()
    monkeypatch.setattr(ops, "_get_plan", lambda *a, **k: fake)
    x = torch.randn(5, 1)

    def op(per, ls):
        return ops.PeriodicKernelLinearOperator(x, None, torch.tensor(ls), torch.tensor(per), torch.tensor(1.5))

    op(2.0, 0.5).plan(0.1)
    assert [c[0] for c in fake.calls] == ["periodic", "hypers"]
    op(2.0, 0.5).plan(0.1)                 # a new operator over the same plan and values: nothing is re-sent (no re-pack)
    assert len(fake.calls) == 2
    op(2.0, 0.7).plan(0.1)                 # the lengthscale changed: the hyper-parameters only
    assert [c[0] for c in fake.calls[2:]] == ["hypers"]
    op(2.5, 0.7).plan(0.1)                 # the period changed: the period only
    assert [c[0] for c in fake.calls[3:]] == ["periodic"]
