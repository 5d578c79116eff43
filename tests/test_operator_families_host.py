"""Host-side tests of the single-plan kernel operator families (plain, RQ, polynomial, periodic, piecewise polynomial and spectral
mixture): the engine calls each family makes on its plans, the plan-cache keys the operators ask for, and the folding of nested
ScaleKernels.  The engine is replaced by recording fakes, so none of this needs a GPU."""
import itertools

import pytest
import torch

from gpytorch_b200 import kernels, operators


def _norm(v):
    """An engine-call argument as a comparable literal: floats rounded to 6 digits, tensors and lists element by element."""
    if torch.is_tensor(v):
        return _norm(v.reshape(-1).tolist())
    if isinstance(v, (list, tuple)):
        return [_norm(t) for t in v]
    if isinstance(v, float):
        return round(v, 6)
    return v


class _RecPlan:
    """A plan that records every set_* call as (plan number, name, arguments)."""

    def __init__(self, log, plans, x1, x2):
        self._log, self._plans = log, plans
        self.x1, self.x2 = x1, x2
        self._n = len(plans)
        plans.append(self)

    def __getattr__(self, name):
        if not name.startswith("set_"):
            raise AttributeError(name)

        def call(*args):
            if name == "set_lowrank":
                self._lowrank = args[0]
                args = (list(args[0].shape),)
            elif name in ("set_sum", "set_product"):
                args = ([p._n for p in args[0]],)
            self._log.append((self._n, name, _norm(args)))
        return call

    def close(self):
        pass

    def rows(self, idx):
        return torch.zeros(idx.numel(), self.x1.size(0) if self.x2 is None else self.x2.size(0))


def _recorder(monkeypatch):
    """Patch the plan cache with a recording one: one fake plan per (inputs, backend, slot), as the real cache keeps one per key."""
    log, plans, cache = [], [], {}

    def fake_get_plan(x1, x2, backend, row_begin, row_count, comm, slot=0, owner=None):
        key = (x1.data_ptr(), tuple(x1.shape), None if x2 is None else (x2.data_ptr(), tuple(x2.shape)), backend, slot)
        if key not in cache:
            cache[key] = _RecPlan(log, plans, x1, x2)
        return cache[key]

    monkeypatch.setattr(operators, "_get_plan", fake_get_plan)
    monkeypatch.setattr(operators, "Plan", lambda x1, x2, **kw: _RecPlan(log, plans, x1, x2))
    operators.clear_plan_cache()
    return log


def _t(*v):
    return torch.tensor(v[0] if len(v) == 1 else list(v))


# family -> (constructor from (x1, x2, a parameter value, outputscale), may it be a sum term)
FAMILIES = {
    "plain": (lambda x1, x2, a, s: operators.KernelLinearOperator(x1, x2, "matern52", _t(a, 2 * a), s), True),
    "rq": (lambda x1, x2, a, s: operators.RQKernelLinearOperator(x1, x2, _t(a), _t(1.5), s), True),
    "poly": (lambda x1, x2, a, s: operators.PolynomialKernelLinearOperator(x1, x2, 3, _t(a), s), True),
    "periodic": (lambda x1, x2, a, s: operators.PeriodicKernelLinearOperator(x1, x2, _t(a), _t(2.0, 3.0), s), True),
    "ppoly": (lambda x1, x2, a, s: operators.PiecewisePolynomialKernelLinearOperator(x1, x2, 2, _t(a), s), False),
    "spectral": (lambda x1, x2, a, s: operators.SpectralMixtureKernelLinearOperator(
        x1, x2, _t(a, 0.25), _t([[[0.5, 1.0]], [[0.75, 0.125]]]), _t([[[1.0, 2.0]], [[0.5, 0.25]]]), s), False),
}


def _run(family, monkeypatch):
    make, summable = FAMILIES[family]
    log = _recorder(monkeypatch)
    x = torch.arange(12.0).reshape(6, 2) / 8
    xs = torch.arange(8.0).reshape(4, 2) / 5
    n1, n2, U = _t(0.25), _t(0.5), torch.ones(6, 2)
    steps = []

    def step(name, fn):
        start = len(log)
        fn()
        steps.append((name, log[start:]))

    op = make(x, None, 0.5, _t(2.0))
    step("plan twice", lambda: (op.plan(n1), op.plan(n1)))
    step("equal operator", lambda: make(x, None, 0.5, _t(2.0)).plan(n1))
    step("new noise", lambda: make(x, None, 0.5, _t(2.0)).plan(n2))
    op3 = make(x, None, 0.75, _t(2.0))
    step("new parameter", lambda: op3.plan(n2))
    cross = make(x, xs, 0.75, _t(2.0))
    step("cross", lambda: cross.plan())
    step("transpose", lambda: cross._transpose_nonbatch().plan())
    step("slice", lambda: op3[1:4, :].plan())
    step("row", lambda: op3[2])
    step("detach", lambda: op3.detach().plan(n2))
    if summable:
        step("sum", lambda: (op3 + make(x, None, 0.5, _t(3.0))).plan(n2))
    step("low rank", lambda: operators.LowRankUpdatedKernelLinearOperator(op3, U).plan(n2))
    step("plan again", lambda: op3.plan(n2))
    return steps


# Recorded at the commit before the single-plan operators were merged into KernelLinearOperator: the number, order and
# arguments of the engine calls of every family.
EXPECTED = {'plain': [('plan twice', [(0, 'set_hypers', ['matern52', [0.5, 1.0], 2.0, 0.25])]),
                      ('equal operator', [(0, 'set_hypers', ['matern52', [0.5, 1.0], 2.0, 0.25])]),
                      ('new noise', [(0, 'set_hypers', ['matern52', [0.5, 1.0], 2.0, 0.5])]),
                      ('new parameter', [(0, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.5])]),
                      ('cross', [(1, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.0])]),
                      ('transpose', [(2, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.0])]),
                      ('slice', [(3, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.0])]),
                      ('row', [(0, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.0])]),
                      ('detach', [(0, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.5])]),
                      ('sum',
                       [(4, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.0]),
                        (5, 'set_hypers', ['matern52', [0.5, 1.0], 3.0, 0.0]),
                        (6, 'set_sum', [[4, 5]]),
                        (6, 'set_hypers', ['rbf', [1.0], 1.0, 0.5])]),
                      ('low rank', [(7, 'set_hypers', ['matern52', [0.75, 1.5], 2.0, 0.5]), (7, 'set_lowrank', [[6, 2]])]),
                      ('plan again', [])],
            'rq': [('plan twice', [(0, 'set_hypers_rq', [[0.5], 1.5, 2.0, 0.25])]),
                   ('equal operator', [(0, 'set_hypers_rq', [[0.5], 1.5, 2.0, 0.25])]),
                   ('new noise', [(0, 'set_hypers_rq', [[0.5], 1.5, 2.0, 0.5])]),
                   ('new parameter', [(0, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.5])]),
                   ('cross', [(1, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.0])]),
                   ('transpose', [(2, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.0])]),
                   ('slice', [(3, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.0])]),
                   ('row', [(0, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.0])]),
                   ('detach', [(0, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.5])]),
                   ('sum',
                    [(4, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.0]),
                     (5, 'set_hypers_rq', [[0.5], 1.5, 3.0, 0.0]),
                     (6, 'set_sum', [[4, 5]]),
                     (6, 'set_hypers', ['rbf', [1.0], 1.0, 0.5])]),
                   ('low rank', [(7, 'set_hypers_rq', [[0.75], 1.5, 2.0, 0.5]), (7, 'set_lowrank', [[6, 2]])]),
                   ('plan again', [])],
            'poly': [('plan twice', [(0, 'set_hypers_poly', [3, 0.5, 2.0, 0.25])]),
                     ('equal operator', [(0, 'set_hypers_poly', [3, 0.5, 2.0, 0.25])]),
                     ('new noise', [(0, 'set_hypers_poly', [3, 0.5, 2.0, 0.5])]),
                     ('new parameter', [(0, 'set_hypers_poly', [3, 0.75, 2.0, 0.5])]),
                     ('cross', [(1, 'set_hypers_poly', [3, 0.75, 2.0, 0.0])]),
                     ('transpose', [(2, 'set_hypers_poly', [3, 0.75, 2.0, 0.0])]),
                     ('slice', [(3, 'set_hypers_poly', [3, 0.75, 2.0, 0.0])]),
                     ('row', [(0, 'set_hypers_poly', [3, 0.75, 2.0, 0.0])]),
                     ('detach', [(0, 'set_hypers_poly', [3, 0.75, 2.0, 0.5])]),
                     ('sum',
                      [(4, 'set_hypers_poly', [3, 0.75, 2.0, 0.0]),
                       (5, 'set_hypers_poly', [3, 0.5, 3.0, 0.0]),
                       (6, 'set_sum', [[4, 5]]),
                       (6, 'set_hypers', ['rbf', [1.0], 1.0, 0.5])]),
                     ('low rank', [(7, 'set_hypers_poly', [3, 0.75, 2.0, 0.5]), (7, 'set_lowrank', [[6, 2]])]),
                     ('plan again', [])],
            'periodic': [('plan twice', [(0, 'set_periodic', [[2.0, 3.0]]), (0, 'set_hypers', ['rbf', [0.5], 2.0, 0.25])]),
                         ('equal operator', []),
                         ('new noise', [(0, 'set_hypers', ['rbf', [0.5], 2.0, 0.5])]),
                         ('new parameter', [(0, 'set_hypers', ['rbf', [0.75], 2.0, 0.5])]),
                         ('cross', [(1, 'set_periodic', [[2.0, 3.0]]), (1, 'set_hypers', ['rbf', [0.75], 2.0, 0.0])]),
                         ('transpose', [(2, 'set_periodic', [[2.0, 3.0]]), (2, 'set_hypers', ['rbf', [0.75], 2.0, 0.0])]),
                         ('slice', [(3, 'set_periodic', [[2.0, 3.0]]), (3, 'set_hypers', ['rbf', [0.75], 2.0, 0.0])]),
                         ('row', [(0, 'set_hypers', ['rbf', [0.75], 2.0, 0.0])]),
                         ('detach', [(0, 'set_hypers', ['rbf', [0.75], 2.0, 0.5])]),
                         ('sum',
                          [(4, 'set_periodic', [[2.0, 3.0]]),
                           (4, 'set_hypers', ['rbf', [0.75], 2.0, 0.0]),
                           (5, 'set_periodic', [[2.0, 3.0]]),
                           (5, 'set_hypers', ['rbf', [0.5], 3.0, 0.0]),
                           (6, 'set_sum', [[4, 5]]),
                           (6, 'set_hypers', ['rbf', [1.0], 1.0, 0.5])]),
                         ('low rank',
                          [(7, 'set_periodic', [[2.0, 3.0]]), (7, 'set_hypers', ['rbf', [0.75], 2.0, 0.5]), (7, 'set_lowrank', [[6, 2]])]),
                         ('plan again', [])],
            'ppoly': [('plan twice', [(0, 'set_hypers_pp', [2, [0.5], 2.0, 0.25])]),
                      ('equal operator', [(0, 'set_hypers_pp', [2, [0.5], 2.0, 0.25])]),
                      ('new noise', [(0, 'set_hypers_pp', [2, [0.5], 2.0, 0.5])]),
                      ('new parameter', [(0, 'set_hypers_pp', [2, [0.75], 2.0, 0.5])]),
                      ('cross', [(1, 'set_hypers_pp', [2, [0.75], 2.0, 0.0])]),
                      ('transpose', [(2, 'set_hypers_pp', [2, [0.75], 2.0, 0.0])]),
                      ('slice', [(3, 'set_hypers_pp', [2, [0.75], 2.0, 0.0])]),
                      ('row', [(0, 'set_hypers_pp', [2, [0.75], 2.0, 0.0])]),
                      ('detach', [(0, 'set_hypers_pp', [2, [0.75], 2.0, 0.5])]),
                      ('low rank', [(4, 'set_hypers_pp', [2, [0.75], 2.0, 0.5]), (4, 'set_lowrank', [[6, 2]])]),
                      ('plan again', [])],
            'spectral': [('plan twice',
                          [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.25]),
                           (0, 'set_spectral', [[0.5, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('equal operator',
                          [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.25]),
                           (0, 'set_spectral', [[0.5, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('new noise',
                          [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.5]),
                           (0, 'set_spectral', [[0.5, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('new parameter',
                          [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.5]),
                           (0, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('cross',
                          [(1, 'set_hypers', ['rbf', 1.0, 2.0, 0.0]),
                           (1, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('transpose',
                          [(2, 'set_hypers', ['rbf', 1.0, 2.0, 0.0]),
                           (2, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('slice',
                          [(3, 'set_hypers', ['rbf', 1.0, 2.0, 0.0]),
                           (3, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('row', [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.0])]),
                         ('detach',
                          [(0, 'set_hypers', ['rbf', 1.0, 2.0, 0.5]),
                           (0, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]])]),
                         ('low rank',
                          [(4, 'set_hypers', ['rbf', 1.0, 2.0, 0.5]),
                           (4, 'set_spectral', [[0.75, 0.25], [0.5, 1.0, 0.75, 0.125], [1.0, 2.0, 0.5, 0.25]]),
                           (4, 'set_lowrank', [[6, 2]])]),
                         ('plan again', [])]}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_engine_calls_per_family(family, monkeypatch):
    assert _run(family, monkeypatch) == EXPECTED[family]


# ---- plan-cache slots ----------------------------------------------------------------------------------------------------------
FAMILY_NAMES = ("plain", "rq", "poly", "periodic", "ppoly", "spectral", "task", "kron", "deriv", "lcm", "additive", "sum", "product")


def test_slot_keys_are_distinct_except_rq_and_poly_on_plain():
    keys = {(f, r, i): operators._slot(f, r, i) for f in FAMILY_NAMES for r in operators._SLOT_ROLES for i in range(4)}
    for a, b in itertools.combinations(keys, 2):
        shared = {a[0], b[0]} <= {"plain", "rq", "poly"} and a[1:] == b[1:]
        assert (keys[a] == keys[b]) == shared, (a, b)


class _FakePlan:
    def __init__(self, x1, x2, backend="auto", row_begin=0, row_count=0, comm=None):
        self.x1, self.x2 = x1, x2

    def __getattr__(self, name):
        if not name.startswith("set_"):
            raise AttributeError(name)

        def call(*args):
            if name == "set_lowrank":
                self._lowrank = args[0]
        return call

    def refresh_data(self):
        pass

    def close(self):
        pass


@pytest.fixture
def real_cache(monkeypatch):
    """The real plan cache over CPU tensors, with a fake Plan and stream."""
    class _Stream:
        cuda_stream = 0

    monkeypatch.setattr(operators, "Plan", _FakePlan)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
    monkeypatch.setattr(operators, "_get_plan", operators._get_plan_locked)
    operators.clear_plan_cache()
    yield
    operators.clear_plan_cache()


def test_freed_hadamard_plan_never_serves_an_additive_operator(real_cache):
    x, y = torch.rand(6, 2), torch.rand(6, 2)
    one = torch.tensor(1.0)
    had = operators.HadamardKernelLinearOperator(x, None, "rbf", one, one, torch.zeros(6, dtype=torch.long), None, torch.eye(2))
    had.plan()
    task_plan = had._plan
    del had                          # the plan is free to be re-pointed within its slot
    add = operators.AdditiveKernelLinearOperator([operators.KernelLinearOperator(y[:, i:i + 1], None, "rbf", one, one)
                                                  for i in range(2)])
    assert add.x1.shape == x.shape
    add.plan()
    assert add._plan is not task_plan and getattr(add._plan, "_task_src", None) is None


def test_fourth_product_factor_and_low_rank_base_get_different_plans(real_cache):
    x, one = torch.rand(6, 2), torch.tensor(1.0)
    prod = operators.ProductKernelLinearOperator([operators.KernelLinearOperator(x, None, "rbf", one, one) for _ in range(4)])
    lr = operators.LowRankUpdatedKernelLinearOperator(operators.KernelLinearOperator(x, None, "rbf", one, one), torch.ones(6, 2))
    lr.plan()
    prod.ops[3].plan()
    assert prod.ops[3]._plan is not lr.base._plan and getattr(prod.ops[3]._plan, "_lowrank", None) is None


# ---- nested ScaleKernels -------------------------------------------------------------------------------------------------------
SCALED = {
    "plain": (kernels.RBFKernel, 2),
    "deriv": (kernels.RBFKernelGrad, 2),
    "ski": (lambda: kernels.GridInterpolationKernel(kernels.RBFKernel(), grid_size=16, num_dims=1), 1),
    "rq": (kernels.RQKernel, 2),
    "poly": (lambda: kernels.PolynomialKernel(power=2), 2),
    "periodic": (kernels.PeriodicKernel, 2),
    "ppoly": (lambda: kernels.PiecewisePolynomialKernel(q=2), 2),
}


@pytest.mark.parametrize("name", list(SCALED))
def test_nested_scale_kernels_multiply(name):
    make, d = SCALED[name]
    x = torch.rand(8, d)
    inner = kernels.ScaleKernel(make())
    inner.outputscale = 3.0
    outer = kernels.ScaleKernel(inner)
    outer.outputscale = 2.0
    op = outer(x)
    assert abs(float(op.outputscale.detach()) - 6.0) < 1e-5
    # one ScaleKernel around an unscaled kernel: its scale is the operator's outputscale as is, no product is formed
    op = inner(x)
    assert abs(float(op.outputscale.detach()) - 3.0) < 1e-5 and "Mul" not in type(op.outputscale.grad_fn).__name__
