"""Which plan settings every call and role refuses, on the device (run with -m gpu).

For each case (a call, or a role such as the data plan of gp_plan_set_kron) and each base plan (one per setting, plus plain, SKI
and kernel-sum plans, each with and without a low-rank correction where that is allowed) a fresh plan is built at n = 64, d = 2
and the case's C function is called with valid arguments.  Where plan_settings_oracle.py says the pair is refused, the status is
GP_E_STATE and the message names the call, the setting and its setter; everywhere else the call does not fail with such a
refusal."""
import ctypes as C
import threading

import pytest
import torch

import plan_settings_oracle as ps

pytestmark = pytest.mark.gpu

N, D = 64, 2
BIG = 192 * 192   # floats of every scratch buffer: a derivative plan has N (d + 1) = 192 rows


def _f(*v):
    return (C.c_float * len(v))(*v)


class World:
    """Device inputs, scratch buffers and every plan of one case; the plans are destroyed by close()."""

    def __init__(self, lib, dev):
        self.lib, self.dev, self.plans = lib, dev, []
        g = torch.Generator().manual_seed(0)
        self.x = torch.rand(N, D, generator=g).to(dev)
        self.U = (0.01 * torch.rand(N, 2, generator=g)).to(dev)
        self.ids = (torch.arange(192, dtype=torch.int32) % 2).to(dev)
        self.buf = [torch.zeros(BIG, device=dev) for _ in range(8)]
        self.piv = torch.zeros(16, dtype=torch.int64, device=dev)

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def new(self):
        h = C.c_void_p()
        assert self.lib.gp_plan_create(C.byref(h), self.dev.index or 0, C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)) == 0
        self.plans.append(h)
        return h

    def ok(self, st):
        assert st == 0, self.lib.gp_last_error().decode()

    def data(self, h):
        self.ok(self.lib.gp_plan_set_data(h, self.ptr(self.x), N, D, None, N, D, D, 0, 0))
        return h

    def hypers(self, h, kind=0, n_ls=1):
        self.ok(self.lib.gp_plan_set_hypers(h, kind, _f(*[1.0] * n_ls), n_ls, 1.0, 0.1))
        return h

    def plain(self, kind=0):
        return self.hypers(self.data(self.new()), kind)

    def close(self):
        torch.cuda.synchronize(self.dev)
        for h in reversed(self.plans):
            self.lib.gp_plan_destroy(h)


# ---- base plans: the settings each carries, and how to build it --------------------------------------------------------------
def _sum(w):
    p = w.data(w.new())
    terms = (C.c_void_p * 2)(w.plain(), w.plain(2))
    w.ok(w.lib.gp_plan_set_sum(p, terms, 2))
    return w.hypers(p)


def _product(w):
    p = w.plain()
    w.ok(w.lib.gp_plan_set_product(p, (C.c_void_p * 2)(w.plain(), w.plain(2)), 2))
    return p


def _kron(w):
    p = w.new()
    w.ok(w.lib.gp_plan_set_kron(p, w.plain(), 2))
    w.ok(w.lib.gp_plan_set_task_covar(p, _f(1.0, 0.5, 0.5, 1.0), 2))
    return w.hypers(p)


def _deriv(w):
    p = w.new()
    w.ok(w.lib.gp_plan_set_deriv(p, w.plain()))
    return w.hypers(p)


def _tasks(w):
    p = w.plain()
    w.ok(w.lib.gp_plan_set_tasks(p, w.ptr(w.ids), None, 2))
    w.ok(w.lib.gp_plan_set_task_covar(p, _f(1.0, 0.5, 0.5, 1.0), 2))
    return p


def _additive(w):
    p = w.hypers(w.data(w.new()), 0, D)
    w.ok(w.lib.gp_plan_set_additive(p, 1, _f(1.0, 1.0), D))
    return p


def _spectral(w):
    p = w.plain()
    w.ok(w.lib.gp_plan_set_spectral(p, 1, _f(1.0), _f(0.3, 0.2), _f(0.5, 0.4), D))
    return p


def _periodic(w):
    p = w.plain()
    w.ok(w.lib.gp_plan_set_periodic(p, _f(1.0), 1, D))
    return p


def _rq(w):
    p = w.data(w.new())
    w.ok(w.lib.gp_plan_set_hypers_rq(p, _f(1.0), 1, 1.5, 1.0, 0.1))
    return p


def _poly(w):
    p = w.data(w.new())
    w.ok(w.lib.gp_plan_set_hypers_poly(p, 2, 0.5, 1.0, 0.1))
    return p


def _ski(w):
    p = w.data(w.new())
    w.ok(w.lib.gp_plan_set_ski(p, (C.c_int * 2)(10, 10), _f(-0.4, -0.4), _f(0.2, 0.2), D))
    return w.hypers(p)


def _lowrank(make):
    def build(w):
        p = make(w)
        w.ok(w.lib.gp_plan_set_lowrank(p, w.ptr(w.U), 2, 2))
        return p
    return build


_CORE = {"plain": ((), lambda w: w.plain()), "ski": ((), _ski), "sum": ((), _sum), "tasks": (("tasks",), _tasks),
         "kron": (("kron",), _kron), "deriv": (("deriv",), _deriv), "product": (("product",), _product),
         "additive": (("additive",), _additive), "spectral": (("spectral",), _spectral), "periodic": (("periodic",), _periodic),
         "rq": (("rq",), _rq), "poly": (("poly",), _poly)}
BASES = dict(_CORE)
for _k in ("plain", "ski", "sum", "additive", "spectral", "periodic", "rq", "poly"):
    BASES[_k + "+lowrank"] = (_CORE[_k][0] + ("lowrank",), _lowrank(_CORE[_k][1]))


# ---- cases: (rows checked, in the order the call checks them) and the call on a base plan ---------------------------------------
def _calls():
    def b(w, i):
        return w.ptr(w.buf[i])

    def dbl(n=64):
        return (C.c_double * n)()

    it, ts, rk = C.c_int(), C.c_int(), C.c_int()
    res = (C.c_float * 64)()
    L = lambda w: w.lib   # noqa: E731
    return {
        "set_backend": lambda w, p: L(w).gp_plan_set_backend(p, 2),
        "set_hypers_rq": lambda w, p: L(w).gp_plan_set_hypers_rq(p, _f(1.0), 1, 1.5, 1.0, 0.1),
        "set_hypers_poly": lambda w, p: L(w).gp_plan_set_hypers_poly(p, 2, 0.5, 1.0, 0.1),
        "set_ski": lambda w, p: L(w).gp_plan_set_ski(p, (C.c_int * 2)(10, 10), _f(-0.4, -0.4), _f(0.2, 0.2), D),
        "ski_input_grad": lambda w, p: L(w).gp_ski_input_grad(p, b(w, 0), 16, b(w, 1), 16, 1, b(w, 2), 16),
        "set_tasks": lambda w, p: L(w).gp_plan_set_tasks(p, w.ptr(w.ids), None, 2),
        "set_additive": lambda w, p: L(w).gp_plan_set_additive(p, 1, _f(1.0, 1.0), D),
        "set_spectral": lambda w, p: L(w).gp_plan_set_spectral(p, 1, _f(1.0), _f(0.3, 0.2), _f(0.5, 0.4), D),
        "set_periodic": lambda w, p: L(w).gp_plan_set_periodic(p, _f(1.0), 1, D),
        "set_sum": lambda w, p: L(w).gp_plan_set_sum(p, (C.c_void_p * 2)(w.plain(), w.plain(2)), 2),
        "set_product": lambda w, p: L(w).gp_plan_set_product(p, (C.c_void_p * 2)(w.plain(), w.plain(2)), 2),
        "set_kron": lambda w, p: L(w).gp_plan_set_kron(p, w.plain(), 2),
        "set_deriv": lambda w, p: L(w).gp_plan_set_deriv(p, w.plain()),
        "set_deriv_kind": lambda w, p: L(w).gp_plan_set_deriv_kind(p, w.plain(3), 3),
        "set_lowrank": lambda w, p: L(w).gp_plan_set_lowrank(p, w.ptr(w.U), 2, 2),
        "kmv_input_grad": lambda w, p: L(w).gp_kmv_input_grad(p, b(w, 0), 16, b(w, 1), 16, 1, b(w, 2), 16, None, 0),
        "kdense_input_grad": lambda w, p: L(w).gp_kdense_input_grad(p, b(w, 0), 192, b(w, 2), 16, None, 0),
        "pivoted_cholesky": lambda w, p: L(w).gp_pivoted_cholesky(p, 4, 0.0, b(w, 3), w.ptr(w.piv), C.byref(rk)),
        "precond_build": lambda w, p: L(w).gp_precond_build(p, b(w, 3), 4, b(w, 4), dbl()),
        "ciq_precond_build": lambda w, p: L(w).gp_ciq_precond_build(p, b(w, 3), 4, b(w, 4), dbl()),
        "precond_probes": lambda w, p: L(w).gp_precond_probes(p, b(w, 3), 4, b(w, 0), b(w, 1), 1, b(w, 2)),
        "bilinear_grad": lambda w, p: L(w).gp_bilinear_grad(p, b(w, 0), 16, b(w, 1), 16, 1, dbl(), dbl(1)),
        "mbcg_precond": lambda w, p: L(w).gp_mbcg(p, b(w, 0), 16, 1, 0, 1.0, 10, 10, b(w, 4), 4, b(w, 2), 16, b(w, 5),
                                                  C.byref(it), C.byref(ts), res),
        "ciq_sqrt_matmul_precond": lambda w, p: L(w).gp_ciq_sqrt_matmul_precond(p, b(w, 0), 16, 1, b(w, 4), 4, (C.c_double * 1)(0.5),
                                                                                (C.c_double * 1)(1.0), 1, 1e-3, 10, b(w, 2), 16,
                                                                                C.byref(it), res),
        # roles at set time: the base is the plan taken in
        "kron_data": lambda w, p: L(w).gp_plan_set_kron(w.new(), p, 2),
        "deriv_data": lambda w, p: L(w).gp_plan_set_deriv(w.new(), p),
        "deriv_kind_data": lambda w, p: L(w).gp_plan_set_deriv_kind(w.new(), p, 3),
        "product_factor": lambda w, p: L(w).gp_plan_set_product(w.plain(), (C.c_void_p * 2)(p, w.plain()), 2),
        "sum_term": lambda w, p: L(w).gp_plan_set_sum(w.plain(), (C.c_void_p * 2)(p, w.plain()), 2),
    }


# A case is the rows its call checks, in order, with the checks between them that answer first for some bases: a set of base kinds
# (the base's name without "+lowrank") for which an earlier check of another kind (SKI, kernel sum, plain plan, kernel kind) fails.
_NOT_PLAIN = {"ski", "sum", "kron", "deriv", "product"}
_ALL_KINDS = set(_CORE)
CALL_CASES = {r: (r,) for r in _calls() if r in ps.ROW}
CALL_CASES.update({
    "set_kron": ({"ski", "sum"}, "set_kron"), "set_deriv": ({"ski", "sum"}, "set_deriv"),
    "set_deriv_kind": ({"ski", "sum"}, "set_deriv_kind"), "set_product": ({"ski", "sum"}, "set_product"),
    "set_tasks": ("set_tasks", {"ski", "sum"}, "set_tasks_lowrank"),
    "ski_input_grad": (_ALL_KINDS - {"ski"}, "ski_input_grad"),
    "kron_data": ("kron_data", _NOT_PLAIN, "kron_data_refresh"),
    "deriv_data": ("deriv_data", _NOT_PLAIN, "deriv_data_refresh"),
    "deriv_kind_data": ("deriv_kind_data", _ALL_KINDS, "deriv_data_refresh"),   # every base: not a Matern-5/2 plan
    "product_factor": ("product_factor", _NOT_PLAIN, "product_factor_refresh"),
    "sum_term": ("sum_term", _NOT_PLAIN, "sum_term_refresh"),
})


def _expected(steps, settings, kind):
    """The (row, setting) that refuses a base of `kind` carrying `settings`, or None."""
    for step in steps:
        if isinstance(step, set):
            if kind in step:
                return None
        elif ps.refused(step, settings):
            return step, ps.refused(step, settings)
    return None


def _check(lib, st, steps, settings, kind, what):
    msg = lib.gp_last_error().decode() if st else ""
    rows = [s for s in steps if not isinstance(s, set)]
    exp = _expected(steps, settings, kind)
    if exp:
        row, s = exp
        assert st == ps.GP_E_STATE, (what, st, msg)
        text = ps.message(row, s)
        assert text in msg or ps.REWORDED.get((row, s), text) in msg, (what, msg)
        if text in msg:
            assert ps.ROW[row][1] in msg and ps.NOUN[s] in msg and ps.SETTER[s] in msg
    else:
        for r in rows:
            for k in ps.KEYS:
                assert ps.message(r, k) not in msg and ps.REWORDED.get((r, k), "\0") not in msg, (what, msg)


@pytest.mark.parametrize("case", sorted(CALL_CASES))
def test_call_refuses_exactly_its_settings(cuda_dev, case):
    from gpytorch_b200 import _lib

    lib = _lib.load()
    call = _calls()[case]
    for base, (settings, make) in BASES.items():
        w = World(lib, cuda_dev)
        try:
            p = make(w)
            _check(lib, call(w, p), CALL_CASES[case], settings, base.split("+")[0], (case, base))
        finally:
            w.close()


# ---- roles at refresh time: a setting given to a factor, term or data plan after it was taken in -------------------------------
def _attach(w, role):
    q = w.plain()
    if role == "kron":
        p = w.new()
        w.ok(w.lib.gp_plan_set_kron(p, q, 2))
        w.ok(w.lib.gp_plan_set_task_covar(p, _f(1.0, 0.5, 0.5, 1.0), 2))
        return w.hypers(p), q, ("kron_data_refresh",)
    if role == "deriv":
        p = w.new()
        w.ok(w.lib.gp_plan_set_deriv(p, q))
        return w.hypers(p), q, ("deriv_data_refresh",)
    p = w.plain()
    if role == "product":
        w.ok(w.lib.gp_plan_set_product(p, (C.c_void_p * 2)(q, w.plain()), 2))
        return p, q, ("product_factor_refresh",)
    w.ok(w.lib.gp_plan_set_sum(p, (C.c_void_p * 2)(q, w.plain()), 2))
    return p, q, ("sum_term_refresh",)


# a low-rank correction given to a factor and task indices given to a term are not re-checked: neither re-packs the taking plan
_NOT_RECHECKED = {("product", "lowrank"), ("sum", "tasks")}


_LATE = {"rq": lambda w, q: w.lib.gp_plan_set_hypers_rq(q, _f(1.0), 1, 1.5, 1.0, 0.1),
         "poly": lambda w, q: w.lib.gp_plan_set_hypers_poly(q, 2, 0.5, 1.0, 0.1),
         "tasks": lambda w, q: w.lib.gp_plan_set_tasks(q, w.ptr(w.ids), None, 2),
         "lowrank": lambda w, q: w.lib.gp_plan_set_lowrank(q, w.ptr(w.U), 2, 2)}


@pytest.mark.parametrize("role", ["kron", "deriv", "product", "sum"])
@pytest.mark.parametrize("late", sorted(_LATE))
def test_role_refuses_a_setting_given_after_attach(cuda_dev, role, late):
    from gpytorch_b200 import _lib

    lib = _lib.load()
    w = World(lib, cuda_dev)
    try:
        p, q, rows = _attach(w, role)
        if (role, late) in _NOT_RECHECKED:
            rows = ()
        w.ok(_LATE[late](w, q))
        if late == "tasks":
            w.ok(lib.gp_plan_set_task_covar(q, _f(1.0, 0.5, 0.5, 1.0), 2))
        st = lib.gp_kmv(p, w.ptr(w.buf[0]), 16, 1, w.ptr(w.buf[1]), 16, 0)
        _check(lib, st, rows, (late,), "plain", (role, late))
    finally:
        w.close()


def test_comm_with_more_than_one_rank_refuses_its_settings(cuda_dev):
    """gp_plan_set_comm refuses only with a communicator of world > 1, which needs two devices."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from gpytorch_b200 import _lib

    lib = _lib.load()
    uid = (C.c_uint8 * 128)()
    assert lib.gp_comm_unique_id(uid) == 0
    comms = [C.c_void_p(), C.c_void_p()]

    def init(r):
        torch.cuda.set_device(r)
        assert lib.gp_comm_init(C.byref(comms[r]), uid, r, 2) == 0

    th = [threading.Thread(target=init, args=(r,)) for r in (0, 1)]
    [t.start() for t in th]
    [t.join() for t in th]
    torch.cuda.set_device(0)
    try:
        for base, (settings, make) in BASES.items():
            w = World(lib, cuda_dev)
            try:
                p = make(w)
                _check(lib, lib.gp_plan_set_comm(p, comms[0]), ("set_comm",), settings, base.split("+")[0], ("set_comm", base))
                lib.gp_plan_set_comm(p, None)
            finally:
                w.close()
    finally:
        for c in comms:
            if c:
                lib.gp_comm_destroy(c)
