"""Engine-backed covariance operators: the LinearOperator duck-type subset the exact-GP path calls.

Mirrors (reference paths under /root/reference/gpytorch):
  * KernelLinearOperator returned by a kernel's forward, the KeOps plug-in pattern
    (kernels/keops/rbf_kernel.py:44-55, keops/matern_kernel.py:68-80) -- `evaluate_kernel()` hands the
    operator itself to the solver (lazy/lazy_evaluated_kernel_tensor.py:345-373);
  * LazyEvaluatedKernelTensor hooks: _matmul (:245-276), _getitem (:136-243), _diagonal (:107-133),
    _size (:277-318), _bilinear_derivative (:69-105);
  * AddedDiagLinearOperator / InvQuadLogdet / solve of linear_operator (SURVEY.md Appendix A.4-A.5),
    reached from distributions/multivariate_normal.py:248-249 and
    models/exact_prediction_strategies.py:286,444.

All arithmetic runs in libgpbbmm (CUDA); torch supplies memory, streams and the autograd graph.
"""
from __future__ import annotations

import collections
import weakref

import torch

from . import settings
from ._lib import NanError
from .engine import DerivPlan, KronPlan, LcmPlan, Plan
from .sampling import contour_quadrature, psd_safe_cholesky


def _as_list(ls: torch.Tensor):
    return [float(v) for v in ls.detach().reshape(-1).tolist()]


# Plans own device workspaces (packed tiles, CG vectors); re-use them across operators over the same buffers so a
# training loop does not re-allocate every step.  Hyper-parameters / data are re-packed whenever a new operator
# first touches a cached plan.
_PLAN_CACHE: "dict[tuple, Plan]" = {}
_PLAN_CACHE_MAX = 64          # a batch of 16 independent operators (+ their cross-covariances) must fit
_PLAN_LOCK = __import__("threading").RLock()   # BatchLinearOperator drives the cache from worker threads

_SLOT_ROLES = ("own", "lowrank", "sum_term", "product_factor", "data", "lcm_term")
# RQ and polynomial operators run on the plain kernels: they share the plain slots, and their kind and parameters are part of the
# plan's hyper-parameter key, so a plan re-sends them whenever another kind used it last
_SLOT_FAMILY = {"rq": "plain", "poly": "plain"}


def _slot(family, role, index=0):
    """The plan-cache slot of an operator of `family` in `role` (the index-th sum term, product factor or LCM term): operators
    over the same inputs get one plan per slot, and a plan is only ever re-pointed within its slot, so two families (or roles)
    never see each other's engine settings."""
    if role not in _SLOT_ROLES:
        raise ValueError(f"unknown plan-cache role {role!r}")
    return (_SLOT_FAMILY.get(family, family), role, int(index))


# Parent plans of the operators built on other plans (sum, product, Kronecker, LCM, derivative), one dict per family, each the
# 16 most recently used
_SUM_PLANS: "dict[tuple, Plan]" = {}
_PRODUCT_PLANS: "dict[tuple, Plan]" = {}
_KRON_PLANS: "dict[tuple, Plan]" = {}
_LCM_PLANS: "dict[tuple, Plan]" = {}
_DERIV_PLANS: "dict[tuple, Plan]" = {}
_PARENT_PLANS = (_SUM_PLANS, _PRODUCT_PLANS, _KRON_PLANS, _LCM_PLANS, _DERIV_PLANS)


def _parent_plan(plans, key, make, x1=None, x2=None):
    """The parent plan of `key` in `plans` (most recently used last, at most 16), make() on a miss.  With x1 (and x2 for a cross
    operator), a parent whose inputs differ follows its child plans, which the cache re-pointed to new inputs (_get_plan_locked)."""
    with _PLAN_LOCK:
        parent = plans.pop(key, None)
        if parent is None:
            parent = make()
            parent._hyp_key = None
        elif x1 is not None and parent.x1.data_ptr() != x1.data_ptr():
            parent.x1 = x1.contiguous()
            parent.x2 = parent.x1 if x2 is None else x2.contiguous()
            parent.refresh_data()
        plans[key] = parent
        while len(plans) > 16:
            plans.pop(next(iter(plans))).close()
    return parent


def _get_plan(x1, x2, backend, row_begin, row_count, comm, slot=0, owner=None) -> Plan:
    if not x1.is_cuda:
        raise RuntimeError("x1 must live on a CUDA device: gpytorch_b200 has no CPU path")
    with _PLAN_LOCK:
        return _get_plan_locked(x1, x2, backend, row_begin, row_count, comm, slot, owner)


def _get_plan_locked(x1, x2, backend, row_begin, row_count, comm, slot=0, owner=None) -> Plan:
    # a plan enqueues on the stream that was current when it was created: the stream is part of the identity; so is the slot:
    # the terms of a kernel sum over the SAME inputs need one plan each (each holds its own packed lengthscales)
    role = (tuple(x1.shape), x1.stride(0), None if x2 is None else (tuple(x2.shape), x2.stride(0)), backend, str(x1.device),
            row_begin, row_count, id(comm), torch.cuda.current_stream(x1.device).cuda_stream, slot)
    key = (x1.data_ptr(), None if x2 is None else x2.data_ptr(), role)
    plan = _PLAN_CACHE.pop(key, None)
    src_versions = (x1._version, None if x2 is None else x2._version)
    if plan is None:
        # New buffers in a known role: deep kernel learning computes new features every step, and the plan holds the old ones, so
        # their address never comes back.  Re-point a plan of the same role whose operators are all gone instead of growing a
        # new one (with its workspaces) per step; a plan that a live operator uses is never taken.
        for k, cand in _PLAN_CACHE.items():
            if k[2] == role and not cand._owners:
                plan = _PLAN_CACHE.pop(k)
                plan._src_versions = None
                break
    if plan is not None and plan._src_versions != src_versions:
        # same buffers, new contents (x.copy_(new), an optimiser step on the inputs, ...) or a re-pointed plan: the packed tiles
        # are stale.  torch bumps a tensor's version counter on every in-place write, so this is exact, not a heuristic.
        plan.x1 = x1.contiguous()
        plan.x2 = plan.x1 if x2 is None else x2.contiguous()
        plan.refresh_data()
    if plan is None:
        plan = Plan(x1, x2, backend="auto" if backend.startswith("ski:") else backend, row_begin=row_begin, row_count=row_count, comm=comm)
        plan._hyp_key = None
        plan._owners = weakref.WeakSet()
    if owner is not None:
        plan._owners.add(owner)
    plan._src_versions = src_versions
    _PLAN_CACHE[key] = plan  # most recently used last
    while len(_PLAN_CACHE) > _PLAN_CACHE_MAX:
        _PLAN_CACHE.pop(next(iter(_PLAN_CACHE))).close()
    return plan


def clear_plan_cache():
    with _PLAN_LOCK:
        for plans in _PARENT_PLANS:
            while plans:
                plans.popitem()[1].close()
        while _PLAN_CACHE:
            _PLAN_CACHE.popitem()[1].close()
        _ADDITIVE_X.clear()


class ConstantDiagLinearOperator:
    """sigma^2 I (likelihoods/noise_models.py:57-92 returns this for homoskedastic noise)."""

    def __init__(self, diag_value: torch.Tensor, diag_shape: int):
        self.diag_value = diag_value
        self.n = int(diag_shape)

    def __add__(self, other):
        if isinstance(other, ConstantDiagLinearOperator):
            return ConstantDiagLinearOperator(self.diag_value + other.diag_value, self.n)
        if isinstance(other, DiagLinearOperator):
            return other + self
        return NotImplemented

    @property
    def shape(self):
        return torch.Size([self.n, self.n])

    def to_dense(self):
        return self.diag_value.reshape(()) * torch.eye(self.n, device=self.diag_value.device, dtype=self.diag_value.dtype)


class DiagLinearOperator:
    """diag(d) with a per-row vector d (FixedGaussianNoise, likelihoods/noise_models.py:150-190)."""

    def __init__(self, diag: torch.Tensor):
        self.diag_vec = diag
        self.n = int(diag.shape[-1])

    @property
    def shape(self):
        return torch.Size([self.n, self.n])

    def to_dense(self):
        return torch.diag_embed(self.diag_vec)

    def __add__(self, other):
        if isinstance(other, ConstantDiagLinearOperator):
            return DiagLinearOperator(self.diag_vec + other.diag_value.reshape(-1)[:1])
        if isinstance(other, DiagLinearOperator):
            return DiagLinearOperator(self.diag_vec + other.diag_vec)
        return NotImplemented


class RootLinearOperator:
    """R R^T held as its dense root R [..., n, r] (what root_decomposition returns; `.root` as in linear_operator)."""

    def __init__(self, root: torch.Tensor):
        self.root = root

    @property
    def shape(self):
        return torch.Size([*self.root.shape[:-1], self.root.shape[-2]])

    def matmul(self, rhs):
        return self.root @ (self.root.transpose(-1, -2) @ rhs)

    __matmul__ = matmul

    def to_dense(self):
        return self.root @ self.root.transpose(-1, -2)


class _SamplingMixin:
    """zero_mean_mvn_samples / root_decomposition of an engine operator K_hat (the kernel alone, or kernel + noise).

    Three paths, as the reference picks them (linear_operator LinearOperator.zero_mean_mvn_samples / root_decomposition):
      * settings.ciq_samples on: K_hat^{1/2} xi by contour integral quadrature, the shifted solves by multi-shift MINRES on the
        device (csrc/minres.cu), xi ~ N(0, I) from torch's global generator, 16 columns per engine call;
      * n <= max_cholesky_size or fast_computations(covar_root_decomposition=False): a dense psd-safe Cholesky root;
      * otherwise a Lanczos root R = Q V Lambda^{1/2} of rank <= max_root_decomposition_size (negative Ritz values masked).
    Samples of these paths are detached from the hyper-parameters: their gradients are not implemented."""

    def _sampling_plan(self) -> Plan:
        raise NotImplementedError

    def _noise_floor(self):
        """A proven lower bound of the spectrum of K_hat from its noise (None without noise)."""
        return None

    def _ciq_bounds(self, plan: Plan, start: torch.Tensor):
        """(m, M) for the quadrature: M from the largest Ritz value of 20 Lanczos steps (raised by 1%: a Ritz value is a lower
        bound of the largest eigenvalue), m the noise floor, else the smallest Ritz value."""
        n = self.shape[0]
        if not bool(torch.isfinite(start).all()) or float(start.abs().max()) == 0.0:
            start = torch.ones(n, device=self.device)
        _, t = plan.lanczos(start.float().contiguous(), min(20, n))
        t = t.double().cpu()
        if not bool(torch.isfinite(t).all()):
            raise NanError("NaNs encountered when trying to perform matrix-vector multiplication")
        ritz = torch.linalg.eigvalsh(t)
        M = 1.01 * float(ritz.max())
        floor = self._noise_floor()
        if floor is not None and floor > 0.0:
            m = floor
        else:
            m = float(ritz.min())
            if m <= 0.0:
                m = 1e-6 * M
        return m, max(M, m)

    def _ciq_precond(self):
        """(U [n, k], m, M) of the split preconditioner F (csrc/minres.cu header) when settings.ciq_preconditioner applies, else None."""
        return None

    def _ciq_samples(self, xi: torch.Tensor):
        """K_hat^{1/2} xi for xi [n, s] (F A^{1/2} xi with settings.ciq_preconditioner); returns ([n, s], list of CiqInfo)."""
        plan = self._sampling_plan()
        pre = self._ciq_precond() if settings.ciq_preconditioner.on() else None
        if pre is None:
            u = None
            m, M = self._ciq_bounds(plan, xi[:, 0])
        else:
            u, m, M = pre
        tau, w = contour_quadrature(m, M, settings.num_contour_quadrature.value())
        outs, infos = [], []
        for c0 in range(0, xi.size(1), 16):
            o, info = plan.ciq_sqrt_matmul(xi[:, c0:c0 + 16].contiguous(), tau, w, settings.minres_tolerance.value(),
                                           settings.max_cg_iterations.value(), precond_u=u)
            outs.append(o)
            infos.append(info)
        self.last_ciq = (m, M, infos)
        return (outs[0] if len(outs) == 1 else torch.cat(outs, -1)), infos

    def zero_mean_mvn_samples(self, num_samples: int) -> torch.Tensor:
        """[num_samples, n] draws from N(0, K_hat)."""
        n = self.shape[0]
        if settings.ciq_samples.on():
            xi = torch.randn(n, num_samples, device=self.device)
            return self._ciq_samples(xi)[0].t()
        root = self.root_decomposition().root
        eps = torch.randn(root.size(-1), num_samples, device=root.device, dtype=root.dtype)
        return (root @ eps).t()

    def root_decomposition(self, method=None) -> RootLinearOperator:
        """R with R R^T ~= K_hat: "cholesky" (dense, psd-safe) or "lanczos"; None picks as zero_mean_mvn_samples does."""
        if method not in (None, "cholesky", "lanczos"):
            raise RuntimeError(f"root_decomposition: unknown method {method!r} (the engine offers 'cholesky' and 'lanczos')")
        n = self.shape[0]
        if method == "cholesky" or (method is None and _dense_branch(n, settings.fast_computations.covar_root_decomposition)):
            return RootLinearOperator(psd_safe_cholesky(self.to_dense().detach().float()))
        return RootLinearOperator(self._lanczos_root())

    def _lanczos_root(self, init=None) -> torch.Tensor:
        p = self._sampling_plan()
        init = init if init is not None else torch.randn(self.shape[0], device=self.device)
        q, t = p.lanczos(init.float().contiguous(), settings.max_root_decomposition_size.value())
        evals, evecs = torch.linalg.eigh(t.double())
        mask = evals >= 0                                 # lanczos_tridiag_to_diag masks negative Ritz values
        evecs = evecs * mask
        evals = evals.masked_fill(~mask, 0.0)
        return (q.double() @ (evecs * evals.sqrt())).float()


def _a(noun):
    return ("an " if noun[0] in "aeiou" else "a ") + noun


class KernelLinearOperator(_SamplingMixin):
    """K(x1, x2) (outputscale folded in) that never materialises: every product is the fused CUDA kernel.

    This class is also the single-plan operator every kernel family (RQ, polynomial, periodic, piecewise polynomial, spectral
    mixture) derives from.  A family declares its parameters, its engine calls and what it may take part in; plan(), the host
    read of the hyper-parameters, their gradients and the re-wrapping methods are the ones below."""

    # -- what a family declares --
    _family = "plain"          # plan-cache family (_slot)
    _noun = "RBF / Matern"     # names the family in refusals
    _sum_term = True           # may be a term of a kernel sum
    _factor = True             # may be a kernel-product or an IndexKernel factor
    _input_grads = True        # gradients with respect to the inputs
    _row_sharding = True
    _single_plan = True        # one plan, re-wrapped by _with (composite and data-plan operators: False)
    _params = ("lengthscale",)     # the hyper-parameter tensors before the outputscale, in hyper_tensors() order
    _plan_backend = None           # None: settings.backend
    _resend_on_new_plan = True     # re-send every engine setting on a plan newly obtained from the cache
    _scaled = False                # per operator: it carries the outputscale of a ScaleKernel

    def __init__(self, x1, x2, kind, lengthscale, outputscale=None, plan: Plan | None = None, comm=None,
                 row_begin=0, row_count=0):
        if not self._row_sharding:
            if comm is not None or row_begin != 0 or row_count not in (0, x1.size(0)):
                raise NotImplementedError(f"a row-sharded {self._noun} operator is not available on the accelerated path")
            comm, row_begin, row_count = None, 0, 0
        self.x1, self.x2 = x1, x2
        self.kind = kind
        self.lengthscale = lengthscale          # tensor (scalar or [d]); may require grad
        self._scaled = outputscale is not None
        self.outputscale = outputscale if outputscale is not None else torch.ones((), device=x1.device)
        self._plan = plan
        self._plan_slot = _slot(self._family, "own")
        self._comm = comm
        self._row_begin, self._row_count = row_begin, row_count
        self.same = x2 is None or x2 is x1 or (x1.shape == x2.shape and x1.data_ptr() == x2.data_ptr())

    def _ctor_args(self):
        """The constructor arguments between (x1, x2) and the outputscale (_with rebuilds the operator from them)."""
        return (self.kind, self.lengthscale)

    def _engine_calls(self, hyp, nz):
        """[(plan attribute, key, send)] in call order: send(plan) is called when the plan's attribute differs from key.  hyp is
        the host values of _plan_hypers(), one list per tensor; nz the noise."""
        ls, (os_,) = hyp
        return [("_hyp_key", (self.kind, tuple(ls), os_, nz), lambda p: p.set_hypers(self.kind, ls, os_, nz))]

    # -- plumbing --
    @property
    def _scale_is_hyper(self):
        return True

    def _plan_hypers(self):
        """The tensors this operator's own plan is set from: _params, then the outputscale."""
        return [getattr(self, n) for n in self._params] + ([self.outputscale] if self._scale_is_hyper else [])

    def _host_hypers(self, noise_t=None):
        """([values of each _plan_hypers() tensor], noise, noise tensor) as host floats with ONE device->host read per operator
        (cached: the parameter tensors of an operator never change; a new forward builds a new operator)."""
        cached = getattr(self, "_hyp_host", None)
        if cached is None or (noise_t is not None and cached[2] is not noise_t):
            hyp = self._plan_hypers()
            parts = [t.detach().reshape(-1).float().to(self.device) for t in hyp]
            if noise_t is not None:
                parts.append(noise_t.detach().reshape(-1)[:1].float().to(self.device))
            vals = torch.cat(parts).tolist()
            out, k = [], 0
            for t in hyp:
                out.append(vals[k:k + t.numel()])
                k += t.numel()
            cached = (out, vals[k] if noise_t is not None else None, noise_t)
            self._hyp_host = cached
        return cached

    def plan(self, noise=0.0) -> Plan:
        """noise: a host float, or the device tensor of the likelihood (read together with the other hyper-parameters)."""
        fresh = self._plan is None
        if fresh:
            self._plan = _get_plan(self.x1, None if self.same else self.x2, self._plan_backend or settings.backend.value(),
                                   self._row_begin, self._row_count, self._comm, self._plan_slot, owner=self)
        hyp, nz, _ = self._host_hypers(noise if torch.is_tensor(noise) else None)
        if not torch.is_tensor(noise):
            nz = float(noise)
        p = self._plan
        for attr, key, send in self._engine_calls(hyp, nz):
            if (fresh and self._resend_on_new_plan) or getattr(p, attr, None) != key:
                send(p)
                setattr(p, attr, key)
        return p

    @property
    def shape(self):
        n2 = self.x1.size(0) if self.same else self.x2.size(0)
        return torch.Size([self.x1.size(0), n2])

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    @property
    def dtype(self):
        return self.x1.dtype

    @property
    def device(self):
        return self.x1.device

    @property
    def batch_shape(self):
        return torch.Size([])

    @property
    def requires_grad(self):
        return any(t.requires_grad for t in self._plan_hypers())

    def evaluate_kernel(self):
        return self  # "meta LinearOperator" branch, lazy_evaluated_kernel_tensor.py:345-348

    def representation(self):
        return (self.x1, self.x2, *self._plan_hypers())

    def hyper_tensors(self):
        """The differentiable hyper-parameters of this operator, in the order _bilinear_derivative_list returns their
        gradients (the autograd functions below take them as explicit inputs)."""
        return self._plan_hypers()

    def input_tensors(self):
        """The inputs K is differentiated in by the product and dense-block autograd functions below, which take them after
        the hyper-parameters: [x1] for a square operator (both arguments are the same points), [x1, x2] for a cross-covariance;
        none for a family without input gradients."""
        if not self._input_grads:
            return []
        return [self.x1] if self.same else [self.x1, self.x2]

    def solve_input_tensors(self):
        """The inputs _InvQuadLogdet and _Solve differentiate K in, after the hyper-parameters: input_tensors() for an exact
        operator or a kernel sum; a SKI operator adds its points there only (deep kernel learning trains through the MLL)."""
        return self.input_tensors()

    def _bilinear_derivative_list(self, left, right):
        """The gradients of sum(left * (K @ right)) with respect to hyper_tensors(): the engine's flat gradient split over the
        tensors before the outputscale, then the outputscale's."""
        gl, go = self.plan(getattr(self, "_last_noise", 0.0)).bilinear_grad(left, right)
        out, k = [], 0
        for t in self._plan_hypers()[:len(self._params)]:
            out.append(torch.tensor(gl[k:k + t.numel()], device=self.device, dtype=t.dtype).reshape(t.shape))
            k += t.numel()
        if self._scale_is_hyper:
            out.append(torch.tensor(go, device=self.device, dtype=self.outputscale.dtype).reshape(self.outputscale.shape))
        return out

    def _no_input_grads(self):
        return NotImplementedError(f"gradients with respect to the inputs of {_a(self._noun)} operator are not available on the "
                                   "accelerated path")

    def _input_grad_list(self, left, right, needs):
        """Gradients of sum(left * (K @ right)) w.r.t. input_tensors(), None where `needs` is False (gp_kmv_input_grad)."""
        if not any(needs):
            return [None] * len(needs)
        if not self._input_grads:
            raise self._no_input_grads()
        d1, d2 = self.plan(getattr(self, "_last_noise", 0.0)).kmv_input_grad(left, right, needs[0], len(needs) > 1 and needs[1])
        return [d1, d2][: len(needs)]

    def _dense_input_grad_list(self, w, needs):
        """Gradients of sum(w * K) w.r.t. input_tensors(), None where `needs` is False (gp_kdense_input_grad)."""
        if not any(needs):
            return [None] * len(needs)
        if not self._input_grads:
            raise self._no_input_grads()
        d1, d2 = self.plan().dense_input_grad(w, needs[0], len(needs) > 1 and needs[1])
        return [d1, d2][: len(needs)]

    # -- LinearOperator protocol: shape helpers / transpose (lazy_evaluated_kernel_tensor.py:277-341) --
    def _size(self):
        return self.shape

    @property
    def matrix_shape(self):
        return self.shape

    def dim(self):
        return 2

    ndimension = dim

    def numel(self):
        return self.shape[0] * self.shape[1]

    def _with(self, x1, x2, detach=False, outputscale=None):
        """This operator over new inputs (detached, or with the outputscale replaced), rebuilt through its constructor: the
        new operator has its own plan and no row sharding."""
        if not self._single_plan:
            raise NotImplementedError(f"{type(self).__name__} is not rebuilt from its inputs and parameters on the accelerated path")
        f = (lambda t: t.detach() if torch.is_tensor(t) else t) if detach else (lambda t: t)
        if outputscale is None and self._scaled:
            outputscale = self.outputscale
        return type(self)(f(x1), None if x2 is None else f(x2), *map(f, self._ctor_args()),
                          None if outputscale is None else f(outputscale))

    def with_outputscale(self, outputscale):
        """This operator with its outputscale replaced (a ScaleKernel folded in); its other parameters are kept."""
        return self._with(self.x1, None if self.same else self.x2, outputscale=outputscale)

    def _transpose_nonbatch(self):
        """K(x1, x2)^T = K(x2, x1) for every kernel on this path (no data is moved)."""
        return self if self.same else self._with(self.x2, self.x1)

    def transpose(self, dim1, dim2):
        return self if dim1 % 2 == dim2 % 2 else self._transpose_nonbatch()

    def t(self):
        return self._transpose_nonbatch()

    @property
    def mT(self):
        return self._transpose_nonbatch()

    def detach(self):
        return self._with(self.x1, None if self.same else self.x2, detach=True)

    # -- products --
    def matmul(self, rhs):
        return _KernelMatmul.apply(self, rhs, *self.hyper_tensors(), *self.input_tensors())

    __matmul__ = matmul
    _matmul = matmul

    def to_dense(self):
        return _KernelDense.apply(self, *self.input_tensors())

    def diagonal(self, dim1=-2, dim2=-1):
        """kernel(x1, x2, diag=True) (lazy_evaluated_kernel_tensor.py:107-133): the constant outputscale for x2 == x1,
        k(x1_i, x2_i) for a cross-covariance of equal sizes."""
        if not self.same and self.x1.size(0) != self.x2.size(0):
            raise RuntimeError(f"diagonal of a non-square operator {tuple(self.shape)} is undefined")
        return self.plan().diag()

    _diagonal = diagonal

    def _getitem(self, row_index, col_index, *batch_indices):
        return self[row_index, col_index]

    def __getitem__(self, index):
        """Row / column slicing by re-indexing x1 / x2 (lazy_evaluated_kernel_tensor.py:136-243)."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        return self._with(self.x1[ri], (self.x1 if self.same else self.x2)[ci])

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        if isinstance(other, KernelLinearOperator):
            return SumKernelLinearOperator([self, other])     # K_1 + K_2 stays lazy: one engine operator (csrc/sum.cu)
        raise NotImplementedError("a kernel operator adds a (Constant)DiagLinearOperator or another kernel operator")

    def add_jitter(self, jitter_val=1e-3):
        return AddedDiagLinearOperator(self, ConstantDiagLinearOperator(torch.tensor(jitter_val, device=self.device), self.shape[0]))

    def mul(self, other):
        """K o B[t, t'] with an IndexKernel's operator (the Hadamard multitask model, covar_x.mul(covar_i)): one engine operator
        (gp_plan_set_tasks).  RBF / Matern operators, optionally scaled, only.  With another RBF / Matern kernel operator (or a
        product of them) of the same shape: the elementwise product K_1 o K_2 as one engine operator (gp_plan_set_product)."""
        for o in (self, other):
            if isinstance(o, KernelLinearOperator) and not o._factor:
                raise o._no_product()
        if isinstance(other, KernelLinearOperator):
            return ProductKernelLinearOperator([self, other])
        if not isinstance(other, IndexLinearOperator) or type(self) is not KernelLinearOperator:
            raise NotImplementedError("the accelerated path multiplies an RBF / Matern kernel operator (optionally scaled) by an "
                                      "IndexKernel operator only")
        if tuple(other.shape) != tuple(self.shape):
            raise RuntimeError(f"mul: operator shapes {tuple(self.shape)} and {tuple(other.shape)} differ")
        return HadamardKernelLinearOperator(self.x1, None if self.same else self.x2, self.kind, self.lengthscale, self.outputscale,
                                            other.i1, other.i2, other.B)

    __mul__ = mul

    def _sampling_plan(self) -> Plan:
        """The plan of K alone: no noise, no per-row diagonal left over from an earlier K + D."""
        if not self.same:
            raise RuntimeError("sampling needs a square covariance operator (x2 == x1)")
        p = self.plan(0.0)
        if getattr(p, "_noise_diag", None) is not None:
            p.set_noise_diag(None)
        return p

    def _no_product(self):
        return NotImplementedError(f"products that contain {_a(self._noun)} operator (kernel products, IndexKernel multitask "
                                   "models) are not available on the accelerated path: it multiplies an RBF / Matern kernel operator "
                                   "(optionally scaled) by another one or by an IndexKernel operator only")

    def _bilinear_derivative(self, left, right):
        """(d/d lengthscale, d/d outputscale) of sum(left * (K @ right)); lazy_evaluated_kernel_tensor.py:69-105."""
        if self._params != ("lengthscale",) or not self._scale_is_hyper:
            names = ", ".join(self._params) + (" and outputscale" if self._scale_is_hyper else "")
            raise NotImplementedError(f"{_a(self._noun)} operator has {names} gradients: use _bilinear_derivative_list")
        gl, go = self.plan(getattr(self, "_last_noise", 0.0)).bilinear_grad(left, right)
        return torch.tensor(gl, device=self.device, dtype=self.dtype), torch.tensor(go, device=self.device, dtype=self.dtype)


class IndexLinearOperator:
    """B[i1, i2] of an IndexKernel (kernels/index_kernel.py:101-117 returns it as an InterpolatedLinearOperator): lazy, it only
    carries the task ids and B until a kernel operator multiplies it in (KernelLinearOperator.mul)."""

    def __init__(self, i1: torch.Tensor, i2: torch.Tensor, B: torch.Tensor):
        self.i1, self.i2, self.B = i1, i2, B

    @property
    def shape(self):
        return torch.Size([self.i1.numel(), self.i2.numel()])

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    @property
    def device(self):
        return self.B.device

    def to_dense(self):
        return self.B[self.i1][:, self.i2]

    def diagonal(self, dim1=-2, dim2=-1):
        return self.B[self.i1, self.i2]

    def mul(self, other):
        if isinstance(other, KernelLinearOperator):
            return other.mul(self)
        raise NotImplementedError("an IndexKernel operator multiplies an RBF / Matern kernel operator only")

    __mul__ = mul


class HadamardKernelLinearOperator(KernelLinearOperator):
    """s K(x1, x2) o B[t1, t2] (the Hadamard multitask model, examples/03_Multitask_Exact_GPs/Hadamard_Multitask_GP_Regression.ipynb):
    one engine operator whose plan carries the task ids (gp_plan_set_tasks) and B (gp_plan_set_task_covar).  The hyper-parameters
    are lengthscale, outputscale and B; B's gradient comes from gp_task_covar_grad and autograd carries it to the IndexKernel's
    covar_factor / raw_var.  Input gradients are not available: inputs that require grad are refused."""

    _family = "task"    # a plain operator over the same inputs never sees the task ids
    _noun = "Hadamard multitask"
    _sum_term = _factor = _single_plan = False

    def __init__(self, x1, x2, kind, lengthscale, outputscale, t1, t2, B):
        if x1.requires_grad or (x2 is not None and x2.requires_grad):
            raise RuntimeError("gradients with respect to the inputs of a Hadamard multitask operator (K o B) are not implemented: "
                               "pass inputs that do not require grad")
        super().__init__(x1, x2, kind, lengthscale, outputscale)
        self.t1 = t1.reshape(-1)
        if self.same and t2 is not None and t2 is not t1 and not torch.equal(t2.reshape(-1), self.t1):
            raise NotImplementedError("a square kernel operator takes one set of task ids (x2 == x1 needs t2 == t1)")
        self.t2 = self.t1 if self.same else t2.reshape(-1)
        if self.t1.numel() != self.shape[0] or self.t2.numel() != self.shape[1]:
            raise RuntimeError(f"task ids of sizes {self.t1.numel()}, {self.t2.numel()} do not match the operator {tuple(self.shape)}")
        self.B = B

    def plan(self, noise=0.0) -> Plan:
        p = super().plan(noise)
        T = int(self.B.shape[-1])
        src = getattr(p, "_task_src", None)
        # the plan keeps the id tensors it was given alive, so an identity + version match cannot be a recycled buffer
        if src is None or src[0] is not self.t1 or src[1] is not self.t2 or src[2] != (self.t1._version, self.t2._version) \
                or src[3] != T or getattr(p, "_tasks", None) is None:
            p.set_tasks(self.t1, None if self.same else self.t2, T)
            p._task_src = (self.t1, self.t2, (self.t1._version, self.t2._version), T)
            p._b_key = None
        bh = getattr(self, "_b_host", None)
        if bh is None:
            bh = self._b_host = self.B.detach().float().cpu()
        if getattr(p, "_b_key", None) is None or not torch.equal(p._b_key, bh):
            p.set_task_covar(bh)
            p._b_key = bh
        return p

    @property
    def requires_grad(self):
        return bool(super().requires_grad or self.B.requires_grad)

    def representation(self):
        return (self.x1, self.x2, self.lengthscale, self.outputscale, self.B)

    def hyper_tensors(self):
        return [self.lengthscale, self.outputscale, self.B]

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _bilinear_derivative_list(self, left, right):
        p = self.plan(getattr(self, "_last_noise", 0.0))
        gl, go = p.bilinear_grad(left, right)
        dB = p.task_covar_grad(left, right)
        return [torch.tensor(gl, device=self.device, dtype=self.dtype).reshape(self.lengthscale.shape),
                torch.tensor(go, device=self.device, dtype=self.dtype).reshape(self.outputscale.shape),
                dB.to(device=self.device, dtype=self.B.dtype)]

    def _bilinear_derivative(self, left, right):
        gl, go, _ = self._bilinear_derivative_list(left, right)
        return gl, go

    def _transpose_nonbatch(self):
        if self.same:
            return self
        return HadamardKernelLinearOperator(self.x2, self.x1, self.kind, self.lengthscale, self.outputscale, self.t2, self.t1,
                                            self.B.transpose(-1, -2))

    def detach(self):
        return HadamardKernelLinearOperator(self.x1.detach(), None if self.same else self.x2.detach(), self.kind,
                                            self.lengthscale.detach(), self.outputscale.detach(), self.t1,
                                            None if self.same else self.t2, self.B.detach())

    def to_dense(self):
        return _KernelDense.apply(self)

    def __getitem__(self, index):
        """Slices re-index the task ids together with x1 / x2 (prediction slices the joint operator)."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        x2 = self.x1 if self.same else self.x2
        return HadamardKernelLinearOperator(self.x1[ri], x2[ci], self.kind, self.lengthscale, self.outputscale, self.t1[ri],
                                            self.t2[ci], self.B)

    def mul(self, other):
        raise NotImplementedError("a Hadamard multitask operator takes one IndexKernel factor")

    __mul__ = mul

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("a Hadamard multitask operator adds a (Constant)DiagLinearOperator only")


def _aligned(ix, T: int, n: int):
    """The point slice of a row / column slice of a Kronecker operator that starts and stops on multiples of T (None otherwise)."""
    if not isinstance(ix, slice) or ix.step not in (None, 1):
        return None
    a, b, _ = ix.indices(n * T)
    if a % T or b % T or b < a:
        return None
    return slice(a // T, b // T)


class KroneckerKernelLinearOperator(KernelLinearOperator):
    """(s K(x1, x2)) (x) B over interleaved rows i T + a (MultitaskKernel, kernels/multitask_kernel.py:13-61; the reference returns
    KroneckerProductLinearOperator(covar_x, covar_i)): ONE engine operator (gp_plan_set_kron) on the plan of the data kernel.  The
    hyper-parameters are lengthscale, outputscale and B; B's gradient comes from gp_task_covar_grad and autograd carries it to the
    IndexKernel's covar_factor / raw_var.  Input gradients are not available: inputs that require grad are refused."""

    _family = "kron"
    _noun = "Kronecker multitask"
    _sum_term = _factor = _single_plan = False

    def __init__(self, x1, x2, kind, lengthscale, outputscale, B, rows=None, cols=None):
        if x1.requires_grad or (x2 is not None and x2.requires_grad):
            raise RuntimeError("gradients with respect to the inputs of a Kronecker multitask operator (K (x) B) are not implemented: "
                               "pass inputs that do not require grad")
        super().__init__(x1, x2, kind, lengthscale, outputscale)
        if B.dim() != 2 or B.shape[0] != B.shape[1] or not 1 <= B.shape[0] <= 32:
            raise RuntimeError(f"the task covariance must be [T, T] with 1 <= T <= 32 (got {tuple(B.shape)})")
        self.B = B
        self.num_tasks = int(B.shape[-1])
        self._data_op = KernelLinearOperator(x1, x2, kind, lengthscale, outputscale)
        self._data_op._plan_slot = _slot("kron", "data")
        # observed interleaved rows / columns (int64 index tensors, strictly increasing; None: all): the operator is
        # P_r ((s K) (x) B) P_c^T (masked())
        if self.same and cols is not None and cols is not rows and (rows is None or not torch.equal(rows, cols)):
            raise RuntimeError("a square Kronecker operator takes equal row and column masks")
        self.rows, self.cols = rows, (rows if self.same else cols)
        self._obs_host = None

    def masked(self, rows, cols):
        """P_r ((s K) (x) B) P_c^T: the interleaved rows `rows` and columns `cols` (int64 indices, strictly increasing; None: all)
        as one engine operator on the same data plan (gp_plan_set_kron_observed).  On a square operator the two must be equal."""
        if self.rows is not None or self.cols is not None:
            raise NotImplementedError("a masked Kronecker operator cannot be masked again")
        if self.same and rows is not None and cols is not None and rows is not cols and not torch.equal(rows, cols):
            raise NotImplementedError("a square Kronecker operator takes equal row and column masks")
        return KroneckerKernelLinearOperator(self.x1, None if self.same else self.x2, self.kind, self.lengthscale, self.outputscale,
                                             self.B, rows, cols)

    @property
    def shape(self):
        n2 = self.x1.size(0) if self.same else self.x2.size(0)
        T = self.num_tasks
        return torch.Size([self.x1.size(0) * T if self.rows is None else self.rows.numel(),
                           n2 * T if self.cols is None else self.cols.numel()])

    def _observed_host(self):
        """(rows, cols) on the host, read once per operator."""
        if self._obs_host is None:
            self._obs_host = tuple(None if v is None else v.detach().to(device="cpu", dtype=torch.int64) for v in (self.rows, self.cols))
        return self._obs_host

    def plan(self, noise=0.0) -> Plan:
        data = self._data_op.plan(0.0)
        if getattr(data, "_noise_diag", None) is not None:
            data.set_noise_diag(None)
        nz = float(noise.detach().reshape(-1)[0]) if torch.is_tensor(noise) else float(noise)
        T = self.num_tasks
        masked = self.rows is not None or self.cols is not None
        # a parent that holds a mask never serves an unmasked operator, nor the other way round; masked parents are re-masked
        # below only when the indices change
        parent = _parent_plan(_KRON_PLANS, (id(data), T, masked), lambda: KronPlan(data, T))
        # the data plan may have been re-packed or re-pointed since the last use: re-attach it (validation, no allocation)
        parent.attach(data, T)
        if masked:
            rh, ch = self._observed_host()
            ok = parent._observed is not None and getattr(parent, "_obs_key", None) is not None and all(
                (a is None and b is None) or (a is not None and b is not None and torch.equal(a, b)) for a, b in zip(parent._obs_key, (rh, ch)))
            if not ok:
                parent.set_observed(rh, ch)
                parent._obs_key = (rh, ch)
        hk = (nz, data.kind, tuple(data.lengthscale), data.outputscale)
        if parent._hyp_key != hk:
            parent.set_noise(nz)
            parent._hyp_key = hk
        bh = getattr(self, "_b_host", None)
        if bh is None:
            bh = self._b_host = self.B.detach().float().cpu()
        if getattr(parent, "_b_key", None) is None or not torch.equal(parent._b_key, bh):
            parent.set_task_covar(bh)
            parent._b_key = bh
        self._plan = parent
        return parent

    @property
    def requires_grad(self):
        return bool(super().requires_grad or self.B.requires_grad)

    def representation(self):
        return (self.x1, self.x2, self.lengthscale, self.outputscale, self.B)

    def hyper_tensors(self):
        return [self.lengthscale, self.outputscale, self.B]

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _bilinear_derivative_list(self, left, right):
        p = self.plan(getattr(self, "_last_noise", 0.0))
        gl, go = p.bilinear_grad(left, right)
        dB = p.task_covar_grad(left, right)
        return [torch.tensor(gl, device=self.device, dtype=self.dtype).reshape(self.lengthscale.shape),
                torch.tensor(go, device=self.device, dtype=self.dtype).reshape(self.outputscale.shape),
                dB.to(device=self.device, dtype=self.B.dtype)]

    def _bilinear_derivative(self, left, right):
        gl, go, _ = self._bilinear_derivative_list(left, right)
        return gl, go

    def _transpose_nonbatch(self):
        if self.same:
            return self
        return KroneckerKernelLinearOperator(self.x2, self.x1, self.kind, self.lengthscale, self.outputscale, self.B.transpose(-1, -2),
                                             self.cols, self.rows)

    def detach(self):
        return KroneckerKernelLinearOperator(self.x1.detach(), None if self.same else self.x2.detach(), self.kind,
                                             self.lengthscale.detach(), self.outputscale.detach(), self.B.detach(), self.rows, self.cols)

    def to_dense(self):
        return _KernelDense.apply(self)

    def diagonal(self, dim1=-2, dim2=-1):
        """s k(x1_i, x2_i) B[a, a] at row i T + a."""
        if self.shape[0] != self.shape[1]:
            raise RuntimeError(f"diagonal of a non-square operator {tuple(self.shape)} is undefined")
        return self.plan().diag()

    _diagonal = diagonal

    def __getitem__(self, index):
        """Slices that start and stop on multiples of T re-index x1 / x2 (prediction slices the joint operator at n T)."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        if self.rows is not None or self.cols is not None:
            raise NotImplementedError("a masked Kronecker operator takes no slices: mask the sliced operator instead")
        T = self.num_tasks
        x2 = self.x1 if self.same else self.x2
        rs, cs = _aligned(ri, T, self.x1.size(0)), _aligned(ci, T, x2.size(0))
        if rs is None or cs is None:
            raise NotImplementedError("a Kronecker multitask operator takes row / column slices that start and stop on multiples of "
                                      "the number of tasks")
        return KroneckerKernelLinearOperator(self.x1[rs], x2[cs], self.kind, self.lengthscale, self.outputscale, self.B)

    def mul(self, other):
        raise NotImplementedError("a Kronecker multitask operator takes one task covariance")

    __mul__ = mul

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("a Kronecker multitask operator adds a (Constant)DiagLinearOperator only")


class LCMKernelLinearOperator(KernelLinearOperator):
    """sum_q (s_q K_q(x1, x2)) (x) B_q over interleaved rows i T + a, Q = 1..4 (LCMKernel, kernels/lcm_kernel.py; the reference sums
    KroneckerProductLinearOperators into a SumLinearOperator): ONE engine operator (gp_plan_set_kron_terms) on the terms' data plans.
    `terms` are unmasked KroneckerKernelLinearOperators of one shape and T; each keeps its own inputs (active dimensions), kind,
    lengthscale, outputscale and B.  The hyper-parameters are [l_1, s_1, B_1, ..., l_Q, s_Q, B_Q]; their gradients come from
    gp_kron_terms_grad.  Input gradients are not available: the terms refuse inputs that require grad."""

    _family = "lcm"
    _noun = "LCM"
    _sum_term = _factor = _single_plan = False

    def __init__(self, terms):
        terms = list(terms)
        if not 1 <= len(terms) <= 4:
            raise NotImplementedError(f"an LCM operator takes 1 to 4 terms on the accelerated path (got {len(terms)})")
        for t in terms:
            if type(t) is not KroneckerKernelLinearOperator or t.rows is not None or t.cols is not None:
                raise NotImplementedError(f"the terms of an LCM operator are unmasked Kronecker operators (got {type(t).__name__})")
        first = terms[0]
        if any(tuple(t.shape) != tuple(first.shape) or t.num_tasks != first.num_tasks or t.same != first.same for t in terms):
            raise RuntimeError("the terms of an LCM operator must share their shape, number of tasks and squareness")
        super().__init__(first.x1, None if first.same else first.x2, first.kind, first.lengthscale, first.outputscale)
        self.terms = terms
        self.num_tasks = first.num_tasks
        self.same = first.same
        self._data_ops = []
        for i, t in enumerate(terms):
            op = KernelLinearOperator(t.x1, None if t.same else t.x2, t.kind, t.lengthscale, t.outputscale)
            op._plan_slot = _slot("lcm", "lcm_term", i)   # two terms over the same inputs never share a plan
            self._data_ops.append(op)

    @property
    def shape(self):
        return self.terms[0].shape

    def plan(self, noise=0.0) -> Plan:
        datas = []
        for op in self._data_ops:
            d = op.plan(0.0)
            if getattr(d, "_noise_diag", None) is not None:
                d.set_noise_diag(None)
            datas.append(d)
        nz = float(noise.detach().reshape(-1)[0]) if torch.is_tensor(noise) else float(noise)
        T = self.num_tasks
        parent = _parent_plan(_LCM_PLANS, (tuple(id(d) for d in datas), T), lambda: LcmPlan(datas, T))
        # the data plans may have been re-packed or re-pointed since the last use: re-attach them (validation, no allocation)
        parent.attach(datas[0], datas, T)
        hk = (nz, tuple((d.kind, tuple(d.lengthscale), d.outputscale) for d in datas))
        if parent._hyp_key != hk:
            parent.set_noise(nz)
            parent._hyp_key = hk
        bh = getattr(self, "_b_host", None)
        if bh is None:
            bh = self._b_host = torch.stack([t.B.detach().float() for t in self.terms]).cpu()
        if getattr(parent, "_b_key", None) is None or not torch.equal(parent._b_key, bh):
            parent.set_term_covars(bh)
            parent._b_key = bh
        self._plan = parent
        return parent

    @property
    def requires_grad(self):
        return any(t.requires_grad for t in self.terms)

    def representation(self):
        return tuple(v for t in self.terms for v in t.representation())

    def hyper_tensors(self):
        return [h for t in self.terms for h in (t.lengthscale, t.outputscale, t.B)]

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _bilinear_derivative_list(self, left, right):
        gl, go, dB = self.plan(getattr(self, "_last_noise", 0.0)).terms_grad(left, right)
        out = []
        for t, l, o, b in zip(self.terms, gl, go, dB):
            out += [torch.tensor(l, device=self.device, dtype=self.dtype).reshape(t.lengthscale.shape),
                    torch.tensor(o, device=self.device, dtype=self.dtype).reshape(t.outputscale.shape),
                    b.to(device=self.device, dtype=t.B.dtype)]
        return out

    def _bilinear_derivative(self, left, right):
        raise NotImplementedError("an LCM operator has one lengthscale and outputscale per term: use _bilinear_derivative_list")

    def _transpose_nonbatch(self):
        if self.same:
            return self
        return LCMKernelLinearOperator([t._transpose_nonbatch() for t in self.terms])

    def detach(self):
        return LCMKernelLinearOperator([t.detach() for t in self.terms])

    def to_dense(self):
        return _KernelDense.apply(self)

    def diagonal(self, dim1=-2, dim2=-1):
        """sum_q s_q k_q(x1_i, x2_i) B_q[a, a] at row i T + a."""
        if self.shape[0] != self.shape[1]:
            raise RuntimeError(f"diagonal of a non-square operator {tuple(self.shape)} is undefined")
        return self.plan().diag()

    _diagonal = diagonal

    def __getitem__(self, index):
        """Slices that start and stop on multiples of T slice every term (prediction slices the joint operator at n T)."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        return LCMKernelLinearOperator([t[ri, ci] for t in self.terms])

    def mul(self, other):
        raise NotImplementedError("an LCM operator takes no further factor")

    __mul__ = mul

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("an LCM operator adds a (Constant)DiagLinearOperator only")


def _mask_index(mask, n, what):
    """Strictly increasing int64 indices of a boolean mask [n] (None: every index)."""
    if mask is None:
        return None
    mask = torch.as_tensor(mask)
    if mask.dtype != torch.bool or mask.dim() != 1 or mask.numel() != n:
        raise RuntimeError(f"the {what} mask must be a boolean vector of {n} entries (got {mask.dtype}, {tuple(mask.shape)})")
    return mask.nonzero().reshape(-1)


def _take_square(op, idx, memo):
    """op[idx, idx] of a square operator with every input indexed ONCE, so that the result is square again (x2 is x1): two
    fancy indexes of x1 would give two tensors and a cross plan.  The terms of a sum or product and the components of an additive
    operator share their indexed inputs through memo."""
    def take(x):
        if id(x) not in memo:
            memo[id(x)] = (x, x[idx])    # x is kept so that its id stays unique while memo lives
        return memo[id(x)][1]

    if getattr(op, "_comm", None) is not None or getattr(op, "_row_begin", 0) != 0:
        raise NotImplementedError(f"an observation mask on a row-sharded {type(op).__name__} is not available")
    t = type(op)
    if t is HadamardKernelLinearOperator:
        return HadamardKernelLinearOperator(take(op.x1), None, op.kind, op.lengthscale, op.outputscale, take(op.t1), None, op.B)
    if t is SumKernelLinearOperator:
        return SumKernelLinearOperator([_take_square(o, idx, memo) for o in op.ops])
    if t is ProductKernelLinearOperator:
        return ProductKernelLinearOperator([_take_square(o, idx, memo) for o in op.ops])
    if t is AdditiveKernelLinearOperator:
        return AdditiveKernelLinearOperator([_take_square(o, idx, memo) for o in op.ops], op.max_degree)
    if op._single_plan:
        return op._with(take(op.x1), None)
    raise NotImplementedError(f"observation masks are not available for {t.__name__}")


def MaskedLinearOperator(base, row_mask, col_mask):
    """base restricted to the rows where row_mask and the columns where col_mask is True (linear_operator's MaskedLinearOperator,
    used by settings.observation_nan_policy("mask")), as an engine operator:
      * AddedDiagLinearOperator: the kernel and the diagonal are masked separately;
      * KroneckerKernelLinearOperator: the same operator on a plan with the mask set (gp_plan_set_kron_observed);
      * plain, sum, product, additive, periodic, RQ, polynomial, spectral and Hadamard operators: their inputs (and task ids)
        re-indexed; a square operator with equal masks stays square (its inputs are indexed once);
      * derivative, SKI and batched operators: NotImplementedError.
    row_mask / col_mask are boolean vectors over the rows / columns (None: all)."""
    n1, n2 = int(base.shape[-2]), int(base.shape[-1])
    ri, ci = _mask_index(row_mask, n1, "row"), _mask_index(col_mask, n2, "column")
    if isinstance(base, AddedDiagLinearOperator):
        if not ((ri is None and ci is None) or (ri is not None and ci is not None and torch.equal(ri, ci))):
            raise NotImplementedError("a masked K + D takes equal row and column masks")
        if ri is None:
            return base
        if base.per_row:
            diag = DiagLinearOperator(base.diag.diag_vec[..., ri])
        else:
            diag = ConstantDiagLinearOperator(base.diag.diag_value, ri.numel())
        return AddedDiagLinearOperator(MaskedLinearOperator(base.kernel_op, row_mask, col_mask), diag)
    if isinstance(base, KroneckerKernelLinearOperator):
        equal = (ri is None and ci is None) or (ri is not None and ci is not None and torch.equal(ri, ci))
        if base.same and not equal:
            raise NotImplementedError("a square Kronecker operator takes equal row and column masks")
        return base.masked(ri, None if base.same else ci)
    if not isinstance(base, KernelLinearOperator) or isinstance(base, (DerivKernelLinearOperator, SKIKernelLinearOperator)):
        raise NotImplementedError(f"observation masks are not available for {type(base).__name__}")
    if base.same and ri is not None and ci is not None and torch.equal(ri, ci):
        return _take_square(base, ri, {})
    return base[slice(None) if ri is None else ri, slice(None) if ci is None else ci]

_DERIV_NAMES = {"rbf": "RBFKernelGrad", "matern52": "Matern52KernelGrad"}


class DerivKernelLinearOperator(KernelLinearOperator):
    """The covariance of values and gradients over interleaved rows i (d+1) + a, kind "rbf" (RBFKernelGrad,
    kernels/rbf_kernel_grad.py:60-104) or "matern52" (Matern52KernelGrad, kernels/matern52_kernel_grad.py), after the reference's
    perfect shuffle: ONE engine operator (gp_plan_set_deriv / gp_plan_set_deriv_kind) on the plan of the plain kernel of that kind;
    no N (d+1) x N (d+1) matrix is stored.  The hyper-parameters are lengthscale (scalar or ARD) and outputscale.  Input gradients
    are not available: inputs that require grad are refused."""

    _family = "deriv"
    _noun = "derivative"
    _sum_term = _factor = _single_plan = False

    def __init__(self, x1, x2, lengthscale, outputscale=None, kind="rbf"):
        if kind not in _DERIV_NAMES:
            raise ValueError(f"derivative observations are available for the 'rbf' and 'matern52' kernels (got {kind!r})")
        name = _DERIV_NAMES[kind]
        if x1.requires_grad or (x2 is not None and x2.requires_grad):
            raise RuntimeError(f"gradients with respect to the inputs of a derivative operator ({name}) are not implemented: "
                               "pass inputs that do not require grad")
        d = x1.size(-1)
        if d > 16:
            raise RuntimeError(f"{name} on the accelerated path supports d <= 16 input dimensions (got d={d})")
        super().__init__(x1, x2, kind, lengthscale, outputscale)
        self.num_outputs = d + 1
        self._data_op = KernelLinearOperator(x1, x2, kind, lengthscale, self.outputscale)
        self._data_op._plan_slot = _slot("deriv", "data")

    @property
    def shape(self):
        n2 = self.x1.size(0) if self.same else self.x2.size(0)
        return torch.Size([self.x1.size(0) * self.num_outputs, n2 * self.num_outputs])

    def plan(self, noise=0.0) -> Plan:
        data = self._data_op.plan(0.0)
        if getattr(data, "_noise_diag", None) is not None:
            data.set_noise_diag(None)
        nz = float(noise.detach().reshape(-1)[0]) if torch.is_tensor(noise) else float(noise)
        # one parent per (data plan, kind): never re-attached to a data plan of another kind
        parent = _parent_plan(_DERIV_PLANS, (id(data), self.kind), lambda: DerivPlan(data, self.kind))
        # the data plan may have been re-packed or re-pointed since the last use: re-attach it (validation, no allocation)
        parent.attach(data, self.kind)
        hk = (nz, tuple(data.lengthscale), data.outputscale)
        if parent._hyp_key != hk:
            parent.set_noise(nz)
            parent._hyp_key = hk
        self._plan = parent
        return parent

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _transpose_nonbatch(self):
        """K(x1, x2)^T = K(x2, x1): the value / gradient blocks swap with D -> -D."""
        if self.same:
            return self
        return DerivKernelLinearOperator(self.x2, self.x1, self.lengthscale, self.outputscale, self.kind)

    def detach(self):
        return DerivKernelLinearOperator(self.x1.detach(), None if self.same else self.x2.detach(), self.lengthscale.detach(),
                                         self.outputscale.detach(), self.kind)

    def with_outputscale(self, outputscale):
        return DerivKernelLinearOperator(self.x1, None if self.same else self.x2, self.lengthscale, outputscale, self.kind)

    def to_dense(self):
        return _KernelDense.apply(self)

    def diagonal(self, dim1=-2, dim2=-1):
        """s at value rows, s / l_a^2 (RBF, rbf_kernel_grad.py:106-115) or (5/3) s / l_a^2 (Matern-5/2) at derivative rows for
        x2 == x1."""
        if self.shape[0] != self.shape[1]:
            raise RuntimeError(f"diagonal of a non-square operator {tuple(self.shape)} is undefined")
        return self.plan().diag()

    _diagonal = diagonal

    def __getitem__(self, index):
        """Slices that start and stop on multiples of d + 1 re-index x1 / x2 (prediction slices the joint operator at n (d+1))."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        R = self.num_outputs
        x2 = self.x1 if self.same else self.x2
        rs, cs = _aligned(ri, R, self.x1.size(0)), _aligned(ci, R, x2.size(0))
        if rs is None or cs is None:
            raise NotImplementedError("a derivative operator takes row / column slices that start and stop on multiples of d + 1")
        return DerivKernelLinearOperator(self.x1[rs], x2[cs], self.lengthscale, self.outputscale, self.kind)

    def mul(self, other):
        raise NotImplementedError(f"a derivative operator ({_DERIV_NAMES[self.kind]}) does not multiply by a task covariance")

    __mul__ = mul

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("a derivative operator adds a (Constant)DiagLinearOperator only")


class SumKernelLinearOperator(KernelLinearOperator):
    """K_1 + ... + K_m over the same inputs (AdditiveKernel, kernels/kernel.py:592-621).  The reference evaluates every term
    densely and adds the matrices; here the sum is ONE engine operator (gp_plan_set_sum): a product launches the fused kernel of
    every term into disjoint partial slots, the solves / preconditioner / SLQ run on the sum, and the hyper-parameter gradients
    of each term come from that term's own bilinear derivative with the shared left / right factors."""

    _family = "sum"
    _noun = "kernel sum"
    _factor = _single_plan = False

    def __init__(self, ops):
        ops = list(ops)
        flat = []
        for o in ops:
            flat.extend(o.ops if isinstance(o, SumKernelLinearOperator) else [o])
        if not 1 <= len(flat) <= 4:
            raise RuntimeError(f"a kernel sum takes 1 to 4 terms (got {len(flat)})")
        for o in flat:
            if not o._sum_term:
                raise NotImplementedError(f"sums that contain {o._noun} operators are not available on the accelerated path")
        first = flat[0]
        for o in flat[1:]:
            if o.shape != first.shape or o.same != first.same:
                raise RuntimeError(f"cannot add kernels of shapes {tuple(first.shape)} and {tuple(o.shape)}")
        # one engine plan per term even when the terms see the same inputs: re-wrap (the caller's operators stay usable on their
        # own) and give every term its own slot of the plan cache; a term keeps its row sharding
        self.ops = []
        for i, o in enumerate(flat):
            t = o._with(o.x1, o.x2)
            t._plan_slot = _slot(o._family, "sum_term", i)
            t._comm, t._row_begin, t._row_count = o._comm, o._row_begin, o._row_count
            self.ops.append(t)
        self.x1, self.x2, self.same = first.x1, first.x2, first.same
        self.kind = "sum"
        self.lengthscale, self.outputscale = first.lengthscale, first.outputscale   # representative only (device / dtype)
        self._comm, self._row_begin, self._row_count = first._comm, first._row_begin, first._row_count
        self._plan = None
        self._plan_slot = _slot("sum", "own")

    def hyper_tensors(self):
        return [t for o in self.ops for t in o.hyper_tensors()]

    def input_tensors(self):
        return [t for o in self.ops for t in o.input_tensors()]

    def _input_grad_list(self, left, right, needs):
        """One gp_kmv_input_grad call per term (the engine refuses a kernel-sum plan)."""
        out, k = [], 0
        for o in self.ops:
            m = len(o.input_tensors())
            out.extend(o._input_grad_list(left, right, needs[k:k + m]))
            k += m
        return out

    def _dense_input_grad_list(self, w, needs):
        """One gp_kdense_input_grad call per term."""
        out, k = [], 0
        for o in self.ops:
            m = len(o.input_tensors())
            out.extend(o._dense_input_grad_list(w, needs[k:k + m]))
            k += m
        return out

    def _bilinear_derivative_list(self, left, right):
        out = []
        for o in self.ops:
            o._last_noise = 0.0
            out.extend(o._bilinear_derivative_list(left, right))
        return out

    @property
    def requires_grad(self):
        return any(o.requires_grad for o in self.ops)

    def representation(self):
        return tuple(t for o in self.ops for t in o.representation())

    def plan(self, noise=0.0) -> Plan:
        terms = [o.plan(0.0) for o in self.ops]
        nz = float(noise.detach().reshape(-1)[0]) if torch.is_tensor(noise) else float(noise)
        x2 = None if self.same else self.x2
        parent = _parent_plan(_SUM_PLANS, (tuple(id(t) for t in terms), self._plan_slot),
                              lambda: Plan(self.x1, x2, backend="auto", row_begin=self._row_begin, row_count=self._row_count,
                                           comm=self._comm), self.x1, x2)
        # the terms may have been re-created / re-packed since the last use: (re-)attach them every time (validation + a
        # 64-float upload, no allocation), then set the noise of the sum
        parent.set_sum(terms)
        if parent._hyp_key != nz:
            parent.set_hypers("rbf", [1.0], 1.0, nz)
            parent._hyp_key = nz
        self._plan = parent
        return parent

    def _transpose_nonbatch(self):
        return self if self.same else SumKernelLinearOperator([o._transpose_nonbatch() for o in self.ops])

    def detach(self):
        return SumKernelLinearOperator([o.detach() for o in self.ops])

    def to_dense(self):
        out = self.ops[0].to_dense()
        for o in self.ops[1:]:
            out = out + o.to_dense()
        return out

    def diagonal(self, dim1=-2, dim2=-1):
        out = self.ops[0].diagonal()
        for o in self.ops[1:]:
            out = out + o.diagonal()
        return out

    _diagonal = diagonal

    def __getitem__(self, index):
        parts = [o[index] for o in self.ops]
        if torch.is_tensor(parts[0]):
            return sum(parts[1:], parts[0])
        return SumKernelLinearOperator(parts)

    def _bilinear_derivative(self, left, right):
        raise NotImplementedError("a kernel sum has one (lengthscale, outputscale) pair per term: use _bilinear_derivative_list")


class ProductKernelLinearOperator(KernelLinearOperator):
    """K_1 o ... o K_m over the same inputs (ProductKernel, kernels/kernel.py:634-690).  The reference evaluates every factor
    densely and multiplies the matrices; here the product is ONE engine operator (gp_plan_set_product): a product with a block of
    vectors is one fused kernel launch that forms prod_f k_f per pair in registers, the solves / preconditioner / SLQ run on it, and
    one engine call returns every factor's hyper-parameter gradients.  2 to 4 RBF / Matern factors; gradients with respect to the
    inputs are not available through a product."""

    _family = "product"
    _noun = "kernel product"
    _sum_term = _single_plan = False

    def __init__(self, ops):
        flat = []
        for o in ops:
            flat.extend(o.ops if isinstance(o, ProductKernelLinearOperator) else [o])
        if not 2 <= len(flat) <= 4:
            raise NotImplementedError(f"a kernel product takes 2 to 4 factors on the accelerated path (got {len(flat)})")
        first = flat[0]
        for o in flat:
            if not o._factor:
                raise o._no_product()
            if o.shape != first.shape or o.same != first.same:
                raise RuntimeError(f"cannot multiply kernels of shapes {tuple(first.shape)} and {tuple(o.shape)}")
            if o._comm is not None or o._row_begin != 0 or o._row_count not in (0, o.shape[0]):
                raise NotImplementedError("a row-sharded kernel product is not available on the accelerated path")
            if o.x1.requires_grad or (not o.same and o.x2.requires_grad):
                raise NotImplementedError("gradients with respect to the inputs of a kernel product (deep kernel learning, test-input "
                                          "gradients) are not available on the accelerated path")
        # one engine plan per factor even when the factors see the same inputs: re-wrap and give each its own plan-cache slot
        self.ops = []
        for i, o in enumerate(flat):
            t = o._with(o.x1, o.x2)
            t._plan_slot = _slot(o._family, "product_factor", i)
            self.ops.append(t)
        self.x1, self.x2, self.same = first.x1, first.x2, first.same
        self.kind = "product"
        self.lengthscale, self.outputscale = first.lengthscale, first.outputscale   # representative only (device / dtype)
        self._comm, self._row_begin, self._row_count = None, 0, 0
        self._plan = None

    def hyper_tensors(self):
        return [t for o in self.ops for t in o.hyper_tensors()]

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    @staticmethod
    def _split_grads(gl, go, n_ls, scales):
        """The engine's flat result (the factors' lengthscale gradients one after the other, dF/dS of the combined scale
        S = prod_f s_f) as per-factor pairs: (lengthscale gradient [n_ls_f], dF/ds_f = S / s_f dF/dS)."""
        S = 1.0
        for s in scales:
            S *= s
        out, k = [], 0
        for n, s in zip(n_ls, scales):
            out.append((gl[k:k + n], go * S / s))
            k += n
        return out

    def _bilinear_derivative_list(self, left, right):
        gl, go = self.plan(0.0).bilinear_grad(left, right)
        parts = self._split_grads(gl, go, [o.lengthscale.numel() for o in self.ops], [o._host_hypers()[0][-1][0] for o in self.ops])
        out = []
        for o, (g, gs) in zip(self.ops, parts):
            out.append(torch.tensor(g, device=self.device, dtype=self.dtype).reshape(o.lengthscale.shape))
            out.append(torch.tensor(gs, device=self.device, dtype=self.dtype).reshape(o.outputscale.shape))
        return out

    def _bilinear_derivative(self, left, right):
        raise NotImplementedError("a kernel product has one (lengthscale, outputscale) pair per factor: use _bilinear_derivative_list")

    @property
    def requires_grad(self):
        return any(o.requires_grad for o in self.ops)

    def representation(self):
        return tuple(t for o in self.ops for t in o.representation())

    def plan(self, noise=0.0) -> Plan:
        factors = [o.plan(0.0) for o in self.ops]
        nz = float(noise.detach().reshape(-1)[0]) if torch.is_tensor(noise) else float(noise)
        x2 = None if self.same else self.x2
        parent = _parent_plan(_PRODUCT_PLANS, tuple(id(f) for f in factors), lambda: Plan(self.x1, x2, backend="auto"), self.x1, x2)
        # the factors may have been re-created / re-packed since the last use: (re-)attach them every time (validation only),
        # then set the noise of the product
        parent.set_product(factors)
        if parent._hyp_key != nz:
            parent.set_hypers("rbf", [1.0], 1.0, nz)
            parent._hyp_key = nz
        self._plan = parent
        return parent

    def _transpose_nonbatch(self):
        return self if self.same else ProductKernelLinearOperator([o._transpose_nonbatch() for o in self.ops])

    def detach(self):
        return ProductKernelLinearOperator([o.detach() for o in self.ops])

    def __getitem__(self, index):
        parts = [o[index] for o in self.ops]
        if torch.is_tensor(parts[0]):
            out = parts[0]
            for t in parts[1:]:
                out = out * t
            return out
        return ProductKernelLinearOperator(parts)

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("a kernel product adds a (Constant)DiagLinearOperator only: sums that contain products are not "
                                  "available on the accelerated path")


ADDITIVE_MAX_COMPONENTS = 32
ADDITIVE_MAX_DEGREE = 8
_ADDITIVE_KINDS = ("rbf", "matern12", "matern32", "matern52")
_ADDITIVE_X: "collections.OrderedDict[tuple, list]" = collections.OrderedDict()
_ADDITIVE_X_ROLES = 8      # stacked inputs kept: the most recently used roles (shape, side, device), two buffers each


def _stable_stack(cols, role):
    """torch.cat(cols, -1), or the tensor an earlier operator stacked from the same values: the kernels of an additive model are
    called on fresh [n, 1] slices every forward, and the engine plan is keyed on its input buffer, so equal inputs keep one buffer
    and their plan is neither re-pointed nor re-packed."""
    x = torch.cat([c.detach() for c in cols], -1)
    with _PLAN_LOCK:
        seen = _ADDITIVE_X.pop(role, [])
        _ADDITIVE_X[role] = seen   # most recently used last
        found = next((old for old in seen if torch.equal(old, x)), None)   # one device comparison per kept buffer of this role
        if found is None:
            seen.append(x)
            del seen[:-2]
        while len(_ADDITIVE_X) > _ADDITIVE_X_ROLES:
            _ADDITIVE_X.popitem(last=False)
    return x if found is None else found


def _additive_components(ops, what):
    """The D one-dimensional RBF / Matern operators of an additive model, checked; raises NotImplementedError naming what it refuses."""
    ops = list(ops)
    if not 1 <= len(ops) <= ADDITIVE_MAX_COMPONENTS:
        raise NotImplementedError(f"{what}: an additive operator takes 1 to {ADDITIVE_MAX_COMPONENTS} components on the accelerated "
                                  f"path (got {len(ops)})")
    first = ops[0]
    for o in ops:
        if type(o) is not KernelLinearOperator:
            raise NotImplementedError(f"{what}: every component must be a plain RBF / Matern kernel operator (optionally scaled) on "
                                      f"the accelerated path, not {type(o).__name__}")
        if o.kind not in _ADDITIVE_KINDS or o.kind != first.kind:
            raise NotImplementedError(f"{what}: the components must share one RBF / Matern kind (got {o.kind!r} and {first.kind!r})")
        if o.x1.dim() != 2 or o.x1.size(-1) != 1:
            raise NotImplementedError(f"{what}: every component must act on one input dimension ([n, 1] inputs), got "
                                      f"{tuple(o.x1.shape)}")
        if o.lengthscale.numel() != 1 or o.outputscale.numel() != 1:
            raise NotImplementedError(f"{what}: every component needs one lengthscale and one outputscale")
        if o.shape != first.shape or o.same != first.same:
            raise RuntimeError(f"{what}: component shapes {tuple(first.shape)} and {tuple(o.shape)} differ")
        if o._comm is not None or o._row_begin != 0 or o._row_count not in (0, o.shape[0]):
            raise NotImplementedError(f"{what}: a row-sharded additive operator is not available on the accelerated path")
        if o.x1.requires_grad or (not o.same and o.x2.requires_grad):
            raise NotImplementedError(f"{what}: gradients with respect to the inputs of an additive operator (deep kernel learning, "
                                      "test-input gradients) are not available on the accelerated path")
    return ops


class AdditiveKernelLinearOperator(KernelLinearOperator):
    """sum_{m=1}^{M} e_m(K_1, .., K_D) over D one-dimensional kernel operators K_i = s_i k_i(x_i, x'_i), e_m the elementary symmetric
    polynomial of degree m taken entry by entry (Duvenaud et al.'s additive GPs): M = 1 is `.sum(dim=-3)` of the batch of
    components, M >= 2 `sum_interaction_terms(..., max_degree=M)`.  The reference evaluates the D components densely and combines
    them by Newton-Girard; here the operator is ONE engine plan (gp_plan_set_additive) whose kernels form the positive recurrence
    e_m += c_i e_{m-1} per pair, so products, solves, the preconditioner and SLQ never hold an N x N matrix.  The components' [n, 1]
    inputs are stacked into one [n, D] block; a component's lengthscale and scale stay its own tensors (hyper_tensors), so autograd
    reaches batched [D, 1, 1] / [D] parameters and sums the gradients of a shared one.  1 <= D <= 32, M <= 8 after clamping to D;
    gradients with respect to the inputs are not available."""

    _family = "additive"
    _noun = "additive"
    _sum_term = _factor = _single_plan = False

    def __init__(self, ops, max_degree=1):
        self.ops = _additive_components(ops, "AdditiveKernelLinearOperator")
        D = len(self.ops)
        if int(max_degree) < 1:
            raise ValueError(f"max_degree must be >= 1 (got {max_degree})")
        self.max_degree = min(int(max_degree), D)     # e_m = 0 for m > D
        if self.max_degree > ADDITIVE_MAX_DEGREE:
            raise NotImplementedError(f"an additive operator takes interaction terms up to degree {ADDITIVE_MAX_DEGREE} on the "
                                      f"accelerated path (got max_degree={max_degree} with {D} components)")
        first = self.ops[0]
        self.same = first.same
        n1 = first.shape[0]
        self.x1 = _stable_stack([o.x1 for o in self.ops], ("x1", n1, D, str(first.x1.device)))
        self.x2 = self.x1 if self.same else _stable_stack([o.x2 for o in self.ops], ("x2", first.shape[1], D, str(first.x1.device)))
        self.kind = first.kind
        self.lengthscale, self.outputscale = first.lengthscale, first.outputscale   # representative only (device / dtype)
        self._comm, self._row_begin, self._row_count = None, 0, 0
        self._plan = None
        self._plan_slot = _slot("additive", "own")

    def hyper_tensors(self):
        return [t for o in self.ops for t in o.hyper_tensors()]

    def input_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _host_hypers(self, noise_t=None):
        """([l_1 .. l_D], [s_1 .. s_D], noise) with one device -> host read."""
        cached = getattr(self, "_hyp_host", None)
        if cached is None or (noise_t is not None and cached[3] is not noise_t):
            parts = [o.lengthscale.detach().reshape(1).float() for o in self.ops]
            parts += [o.outputscale.detach().reshape(1).float().to(o.lengthscale.device) for o in self.ops]
            if noise_t is not None:
                parts.append(noise_t.detach().reshape(-1)[:1].float())
            vals = torch.cat(parts).tolist()
            D = len(self.ops)
            cached = (vals[:D], vals[D:2 * D], vals[2 * D] if noise_t is not None else None, noise_t)
            self._hyp_host = cached
        return cached

    def plan(self, noise=0.0) -> Plan:
        fresh = False
        if self._plan is None:
            self._plan = _get_plan(self.x1, None if self.same else self.x2, "auto", 0, 0, None,
                                   self._plan_slot, owner=self)
            fresh = True
        if torch.is_tensor(noise):
            ls, sc, nz, _ = self._host_hypers(noise)
        else:
            ls, sc, _, _ = self._host_hypers(None)
            nz = float(noise)
        p = self._plan
        akey = (self.max_degree, tuple(sc))
        if fresh or getattr(p, "_add_key", None) != akey:
            p.set_additive(self.max_degree, sc)
            p._add_key = akey
        key = (self.kind, tuple(ls), 1.0, nz)
        if fresh or getattr(p, "_hyp_key", None) != key:
            p.set_hypers(self.kind, ls, 1.0, nz)
            p._hyp_key = key
        return p

    def _bilinear_derivative_list(self, left, right):
        gl, gs = self.plan(getattr(self, "_last_noise", 0.0)).bilinear_grad(left, right)
        vals = torch.tensor(list(gl) + list(gs), device=self.device, dtype=self.dtype)
        D = len(self.ops)
        out = []
        for i, o in enumerate(self.ops):
            out.append(vals[i].reshape(o.lengthscale.shape))
            out.append(vals[D + i].reshape(o.outputscale.shape))
        return out

    def _bilinear_derivative(self, left, right):
        raise NotImplementedError("an additive operator has one (lengthscale, scale) pair per component: use _bilinear_derivative_list")

    def _input_grad_list(self, left, right, needs):
        raise NotImplementedError("gradients with respect to the inputs of an additive operator are not available on the accelerated path")

    _dense_input_grad_list = _input_grad_list

    @property
    def requires_grad(self):
        return any(o.requires_grad for o in self.ops)

    def representation(self):
        return tuple(t for o in self.ops for t in o.representation())

    def _transpose_nonbatch(self):
        return self if self.same else AdditiveKernelLinearOperator([o._transpose_nonbatch() for o in self.ops], self.max_degree)

    def detach(self):
        return AdditiveKernelLinearOperator([o.detach() for o in self.ops], self.max_degree)

    def diagonal(self, dim1=-2, dim2=-1):
        """The constant sum_m e_m(s_1 .. s_D) for x2 == x1, K(x1_i, x2_i) for a cross operator of equal sizes."""
        if not self.same and self.ops[0].x1.size(0) != self.ops[0].x2.size(0):
            raise RuntimeError(f"diagonal of a non-square operator {tuple(self.shape)} is undefined")
        return self.plan().diag()

    _diagonal = diagonal

    def __getitem__(self, index):
        """Row / column blocks (the train / test blocks of prediction) re-index every component: a cross plan for x1 != x2."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        if isinstance(ri, int):
            return self.plan().rows(torch.tensor([ri], device=self.device))[0][ci]
        return AdditiveKernelLinearOperator([o[ri, ci] for o in self.ops], self.max_degree)

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("an additive operator adds a (Constant)DiagLinearOperator only: sums that contain additive "
                                  "operators are not available on the accelerated path")

    def mul(self, other):
        raise NotImplementedError("products that contain an additive operator are not available on the accelerated path")

    __mul__ = mul


SPECTRAL_MAX_MIXTURES = 16
SPECTRAL_MAX_DIMS = 8
SPECTRAL_MAX_QD = 32


class SpectralMixtureKernelLinearOperator(KernelLinearOperator):
    """S prod_d sum_q w_q exp(-2 pi^2 v_qd^2 tau_d^2) cos(2 pi mu_qd tau_d), tau = x1 - x2 (kernels/spectral_mixture_kernel.py, which
    sums the components of each dimension and multiplies over the dimensions, through dense [Q, n, m, d] temporaries) as ONE engine
    plan (gp_plan_set_spectral): products, solves, the preconditioner and SLQ never hold an N x N matrix.  weights [Q], means and
    scales [Q, 1, d] (or [Q, d]) are the constrained parameter tensors, or their slices for one element of a batch; autograd reaches
    them through _bilinear_derivative_list.  S is the outputscale of a ScaleKernel around the kernel (None: 1, no gradient).
    1 <= Q <= 16, 1 <= d <= 8, Q d <= 32; gradients with respect to the inputs are not available."""

    _family = "spectral"
    _noun = "spectral mixture"
    _sum_term = _factor = _input_grads = _row_sharding = False
    _params = ("weights", "means", "scales")
    _plan_backend = "auto"

    def __init__(self, x1, x2, weights, means, scales, outputscale=None):
        super().__init__(x1, x2, "rbf", torch.ones((), device=x1.device), outputscale)
        Q, d = weights.numel(), x1.size(-1)
        if means.numel() != Q * d or scales.numel() != Q * d:
            raise RuntimeError(f"spectral mixture: means {tuple(means.shape)} and scales {tuple(scales.shape)} do not hold {Q} x {d} "
                               "values")
        if not (1 <= Q <= SPECTRAL_MAX_MIXTURES and 1 <= d <= SPECTRAL_MAX_DIMS and Q * d <= SPECTRAL_MAX_QD):
            raise NotImplementedError(f"a spectral mixture operator takes 1 <= num_mixtures <= {SPECTRAL_MAX_MIXTURES} over 1 <= d <= "
                                      f"{SPECTRAL_MAX_DIMS} input dimensions with num_mixtures * d <= {SPECTRAL_MAX_QD} on the "
                                      f"accelerated path (got {Q} and d = {d})")
        if x1.requires_grad or (x2 is not None and x2.requires_grad):
            raise NotImplementedError("gradients with respect to the inputs of a spectral mixture operator (deep kernel learning, "
                                      "test-input gradients) are not available on the accelerated path")
        self.weights, self.means, self.scales = weights, means, scales
        self.num_mixtures = Q

    @property
    def _scale_is_hyper(self):
        return self._scaled      # without a ScaleKernel S = 1 has no gradient

    def _ctor_args(self):
        return (self.weights, self.means, self.scales)

    def _engine_calls(self, hyp, nz):
        w, mu, v = hyp[:3]
        os_ = hyp[3][0] if self._scaled else 1.0
        Q = len(w)
        # set_hypers carries the outputscale and noise (the kind and lengthscale are not used); set_spectral is re-sent only when
        # the parameters' host values change
        return [("_hyp_key", ("rbf", (1.0,), os_, nz), lambda p: p.set_hypers("rbf", 1.0, os_, nz)),
                ("_sm_key", (tuple(w), tuple(mu), tuple(v)),
                 lambda p: p.set_spectral(w, torch.tensor(mu).reshape(Q, -1), torch.tensor(v).reshape(Q, -1)))]


PERIODIC_MAX_DIMS = 16


class PeriodicKernelLinearOperator(KernelLinearOperator):
    """S exp(-2 sum_d sin^2(pi tau_d / p_d) / l_d), tau = x1 - x2 (kernels/periodic_kernel.py, which forms the dense matrix) as ONE
    engine plan (gp_plan_set_periodic).  The engine runs it as the RBF kernel of unit lengthscale over the embedding
    (cos, sin)(2 pi x_d / p_d) / sqrt(l_d), so products, solves, the preconditioner and SLQ run on the plain tensor-core path.
    lengthscale and period hold 1 or d values (the parameter tensors or their slices for one element of a batch); autograd reaches
    them through _bilinear_derivative_list.  S is the outputscale of a ScaleKernel around the kernel (None: 1, no gradient).
    1 <= d <= 16; gradients with respect to the inputs are not available."""

    _family = "periodic"
    _noun = "periodic"
    _factor = _input_grads = _row_sharding = False
    _params = ("lengthscale", "period")
    # set_periodic repacks the embedding: a cached plan keeps the setting its keys record, so a new operator over the same plan
    # with the same parameters packs nothing
    _resend_on_new_plan = False

    def __init__(self, x1, x2, lengthscale, period, outputscale=None, comm=None, row_begin=0, row_count=0):
        d = x1.size(-1)
        if not 1 <= d <= PERIODIC_MAX_DIMS:
            raise NotImplementedError(f"a periodic operator takes 1 <= d <= {PERIODIC_MAX_DIMS} input dimensions on the accelerated "
                                      f"path (got d = {d})")
        if lengthscale.numel() not in (1, d) or period.numel() not in (1, d):
            raise RuntimeError(f"periodic kernel: lengthscale {tuple(lengthscale.shape)} and period {tuple(period.shape)} must hold 1 "
                               f"or {d} values")
        if x1.requires_grad or (x2 is not None and x2.requires_grad):
            raise NotImplementedError("gradients with respect to the inputs of a periodic operator (deep kernel learning, test-input "
                                      "gradients) are not available on the accelerated path")
        super().__init__(x1, x2, "rbf", lengthscale, outputscale, comm=comm, row_begin=row_begin, row_count=row_count)
        self.period = period

    def _ctor_args(self):
        return (self.lengthscale, self.period)

    def _engine_calls(self, hyp, nz):
        ls, per, (os_,) = hyp
        return [("_per_key", tuple(per), lambda p: p.set_periodic(per)),
                ("_hyp_key", ("rbf", tuple(ls), os_, nz), lambda p: p.set_hypers("rbf", ls, os_, nz))]


class RQKernelLinearOperator(KernelLinearOperator):
    """S (1 + r^2 / (2 alpha))^-alpha, r^2 = |(x1 - x2) / l|^2 (kernels/rq_kernel.py, which forms the dense matrix) as ONE engine
    plan of kind GP_RQ (gp_plan_set_hypers_rq): products, solves, the preconditioner, SLQ, rows and input gradients run on the plain
    tensor-core / CUDA-core kernels with the RQ covariance in their epilogue.  lengthscale holds 1 or d values and alpha one (the
    parameter tensors or their slices for one element of a batch); autograd reaches them through _bilinear_derivative_list.  S is
    the outputscale of a ScaleKernel around the kernel (None: 1, no gradient).  The plan-cache slots are the plain ones (_slot)."""

    _family = "rq"
    _noun = "rational quadratic (RQ)"
    _factor = _row_sharding = False
    _params = ("lengthscale", "alpha")

    def __init__(self, x1, x2, lengthscale, alpha, outputscale=None, comm=None, row_begin=0, row_count=0):
        super().__init__(x1, x2, "rq", lengthscale, outputscale, comm=comm, row_begin=row_begin, row_count=row_count)
        if alpha.numel() != 1:
            raise RuntimeError(f"RQ kernel: alpha must hold one value (got shape {tuple(alpha.shape)})")
        self.alpha = alpha

    def _ctor_args(self):
        return (self.lengthscale, self.alpha)

    def _engine_calls(self, hyp, nz):
        ls, (al,), (os_,) = hyp
        return [("_hyp_key", ("rq", tuple(ls), al, os_, nz), lambda p: p.set_hypers_rq(ls, al, os_, nz))]


class PolynomialKernelLinearOperator(KernelLinearOperator):
    """S (x1 . x2 + c)^p (kernels/polynomial_kernel.py, which forms the dense matrix with addmm(...).pow(p)) as ONE engine plan of
    kind GP_POLY (gp_plan_set_hypers_poly) over the raw inputs: products, solves, the preconditioner, SLQ, rows and input gradients
    run on the plain tensor-core / CUDA-core kernels with (x . x' + c)^p in their epilogue.  power is a Python int in [1, 8], offset
    one value (the parameter tensor or its slice for one element of a batch); autograd reaches the offset and S through
    _bilinear_derivative_list.  The kernel is not stationary: diagonal() is S (|x_i|^2 + c)^p from the plan.  The plan-cache slots
    are the plain ones (_slot)."""

    _family = "poly"
    _noun = "PolynomialKernel"
    _factor = _row_sharding = False
    _params = ("offset",)

    def __init__(self, x1, x2, power, offset, outputscale=None, comm=None, row_begin=0, row_count=0):
        # no lengthscale: a constant stands in where the generic code reads one (device / dtype only)
        super().__init__(x1, x2, "poly", torch.ones((), device=x1.device, dtype=offset.dtype), outputscale, comm=comm,
                         row_begin=row_begin, row_count=row_count)
        if offset.numel() != 1:
            raise RuntimeError(f"polynomial kernel: offset must hold one value (got shape {tuple(offset.shape)})")
        self.power = int(power)
        self.offset = offset

    def _ctor_args(self):
        return (self.power, self.offset)

    def _engine_calls(self, hyp, nz):
        (off,), (os_,) = hyp
        return [("_hyp_key", ("poly", self.power, off, os_, nz), lambda p: p.set_hypers_poly(self.power, off, os_, nz))]


class PiecewisePolynomialKernelLinearOperator(KernelLinearOperator):
    """S (1 - r)_+^(j+q) poly_q(r), r = |(x1 - x2) / l|, j = floor(d / 2) + q + 1 (kernels/piecewise_polynomial_kernel.py, which forms
    the dense matrix) as ONE engine plan on the compact-support backend (gp_plan_set_hypers_pp): the points are kept in Morton order
    inside the engine and a product evaluates only the tile pairs within one lengthscale, so its cost follows the sparsity of K.
    Solves, the preconditioner, SLQ, rows, the diagonal, Lanczos and CIQ run on the plan as on a plain one.  q is a Python int in
    {0, 1, 2, 3}, lengthscale holds 1 or d values, S is the outputscale of a ScaleKernel around the kernel (None: 1, no gradient);
    autograd reaches the lengthscale and S through _bilinear_derivative_list.  Sums, products, multitask use, row sharding and
    gradients with respect to the inputs are refused."""

    _family = "ppoly"
    _noun = "PiecewisePolynomialKernel"
    _sum_term = _factor = _input_grads = _row_sharding = False

    def __init__(self, x1, x2, q, lengthscale, outputscale=None, comm=None, row_begin=0, row_count=0):
        super().__init__(x1, x2, "ppoly", lengthscale, outputscale, comm=comm, row_begin=row_begin, row_count=row_count)
        if torch.is_grad_enabled() and (x1.requires_grad or (x2 is not None and x2.requires_grad)):
            raise NotImplementedError("gradients with respect to the inputs of a PiecewisePolynomialKernel (deep kernel learning, "
                                      "posterior input gradients) are not available on the accelerated path")
        self.q = int(q)

    def _ctor_args(self):
        return (self.q, self.lengthscale)

    def _engine_calls(self, hyp, nz):
        ls, (os_,) = hyp
        return [("_hyp_key", ("ppoly", self.q, tuple(ls), os_, nz), lambda p: p.set_hypers_pp(self.q, ls, os_, nz))]


class SKIKernelLinearOperator(KernelLinearOperator):
    """K_ski = s W (T_0 x ... x T_{d-1}) W^T (kernels/grid_interpolation_kernel.py:132-213): the engine's SKI backend -- cubic
    interpolation weights kept in compact per-dimension form, Kronecker / Toeplitz grid covariance applied mode by mode."""

    _noun = "SKI"
    _sum_term = _factor = _single_plan = False

    def __init__(self, x1, kind, lengthscale, outputscale, grid_sizes, grid_lo, grid_step):
        super().__init__(x1, None, kind, lengthscale, outputscale)
        self.grid_sizes, self.grid_lo, self.grid_step = tuple(grid_sizes), tuple(grid_lo), tuple(grid_step)

    def plan(self, noise=0.0) -> Plan:
        if self._plan is None:
            key = "ski:" + repr((self.grid_sizes, self.grid_lo, self.grid_step))
            self._plan = _get_plan(self.x1, None, key, 0, 0, None, self._plan_slot, owner=self)
            if getattr(self._plan, "_ski_key", None) != key:
                self._plan.set_ski(self.grid_sizes, self.grid_lo, self.grid_step)
                self._plan._ski_key = key
                self._plan._hyp_key = None
        (ls, (os_,)), nz, _ = self._host_hypers(noise if torch.is_tensor(noise) else None)
        if not torch.is_tensor(noise):
            nz = float(noise)
        hk = (self.kind, tuple(ls), os_, nz)
        if getattr(self._plan, "_hyp_key", None) != hk:
            self._plan.set_hypers(self.kind, ls, os_, nz)
            self._plan._hyp_key = hk
        return self._plan

    def input_tensors(self):
        """No inputs: products, slices and the posterior paths of the interpolated operator stay detached from its inputs."""
        return []

    def solve_input_tensors(self):
        """[x1]: the MLL and solves reach the points through gp_ski_input_grad (deep kernel learning on KISS-GP)."""
        return [self.x1]

    def _input_grad_list(self, left, right, needs):
        """[dF/dx1] of F = sum(left * (K_ski @ right)) (gp_ski_input_grad), [None] when not needed."""
        if not any(needs):
            return [None] * len(needs)
        return [self.plan(getattr(self, "_last_noise", 0.0)).ski_input_grad(left, right)]

    def _dense_input_grad_list(self, w, needs):
        """[dF/dx1] of F = sum(w * K_ski): the product form with the identity, n columns.  Only the Cholesky branch of the solves
        (n <= max_cholesky_size) asks for it; the engine has no dense SKI block."""
        if not any(needs):
            return [None] * len(needs)
        return self._input_grad_list(w, torch.eye(w.size(0), device=w.device, dtype=w.dtype), needs)

    def detach(self):
        return SKIKernelLinearOperator(self.x1, self.kind, self.lengthscale.detach(), self.outputscale.detach(), self.grid_sizes,
                                       self.grid_lo, self.grid_step)

    def with_outputscale(self, outputscale):
        return SKIKernelLinearOperator(self.x1, self.kind, self.lengthscale, outputscale, self.grid_sizes, self.grid_lo, self.grid_step)

    def to_dense(self):
        n = self.x1.size(0)
        eye = torch.eye(n, device=self.device, dtype=torch.float32)
        return torch.cat([self.plan().kmv(eye[:, c0:c0 + 16].contiguous()) for c0 in range(0, n, 16)], -1)

    def diagonal(self, dim1=-2, dim2=-1):
        """s w_i^T K_uu w_i per row (gp_kdiag on the SKI plan): not constant, unlike a stationary kernel's."""
        return self.plan().diag()

    _diagonal = diagonal

    def same_grid(self, other) -> bool:
        """other is a SKI operator on the same grid with the same kind and hyper-parameter values: its points interpolate the
        same K_uu, so the grid caches of one operator serve the other (models._ski_grid_mode)."""
        if type(other) is not type(self):
            return False
        if (self.grid_sizes, self.grid_lo, self.grid_step, self.kind) != (other.grid_sizes, other.grid_lo, other.grid_step, other.kind):
            return False
        return (self.lengthscale.shape == other.lengthscale.shape and bool(torch.equal(self.lengthscale.detach(), other.lengthscale.detach()))
                and bool(torch.equal(self.outputscale.detach().reshape(-1), other.outputscale.detach().reshape(-1))))

    def grid_matmul(self, rhs):
        """s K_uu W^T rhs: rhs [n] or [n, t] over this operator's points -> [M] or [M, t] on the grid (gp_ski_grid_matmul; the
        caches c = s K_uu W^T alpha and C = s K_uu W^T R of the reference's InterpolatedPredictionStrategy).  Detached."""
        return self.plan().ski_grid_matmul(rhs.detach().float())

    def interp_matmul(self, grid):
        """W grid: grid values [M] or [M, t] interpolated to this operator's points (gp_ski_interp_matmul; the reference's
        left_interp).  Detached."""
        return self.plan().ski_interp_matmul(grid.detach().float())

    def __getitem__(self, index):
        """Rows / columns of the interpolated operator: K[r, c] = W[r] K_uu W[c]^T (the reference slices the interpolation
        indices / values of InterpolatedLinearOperator).  Used by the prediction strategy on the joint train + test operator."""
        if not isinstance(index, tuple):
            index = (index, slice(None))
        ri, ci = index
        n = self.x1.size(0)
        ar = torch.arange(n, device=self.device)
        rows = ar[ri].reshape(-1)
        cols = ar[ci].reshape(-1)
        sub = _SKISliceOperator(self, rows, cols)
        return sub.to_dense()[0] if isinstance(ri, int) else sub


class _SKISliceOperator:
    """K_ski[rows, cols] of a square SKI operator, never materialised: a product zero-pads the right-hand side to the full point
    set, runs the parent's scatter / mode products / gather, and keeps the requested rows (evaluation mode: no autograd)."""

    def __init__(self, parent, rows, cols):
        self.parent, self.rows, self.cols = parent, rows, cols

    @property
    def shape(self):
        return torch.Size([self.rows.numel(), self.cols.numel()])

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    @property
    def device(self):
        return self.parent.device

    @property
    def dtype(self):
        return self.parent.dtype

    def evaluate_kernel(self):
        return self

    def _transpose_nonbatch(self):
        return _SKISliceOperator(self.parent, self.cols, self.rows)      # the parent is symmetric

    t = _transpose_nonbatch

    def transpose(self, dim1, dim2):
        return self if dim1 % 2 == dim2 % 2 else self._transpose_nonbatch()

    def matmul(self, rhs):
        vec = rhs.dim() == 1
        r2 = (rhs.unsqueeze(-1) if vec else rhs).detach().float()
        if r2.size(0) != self.cols.numel():
            raise RuntimeError(f"LinearOperator (size={tuple(self.shape)}) cannot be multiplied with right-hand-side Tensor "
                               f"(size={tuple(rhs.shape)})")
        plan = self.parent.plan(getattr(self.parent, "_last_noise", 0.0))
        outs = []
        for c0 in range(0, r2.size(1), 16):
            full = torch.zeros(self.parent.x1.size(0), min(16, r2.size(1) - c0), device=self.device)
            full[self.cols] = r2[:, c0:c0 + 16]
            outs.append(plan.kmv(full)[self.rows])
        out = outs[0] if len(outs) == 1 else torch.cat(outs, -1)
        return out.squeeze(-1) if vec else out

    __matmul__ = matmul
    _matmul = matmul

    def to_dense(self):
        return self.matmul(torch.eye(self.cols.numel(), device=self.device))


LOWRANK_MAX_RANK = 128


class LowRankUpdatedKernelLinearOperator(_SamplingMixin):
    """K** - U U^T kept lazy: the LOVE posterior covariance K** - K*x R R^T Kx* with U = K*x R [m, J] (the reference's
    `test_test_covar + MatmulLinearOperator(root, -root^T)`, models/exact_prediction_strategies.py:464-478).  Every product,
    diagonal and row runs on the engine plan of K** with the correction as one more partial slot (csrc/lowrank.cu), so nothing
    m x m exists unless to_dense() is asked for.

    `base` is a plan-backed square KernelLinearOperator or SumKernelLinearOperator (not SKI, not row-sharded), 1 <= J <= 128.  The
    operator has its own plan-cache slot and sets U on that plan whenever U's storage or version changes.  It is detached: it
    exposes no hyper-parameter tensors (gradients still reach the posterior mean and the right-hand side of log_prob).  No
    preconditioner is built for it (AddedDiagLinearOperator._preconditioner returns none).

    Sampling is _SamplingMixin's: CIQ with settings.ciq_samples, the dense psd-safe Cholesky up to max_cholesky_size, else a device
    Lanczos root.  For the observed posterior K** - U U^T + sigma^2 I the CIQ interval starts at the noise floor sigma^2 (min d_i
    for a per-row diagonal).  That floor is valid because the LOVE posterior dominates the exact one: R R^T = Q (Q^T K_hat Q)^-1 Q^T
    <= K_hat^-1 for the Lanczos basis Q of K_hat = K_xx + D, hence K** - K*x R R^T Kx* >= K** - K*x K_hat^-1 Kx* >= 0.  The
    noise-free latent posterior has no floor and falls back to the Ritz interval."""

    def __init__(self, base, U: torch.Tensor):
        if not self.supports(base):
            raise RuntimeError("LowRankUpdatedKernelLinearOperator needs a square, unsharded, plan-backed kernel operator or "
                               "kernel sum (not SKI)")
        self._setup(base, U)

    def _setup(self, base, U):
        if U.dim() != 2 or U.size(0) != base.shape[0] or not 1 <= U.size(1) <= LOWRANK_MAX_RANK:
            raise RuntimeError(f"low-rank factor must be [{base.shape[0]}, r] with 1 <= r <= {LOWRANK_MAX_RANK} (got {tuple(U.shape)})")
        self.base = base.detach()
        self.base._plan_slot = _slot(self.base._family, "lowrank")   # a plan carrying U never serves an operator without it
        self.U = U.detach().float().contiguous()

    @classmethod
    def on_ski(cls, base, U: torch.Tensor):
        """K**_test - U U^T on a standalone SKI operator, i.e. one whose plan is over the test points only (the KISS-GP grid
        prediction of models.ExactGP, settings.ski_grid_prediction).  The SKI plan takes the correction like any other backend.
        Kept out of supports() / the default constructor: the joint path's SKI blocks are slices of a train + test operator."""
        if type(base) is not SKIKernelLinearOperator:
            raise RuntimeError("LowRankUpdatedKernelLinearOperator.on_ski needs a standalone SKIKernelLinearOperator")
        op = cls.__new__(cls)
        op._setup(base, U)
        return op

    @staticmethod
    def supports(base) -> bool:
        """A plan-backed non-SKI kernel operator (or kernel sum) without batch dimension on an unsharded square plan."""
        return (isinstance(base, KernelLinearOperator)
                and (base._single_plan or isinstance(base, (SumKernelLinearOperator, AdditiveKernelLinearOperator)))
                and base.same
                and base._comm is None and base._row_begin == 0 and base._row_count in (0, base.shape[0]))

    def plan(self, noise=0.0) -> Plan:
        p = self.base.plan(noise)
        cur = getattr(p, "_lowrank", None)
        if cur is None or cur.data_ptr() != self.U.data_ptr() or cur.shape != self.U.shape or p._lowrank_version != self.U._version:
            p.set_lowrank(self.U)
            p._lowrank_version = self.U._version
        return p

    def _sampling_plan(self) -> Plan:
        """The plan of K** - U U^T alone: no noise, no per-row diagonal left over from an earlier + D."""
        p = self.plan(0.0)
        if getattr(p, "_noise_diag", None) is not None:
            p.set_noise_diag(None)
        return p

    def _any_plan(self) -> Plan:
        return self.plan(getattr(self, "_last_noise", 0.0))   # products / rows / diagonal ignore the plan's noise

    @property
    def shape(self):
        return self.base.shape

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    @property
    def dtype(self):
        return self.base.dtype

    @property
    def device(self):
        return self.base.device

    @property
    def batch_shape(self):
        return torch.Size([])

    @property
    def matrix_shape(self):
        return self.shape

    def _size(self):
        return self.shape

    def dim(self):
        return 2

    ndimension = dim

    def numel(self):
        return self.shape[0] * self.shape[1]

    @property
    def requires_grad(self):
        return False

    def evaluate_kernel(self):
        return self

    def representation(self):
        return (self.U,)

    def hyper_tensors(self):
        return []

    def solve_input_tensors(self):
        return []

    def _bilinear_derivative_list(self, left, right):
        return []

    def transpose(self, dim1, dim2):
        return self          # symmetric

    def t(self):
        return self

    _transpose_nonbatch = t

    @property
    def mT(self):
        return self

    def detach(self):
        return self

    def matmul(self, rhs):
        return _LowRankMatmul.apply(self, rhs)

    __matmul__ = matmul
    _matmul = matmul

    def diagonal(self, dim1=-2, dim2=-1):
        """diag(K**) - sum_j U_ij^2 (gp_kdiag on the low-rank plan)."""
        return self._any_plan().diag()

    _diagonal = diagonal

    def to_dense(self):
        """Rows of K** - U U^T (gp_krows on the low-rank plan): the m x m matrix, for the dense branch only."""
        p = self._any_plan()
        return p.rows(torch.arange(self.shape[0], device=self.device))

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):
            return AddedDiagLinearOperator(self, other)
        raise NotImplementedError("LowRankUpdatedKernelLinearOperator only adds a (Constant)DiagLinearOperator")

    def _with_zero_diag(self):
        return AddedDiagLinearOperator(self, ConstantDiagLinearOperator(torch.zeros((), device=self.device), self.shape[0]))

    def inv_quad_logdet(self, inv_quad_rhs=None, logdet=False, reduce_inv_quad=True):
        """log_prob of the latent (noise-free) posterior: the solves of K** - U U^T itself -- the dense Cholesky up to
        max_cholesky_size, else unpreconditioned mBCG + SLQ -- as a dense posterior covariance gets them from its Cholesky
        factor.  The latent posterior can be close to singular; likelihood(post) adds the noise."""
        return self._with_zero_diag().inv_quad_logdet(inv_quad_rhs, logdet=logdet, reduce_inv_quad=reduce_inv_quad)

    def solve(self, rhs, lhs=None):
        return self._with_zero_diag().solve(rhs, lhs)

    def add_jitter(self, jitter_val=1e-3):
        return AddedDiagLinearOperator(self, ConstantDiagLinearOperator(torch.tensor(jitter_val, device=self.device), self.shape[0]))


class _LowRankMatmul(torch.autograd.Function):
    """(K** - U U^T) rhs; the operator is symmetric and detached, so only the right-hand side gets a gradient."""

    @staticmethod
    def forward(ctx, op, rhs):
        ctx.op = op
        return op._any_plan().kmv(rhs.detach().float())

    @staticmethod
    def backward(ctx, grad_out):
        return None, ctx.op._any_plan().kmv(grad_out.contiguous())


class _KernelMatmul(torch.autograd.Function):
    """K @ rhs.  Takes the operator's hyper_tensors() and then its input_tensors(): the backward returns the hyper-parameter
    gradients (gp_bilinear_grad) and the input gradients (gp_kmv_input_grad, one call per term of a kernel sum) only for the
    tensors whose gradient autograd asks for."""

    @staticmethod
    def forward(ctx, op, rhs, *tensors):
        ctx.op = op
        ctx.nh = len(op.hyper_tensors())
        out = op.plan(getattr(op, "_last_noise", 0.0)).kmv(rhs.detach())
        ctx.save_for_backward(rhs.detach())
        return out

    @staticmethod
    def backward(ctx, grad_out):
        op = ctx.op
        (rhs,) = ctx.saved_tensors
        g = grad_out.contiguous()
        vec = g.dim() == 1
        g2 = g.unsqueeze(-1) if vec else g
        r2 = rhs.unsqueeze(-1) if vec else rhs
        grad_rhs = None
        nh = ctx.nh
        grads = [None] * nh
        need_h, need_x = ctx.needs_input_grad[2:2 + nh], ctx.needs_input_grad[2 + nh:]
        if ctx.needs_input_grad[1]:
            # K^T g: for x1 == x2 the operator is symmetric
            if not op.same:
                grad_rhs = op._transpose_nonbatch().plan().kmv(g)
            else:
                grad_rhs = op.plan(getattr(op, "_last_noise", 0.0)).kmv(g)
        if any(need_h):
            gs = op._bilinear_derivative_list(g2, r2)
            grads = [gi if need else None for gi, need in zip(gs, need_h)]
        return (None, grad_rhs, *grads, *op._input_grad_list(g2, r2, need_x))


class _KernelDense(torch.autograd.Function):
    """K(x1, x2) as a dense block (gp_krows; the local rows of a row-sharded plan) whose backward reaches the input tensors
    (gp_kdense_input_grad).  Hyper-parameter gradients through to_dense() are not implemented: the block is detached from the
    lengthscale and outputscale, as it always was."""

    @staticmethod
    def forward(ctx, op, *inputs):
        ctx.op = op
        p = op.plan()
        return p.rows(torch.arange(p.row_count, device=op.device))

    @staticmethod
    def backward(ctx, grad):
        return (None, *ctx.op._dense_input_grad_list(grad.contiguous(), ctx.needs_input_grad[1:]))


class AddedDiagLinearOperator(_SamplingMixin):
    """K + D with the BBMM solves (linear_operator AddedDiagLinearOperator): D = sigma^2 I (constant-diagonal branch, Appendix
    A.4) or a per-row diagonal (FixedNoiseGaussianLikelihood; the non-constant-diagonal branch of the preconditioner)."""

    def __init__(self, kernel_op: KernelLinearOperator, diag):
        if kernel_op.shape[0] != kernel_op.shape[1]:
            raise RuntimeError("AddedDiagLinearOperator needs a square operator")
        self.kernel_op = kernel_op
        self.diag = diag
        self.per_row = isinstance(diag, DiagLinearOperator)
        self._precond_cache = None

    @property
    def noise(self) -> torch.Tensor:
        """sigma^2 (0-d) for the constant diagonal, the vector d [n] for a per-row diagonal."""
        return self.diag.diag_vec if self.per_row else self.diag.diag_value.reshape(())

    @property
    def _noise_param(self) -> torch.Tensor:
        return self.diag.diag_vec if self.per_row else self.diag.diag_value

    def _noise_col(self):
        return self.diag.diag_vec.unsqueeze(-1) if self.per_row else self.noise

    @property
    def shape(self):
        return self.kernel_op.shape

    def size(self, dim=None):
        return self.kernel_op.size(dim)

    @property
    def dtype(self):
        return self.kernel_op.dtype

    @property
    def device(self):
        return self.kernel_op.device

    @property
    def batch_shape(self):
        return torch.Size([])

    def evaluate_kernel(self):
        return self

    def _plan(self) -> Plan:
        if self.per_row:
            p = self.kernel_op.plan(0.0)
            d = self.diag.diag_vec.detach().float().contiguous()
            if getattr(p, "_noise_diag", None) is None or p._noise_diag.data_ptr() != d.data_ptr() or p._noise_diag_version != d._version:
                p.set_noise_diag(d)
                p._noise_diag_version = d._version
            self.kernel_op._last_noise = 0.0
            return p
        p = self.kernel_op.plan(self.diag.diag_value)
        if getattr(p, "_noise_diag", None) is not None:   # a cached plan last used with a per-row diagonal
            p.set_noise_diag(None)
        self.kernel_op._last_noise = p.noise
        return p

    def _sampling_plan(self) -> Plan:
        return self._plan()

    def _noise_floor(self):
        return float(self.diag.diag_vec.detach().min()) if self.per_row else float(self.diag.diag_value.detach().reshape(-1)[0])

    def matmul(self, rhs):
        d = self._noise_col() if (self.per_row and rhs.dim() > 1) else self.noise
        return self.kernel_op.matmul(rhs) + d * rhs

    __matmul__ = matmul
    _matmul = matmul

    # -- LinearOperator protocol subset the callers use (SURVEY.md section 8b "Operator seam") --
    def _size(self):
        return self.shape

    @property
    def matrix_shape(self):
        return self.shape

    def dim(self):
        return 2

    ndimension = dim

    def numel(self):
        return self.shape[0] * self.shape[1]

    @property
    def requires_grad(self):
        return bool(self.kernel_op.requires_grad or self._noise_param.requires_grad)

    def representation(self):
        return self.kernel_op.representation() + (self._noise_param,)

    def transpose(self, dim1, dim2):
        return self          # K + sigma^2 I is symmetric

    def t(self):
        return self

    _transpose_nonbatch = t

    @property
    def mT(self):
        return self

    def detach(self):
        d = DiagLinearOperator(self.diag.diag_vec.detach()) if self.per_row else ConstantDiagLinearOperator(self.diag.diag_value.detach(), self.shape[0])
        return AddedDiagLinearOperator(self.kernel_op.detach(), d)

    def __add__(self, other):
        if isinstance(other, (ConstantDiagLinearOperator, DiagLinearOperator)):   # (K + D1) + D2
            return AddedDiagLinearOperator(self.kernel_op, self.diag + other)
        raise NotImplementedError("AddedDiagLinearOperator only adds a (Constant)DiagLinearOperator")

    def logdet(self):
        return self.inv_quad_logdet(None, logdet=True)[1]

    def inv_quad(self, inv_quad_rhs, reduce_inv_quad=True):
        return self.inv_quad_logdet(inv_quad_rhs, logdet=False, reduce_inv_quad=reduce_inv_quad)[0]

    def to_dense(self):
        return self.kernel_op.to_dense() + self.diag.to_dense()

    def diagonal(self, dim1=-2, dim2=-1):
        return self.kernel_op.diagonal() + self.noise

    _diagonal = diagonal

    def add_jitter(self, jitter_val=1e-3):
        jit = ConstantDiagLinearOperator(torch.as_tensor(jitter_val, device=self.device, dtype=self.dtype), self.shape[0])
        return AddedDiagLinearOperator(self.kernel_op, self.diag + jit)

    # -- preconditioner (AddedDiagLinearOperator._preconditioner, Appendix A.4) --
    def _preconditioner(self):
        """Returns (W [n,k] | None, Lt [k,n] | None, logdet_P)."""
        n = self.shape[0]
        if settings.max_preconditioner_size.value() == 0 or n < settings.min_preconditioning_size.value():
            return None, None, 0.0
        if isinstance(self.kernel_op, LowRankUpdatedKernelLinearOperator):
            return None, None, 0.0           # no pivoted Cholesky of a downdated operator (the engine refuses it)
        if isinstance(self.kernel_op, SKIKernelLinearOperator) and settings.ski_preconditioner.off():
            # Off by default so that existing SKI results do not change; whether the reference preconditions interpolated
            # operators (linear_operator, absent here) is not established.  settings.ski_preconditioner documents the choice.
            return None, None, 0.0
        if self._precond_cache is None:
            p = self._plan()
            lt, piv, st = p.pivoted_cholesky(settings.max_preconditioner_size.value(), settings.preconditioner_tolerance.value())
            if st != 0 or lt.size(0) == 0:
                self._precond_cache = (None, None, 0.0)
            else:
                w, logdet, st2 = p.precond_build(lt)
                self._precond_cache = (None, None, 0.0) if st2 != 0 else (w, lt, logdet)
        return self._precond_cache

    def _ciq_precond(self):
        """The split factor of the solves' preconditioner P = L L^T + D, built from the Lt of _preconditioner() (no second pivoted
        Cholesky) and rebuilt whenever that cache is.  Interval: 1 <= lambda(F^-1 K_hat F^-T) <= 1 + tr(K - L L^T) / min d; the
        bounds used are [1/2, 2 (1 + max(tr, 1e-6 tr K) / min d)], the margins absorbing the fp32 rounding of L."""
        cache = self._preconditioner()
        lt = cache[1]
        if lt is None:
            return None
        if getattr(self, "_ciq_cache", None) is None or self._ciq_cache[0] is not cache:
            u, tr_e, st = self._plan().ciq_precond_build(lt)
            if st != 0:
                self._ciq_cache = (cache, None)
            else:
                tr_k = tr_e + float(lt.double().square().sum())
                self._ciq_cache = (cache, (u, 0.5, 2.0 * (1.0 + max(tr_e, 1e-6 * tr_k) / self._noise_floor())))
        return self._ciq_cache[1]

    def _probes(self, lt, tp):
        n = self.shape[0]
        seed = settings.probe_seed.value()
        if seed is None and settings.deterministic_probes.on():
            seed = settings.deterministic_probes.seed       # one set of base samples for every estimate while the flag is on
        gen = None
        if seed is not None:
            gen = torch.Generator(device=self.device).manual_seed(int(seed))
        if lt is None:
            z = torch.randint(0, 2, (n, tp), device=self.device, generator=gen).to(torch.float32) * 2 - 1
            return z
        eps1 = torch.randn(lt.size(0), tp, device=self.device, generator=gen)
        eps2 = torch.randn(n, tp, device=self.device, generator=gen)
        return self._plan().precond_probes(lt, eps1, eps2)

    def _dense_cholesky(self):
        return torch.linalg.cholesky(self.to_dense())

    def solve(self, rhs, lhs=None):
        """K_hat^{-1} rhs by preconditioned CG (LinearOperator.solve -> linear_cg, n_tridiag = 0)."""
        out = _Solve.apply(self, rhs, self._noise_param, *self.kernel_op.hyper_tensors(), *self.kernel_op.solve_input_tensors())
        return out if lhs is None else lhs @ out

    def inv_quad_logdet(self, inv_quad_rhs=None, logdet=False, reduce_inv_quad=True):
        """(rhs^T K_hat^{-1} rhs, log det K_hat): distributions/multivariate_normal.py:249."""
        if inv_quad_rhs is not None and inv_quad_rhs.size(0) != self.shape[0]:
            raise RuntimeError(
                f"LinearOperator (size={tuple(self.shape)}) cannot be multiplied with right-hand-side Tensor "
                f"(size={tuple(inv_quad_rhs.shape)})")
        rhs = inv_quad_rhs
        if rhs is not None and rhs.dim() == 1:
            rhs = rhs.unsqueeze(-1)
        iq, ld = _InvQuadLogdet.apply(self, rhs, bool(logdet), self._noise_param, *self.kernel_op.hyper_tensors(),
                                      *self.kernel_op.solve_input_tensors())
        if rhs is None:
            iq = torch.empty(0, device=self.device)
        elif reduce_inv_quad:
            iq = iq.sum(-1)
        return iq, (ld if logdet else None)

    def root_inv_decomposition(self, initial_vectors=None):
        """Lanczos root of K_hat^{-1}: R with R R^T ~= K_hat^{-1} (exact_prediction_strategies.py:268-272)."""
        n = self.shape[0]
        if settings.fast_computations.covar_root_decomposition.off():
            # exact root through the dense Cholesky factor: K_hat = L L^T  =>  K_hat^{-1} = L^{-T} L^{-1}
            chol = self._dense_cholesky()
            return torch.linalg.solve_triangular(chol.transpose(-1, -2), torch.eye(n, device=self.device, dtype=chol.dtype), upper=True)
        p = self._plan()
        init = initial_vectors if initial_vectors is not None else torch.randn(n, device=self.device)
        if init.dim() == 2:
            init = init[:, 0]
        q, t = p.lanczos(init.float(), settings.max_root_decomposition_size.value())
        evals, evecs = torch.linalg.eigh(t.double())      # J x J, J <= 100: plumbing-sized
        mask = evals >= 0                                 # lanczos_tridiag_to_diag masks negative Ritz values
        evecs = evecs * mask
        evals = evals.masked_fill(~mask, 1.0)
        return (q.double() @ (evecs / evals.sqrt())).float()


class BatchLinearOperator:
    """One leading batch dimension of independent operators (BASELINE config 4: batch = 16, independent hyper-parameters per
    element; the reference broadcasts every LinearOperator op over leading dims, kernels/kernel.py:119-121,
    distributions/multivariate_normal.py:236-245).  Each element owns an engine plan on its own CUDA stream; solver calls
    (inv_quad_logdet / solve) of all elements run concurrently from a thread pool (the C ABI releases the GIL), so the small
    per-element grids and launch chains overlap on the device."""

    _pool = None

    def __init__(self, ops):
        self.ops = list(ops)
        first = self.ops[0]
        self._mshape = first.shape

    @property
    def batch_shape(self):
        return torch.Size([len(self.ops)])

    @property
    def shape(self):
        return torch.Size([len(self.ops), *self._mshape])

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    @property
    def device(self):
        return self.ops[0].device

    @property
    def dtype(self):
        return self.ops[0].dtype

    def evaluate_kernel(self):
        return self

    def __getitem__(self, b):
        return self.ops[b]

    def __add__(self, other):
        # batched homoskedastic noise: ConstantDiagLinearOperator with diag_value [B, 1]
        if isinstance(other, ConstantDiagLinearOperator):
            dv = other.diag_value
            outs = []
            for b, op in enumerate(self.ops):
                d_b = dv[b] if dv.dim() >= 2 or (dv.dim() == 1 and dv.numel() == len(self.ops) and dv.numel() > 1) else dv
                outs.append(op + ConstantDiagLinearOperator(d_b.reshape(-1)[:1], other.n))
            return BatchLinearOperator(outs)
        if isinstance(other, DiagLinearOperator):
            dv = other.diag_vec
            return BatchLinearOperator([op + DiagLinearOperator(dv[b] if dv.dim() == 2 else dv) for b, op in enumerate(self.ops)])
        raise NotImplementedError("BatchLinearOperator only adds a (Constant)DiagLinearOperator")

    def _map(self, fn):
        """Run fn(b, op) for every element concurrently, element b on its own stream."""
        import concurrent.futures as cf

        B = len(self.ops)
        dev = self.device
        main = torch.cuda.current_stream(dev)
        streams = _batch_streams(dev, B)
        grad = torch.is_grad_enabled()
        ctxs = settings.snapshot()

        def work(b):
            with torch.cuda.device(dev), torch.cuda.stream(streams[b]), torch.set_grad_enabled(grad), settings.restore(ctxs):
                return fn(b, self.ops[b])

        for st in streams:
            st.wait_stream(main)
        if BatchLinearOperator._pool is None:
            BatchLinearOperator._pool = cf.ThreadPoolExecutor(max_workers=16, thread_name_prefix="gpbatch")
        outs = list(BatchLinearOperator._pool.map(work, range(B)))
        for st in streams:
            main.wait_stream(st)
        return outs

    def matmul(self, rhs):
        return torch.stack(self._map(lambda b, op: op.matmul(rhs[b] if rhs.dim() == 3 else rhs)))

    def zero_mean_mvn_samples(self, num_samples: int) -> torch.Tensor:
        """[num_samples, B, n]: every element samples concurrently on its own stream; the base samples are drawn here, in element
        order, so that a reseeded generator reproduces them."""
        n = self._mshape[-1]
        if settings.ciq_samples.on():
            xi = torch.randn(len(self.ops), n, num_samples, device=self.device)
            outs = self._map(lambda b, op: op._ciq_samples(xi[b])[0])
            return torch.stack(outs).permute(2, 0, 1)
        root = self.root_decomposition().root
        eps = torch.randn(len(self.ops), root.size(-1), num_samples, device=root.device, dtype=root.dtype)
        return (root @ eps).permute(2, 0, 1)

    def root_decomposition(self, method=None) -> RootLinearOperator:
        """Stacked roots [B, n, r]; Lanczos roots of different ranks are padded with zero columns."""
        roots = self._map(lambda b, op: op.root_decomposition(method).root)
        r = max(x.size(-1) for x in roots)
        return RootLinearOperator(torch.stack([torch.nn.functional.pad(x, (0, r - x.size(-1))) for x in roots]))

    __matmul__ = matmul

    def diagonal(self, dim1=-2, dim2=-1):
        return torch.stack([op.diagonal() for op in self.ops])

    def to_dense(self):
        return torch.stack([op.to_dense() for op in self.ops])

    def sum(self, dim=-3):
        """sum_b K_b over the batch dimension as ONE engine operator: the additive GP of D one-dimensional RBF / Matern components
        (AdditiveKernelLinearOperator with max_degree 1).  Only the batch dimension (-3 or 0) is summed."""
        if dim not in (-3, 0):
            raise NotImplementedError(f"BatchLinearOperator.sum(dim={dim}): only the batch dimension (-3 or 0) is summed on the "
                                      "accelerated path")
        return AdditiveKernelLinearOperator(_additive_components(self.ops, "BatchLinearOperator.sum"), 1)

    def solve(self, rhs, lhs=None):
        return torch.stack(self._map(lambda b, op: op.solve(rhs[b] if rhs.dim() >= 2 and rhs.size(0) == len(self.ops) else rhs)))

    def inv_quad_logdet(self, inv_quad_rhs=None, logdet=False, reduce_inv_quad=True):
        def one(b, op):
            r = None if inv_quad_rhs is None else inv_quad_rhs[b]
            return op.inv_quad_logdet(r, logdet=logdet, reduce_inv_quad=reduce_inv_quad)

        outs = self._map(one)
        iq = torch.stack([o[0] for o in outs])
        ld = torch.stack([o[1] for o in outs]) if logdet else None
        return iq, ld


_BATCH_STREAMS = {}


def _batch_streams(dev, n):
    key = str(dev)
    pool = _BATCH_STREAMS.setdefault(key, [])
    while len(pool) < n:
        pool.append(torch.cuda.Stream(dev))
    return pool[:n]


def _cg_tolerance():
    return settings.eval_cg_tolerance.value() if settings._use_eval_tolerance.on() else settings.cg_tolerance.value()


def _run_cg(op: AddedDiagLinearOperator, rhs, n_tridiag, w):
    """linear_cg over <= 16 columns per call."""
    p = op._plan()
    outs, tmat, iters = [], None, 0
    max_iter = settings.max_cg_iterations.value()
    if settings.terminate_cg_by_size.on():
        max_iter = min(max_iter, op.shape[0])
    for c0 in range(0, rhs.size(1), 16):
        blk = rhs[:, c0 : c0 + 16].contiguous()
        nt = n_tridiag if c0 == 0 else 0
        s, tm, info = p.mbcg(blk, nt, _cg_tolerance(), max_iter,
                             settings.max_lanczos_quadrature_iterations.value(), w)
        outs.append(s)
        iters = max(iters, info.iters)
        if nt:
            tmat = tm
    if settings.verbose_linalg.on():
        settings.verbose_linalg.logger.debug(
            f"Running CG on a {tuple(rhs.shape)} RHS for {iters} iterations (tol={_cg_tolerance()}). Output: {tuple(rhs.shape)}.")
    return (outs[0] if len(outs) == 1 else torch.cat(outs, -1)), tmat, iters


def _dense_branch(n: int, fast_flag) -> bool:
    """The reference's Cholesky branch: small systems (max_cholesky_size) or the Krylov path switched off (fast_computations)."""
    dense = n <= settings.max_cholesky_size.value() or fast_flag.off()
    if dense and settings.verbose_linalg.on():
        settings.verbose_linalg.logger.debug(f"Running Cholesky on a matrix of size {(n, n)}.")
    return dense


class _Solve(torch.autograd.Function):
    """K_hat^{-1} rhs.  Takes the kernel operator's hyper_tensors() and then its solve_input_tensors(); the backward asks the
    engine for the input gradients autograd needs with the factors of the hyper-parameter backward, (-K_hat^-1 g, solve)."""

    @staticmethod
    def forward(ctx, op, rhs, noise, *tensors):
        ctx.nh = len(op.kernel_op.hyper_tensors())
        vec = rhs.dim() == 1
        r2 = (rhs.unsqueeze(-1) if vec else rhs).detach().float().contiguous()
        n = op.shape[0]
        ctx.dense = _dense_branch(n, settings.fast_computations.solves)
        if ctx.dense:
            chol = op._dense_cholesky()
            sol = torch.cholesky_solve(r2, chol)
        else:
            w, _, _ = op._preconditioner()
            sol, _, _ = _run_cg(op, r2, 0, w)
        ctx.op, ctx.vec = op, vec
        ctx.save_for_backward(sol)
        return sol.squeeze(-1) if vec else sol

    @staticmethod
    def backward(ctx, grad_out):
        op = ctx.op
        (sol,) = ctx.saved_tensors
        g = (grad_out.unsqueeze(-1) if ctx.vec else grad_out).contiguous()
        if ctx.dense:
            gsol = torch.cholesky_solve(g, op._dense_cholesky())
        else:
            w, _, _ = op._preconditioner()
            gsol, _, _ = _run_cg(op, g, 0, w)
        grad_rhs = (gsol.squeeze(-1) if ctx.vec else gsol) if ctx.needs_input_grad[1] else None
        gn = None
        need_h, need_x = ctx.needs_input_grad[3:3 + ctx.nh], ctx.needs_input_grad[3 + ctx.nh:]
        grads = [None] * ctx.nh
        if any(ctx.needs_input_grad[2:3 + ctx.nh]):
            if any(need_h):
                gs = op.kernel_op._bilinear_derivative_list(-gsol, sol)
                grads = [gi if need else None for gi, need in zip(gs, need_h)]
            if ctx.needs_input_grad[2]:
                gn = (-(gsol * sol).sum(-1)) if op.per_row else (-(gsol * sol).sum()).reshape(op.diag.diag_value.shape)
        xgrads = op.kernel_op._input_grad_list((-gsol).contiguous(), sol, need_x) if any(need_x) else [None] * len(need_x)
        return (None, grad_rhs, gn, *grads, *xgrads)


class _InvQuadLogdet(torch.autograd.Function):
    """linear_operator.functions._inv_quad_logdet.InvQuadLogdet (SURVEY.md Appendix A.5).  Takes the kernel operator's
    hyper_tensors() and then its solve_input_tensors().  The input gradients use the left / right factors of the hyper-parameter
    backward on the CG branch, and the dense weight W = -sol diag(grad_iq) sol^T + grad_ld K_hat^-1 on the Cholesky branch."""

    @staticmethod
    def forward(ctx, op, rhs, want_logdet, noise, *tensors):
        ctx.nh = len(op.kernel_op.hyper_tensors())
        n = op.shape[0]
        dev = op.device
        ctx.op, ctx.want_logdet, ctx.has_rhs = op, want_logdet, rhs is not None
        nr = 0 if rhs is None else rhs.size(1)
        r = None if rhs is None else rhs.detach().float().contiguous()
        if _dense_branch(n, settings.fast_computations.log_prob):  # the reference's dense branch (not the accelerated path)
            chol = op._dense_cholesky()
            sol = torch.cholesky_solve(r, chol) if r is not None else None
            iq = (sol * r).sum(-2) if r is not None else torch.zeros(0, device=dev)
            ld = 2 * chol.diagonal().log().sum() if want_logdet else torch.zeros((), device=dev)
            ctx.mode = "chol"
            ctx.save_for_backward(chol, sol if sol is not None else torch.zeros(0, device=dev))
            return iq, ld
        ctx.mode = "cg"
        w, lt, logdet_p = op._preconditioner()
        tp = settings.num_trace_samples.value() if (want_logdet or op.kernel_op.requires_grad or noise.requires_grad) else 0
        cols = []
        probes = None
        if tp:
            probes = op._probes(lt, tp)
            norms = probes.norm(2, dim=-2, keepdim=True)
            cols.append(probes / norms)
        if r is not None:
            cols.append(r)
        full = torch.cat(cols, -1)
        solves, tmat, iters = _run_cg(op, full, tp, w)
        ld = torch.zeros((), device=dev)
        if want_logdet and settings.skip_logdet_forward.off():
            if torch.isnan(tmat).any():
                ld = torch.tensor(float("nan"), device=dev)
            else:
                ld = torch.tensor(op._plan().slq_logdet(tmat, n) + logdet_p, device=dev, dtype=torch.float32)
        iq = (solves[:, tp:] * r).sum(-2) if r is not None else torch.zeros(0, device=dev)
        ctx.tp, ctx.iters = tp, iters
        ctx.save_for_backward(solves, probes if probes is not None else torch.zeros(0, device=dev),
                              w if w is not None else torch.zeros(0, device=dev))
        op.last_cg_iters = iters
        return iq, ld

    @staticmethod
    def backward(ctx, grad_iq, grad_ld):
        op = ctx.op
        gn = grad_rhs = None
        nh = ctx.nh
        grads = [None] * nh
        need_h, need_x = ctx.needs_input_grad[4:4 + nh], ctx.needs_input_grad[4 + nh:]
        xgrads = [None] * len(need_x)
        need_k = any(ctx.needs_input_grad[3:4 + nh])
        if ctx.mode == "chol":
            chol, sol = ctx.saved_tensors
            n = op.shape[0]
            # dense: d iq = -sol sol^T : dK ; d logdet = K^-1 : dK
            left_cols, right_cols = [], []
            if ctx.has_rhs:
                left_cols.append(-sol * grad_iq.reshape(1, -1)); right_cols.append(sol)
                if ctx.needs_input_grad[1]:
                    grad_rhs = 2 * sol * grad_iq.reshape(1, -1)
            kinv = torch.cholesky_inverse(chol) if (ctx.want_logdet and (need_k or any(need_x))) else None
            if need_k:
                if ctx.want_logdet:
                    left_cols.append(kinv * grad_ld); right_cols.append(torch.eye(n, device=op.device))
                left = torch.cat(left_cols, -1).contiguous(); right = torch.cat(right_cols, -1).contiguous()
            if any(need_x):
                w = torch.zeros(n, n, device=op.device, dtype=torch.float32)
                if ctx.has_rhs:
                    w = w - (sol * grad_iq.reshape(1, -1)) @ sol.t()
                if kinv is not None:
                    w = w + grad_ld * kinv
        else:
            solves, probes, w = ctx.saved_tensors
            tp = ctx.tp
            left_cols, right_cols = [], []
            if ctx.want_logdet and tp and (need_k or any(need_x)):
                coef = 1.0 / tp
                norms = probes.norm(2, dim=-2, keepdim=True)
                pv_solves = solves[:, :tp] * coef * norms * grad_ld   # (1/tp) K^-1 z_i
                pz = probes
                if w.numel():
                    if op.per_row:   # P^-1 z = z / d - W (W^T z), W pre-scaled by D^-1
                        pz = probes / op.diag.diag_vec.detach().unsqueeze(-1) - w @ (w.t() @ probes)
                    else:
                        pz = (probes - w @ (w.t() @ probes)) / op.noise.detach()  # P^-1 z_i
                left_cols.append(pv_solves); right_cols.append(pz)
            if ctx.has_rhs:
                iq_solves = solves[:, tp:]
                neg = -iq_solves * grad_iq.reshape(1, -1)
                left_cols.append(neg); right_cols.append(iq_solves)
                if ctx.needs_input_grad[1]:
                    grad_rhs = -2 * neg
            if (need_k or any(need_x)) and left_cols:
                left = torch.cat(left_cols, -1).contiguous(); right = torch.cat(right_cols, -1).contiguous()
        if need_k and left_cols:
            if any(need_h):
                gs = op.kernel_op._bilinear_derivative_list(left, right)
                grads = [gi if need else None for gi, need in zip(gs, need_h)]
            if ctx.needs_input_grad[3]:
                gn = (left * right).sum(-1) if op.per_row else (left * right).sum().reshape(op.diag.diag_value.shape)
        if any(need_x) and ctx.mode == "chol":
            xgrads = op.kernel_op._dense_input_grad_list(w.contiguous(), need_x)
        elif any(need_x) and left_cols:
            xgrads = op.kernel_op._input_grad_list(left, right, need_x)
        return (None, grad_rhs, None, gn, *grads, *xgrads)

