"""Thin torch-facing wrapper over a gp_plan.  PyTorch is used only for device memory and streams."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import BACKEND, KIND, MllOpts, MllResult, check


def _ptr(t: torch.Tensor | None):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def _ld(t: torch.Tensor) -> int:
    """Leading dimension of a row-major block with unit column stride: a single row may carry any row stride (torch calls an
    expanded [1, t] tensor contiguous), so it gets t."""
    return t.stride(0) if t.size(0) > 1 else t.size(1)


def _row_block(t: torch.Tensor) -> torch.Tensor:
    """t itself when the engine can walk its rows with one leading dimension >= t.size(1) (unit column stride; a single row may
    carry any row stride), else a contiguous copy, e.g. of an expanded [n, s] block with row stride 0."""
    return t if t.stride(-1) == 1 and (t.size(0) == 1 or t.stride(0) >= t.size(1)) else t.contiguous()


def _require_cuda_f32(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must live on a CUDA device: gpytorch_b200 has no CPU path")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32 (got {t.dtype}); the sm_90a engine computes in fp32/3xTF32")


@dataclass
class MbcgInfo:
    iters: int
    tridiag_size: int
    residual_norms: list
    status: int


@dataclass
class CiqInfo:
    iters: int
    residual_norms: list      # [Q][t]: final |phibar| / |b_c| per shift and column
    status: int
    precond_rank: int = 0     # k of the split preconditioner (0: unpreconditioned)


class Plan:
    """Owns a gp_plan: inputs, hyper-parameters and workspaces for one covariance operator K(X1, X2)."""

    def __init__(self, x1: torch.Tensor, x2: torch.Tensor | None = None, backend: str = "auto",
                 row_begin: int = 0, row_count: int = 0, comm=None):
        self.lib = _lib.load()
        _require_cuda_f32(x1, "x1")
        if x1.dim() != 2:
            raise RuntimeError("x1 must be [n, d]")
        self.x1 = x1.contiguous()
        self.same = x2 is None or x2 is x1
        if not self.same:
            _require_cuda_f32(x2, "x2")
            if x2.dim() != 2 or x2.size(1) != x1.size(1):
                raise RuntimeError("x1 and x2 must have the same feature dimension")  # kernels/kernel.py:506-507
            self.x2 = x2.contiguous()
        else:
            self.x2 = self.x1
        self.device = x1.device
        self.n1, self.d = self.x1.shape
        self.n2 = self.x2.size(0)
        self.row_begin = row_begin
        self.row_count = row_count if row_count > 0 else self.n1
        self._h = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(self.lib.gp_plan_create(C.byref(self._h), self.device.index or 0, C.c_void_p(stream)))
        check(self.lib.gp_plan_set_backend(self._h, BACKEND[backend]))
        if comm is not None:
            check(self.lib.gp_plan_set_comm(self._h, comm.handle))
        self.comm = comm
        self.refresh_data()
        self.noise = 0.0
        self.outputscale = 1.0

    def refresh_data(self):
        """(Re-)register the input buffers: the engine re-packs its tiles (centre / scale / 3xTF32 split) from the
        CURRENT contents of x1 / x2.  Call after an in-place update of the inputs (operators._get_plan does, keyed on
        the tensors' version counters)."""
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_data(
                self._h, _ptr(self.x1), self.n1, self.x1.stride(0),
                _ptr(None if self.same else self.x2), self.n2, self.x2.stride(0), self.d,
                self.row_begin, self.row_count if self.row_count != self.n1 else 0))
            tasks = getattr(self, "_tasks", None)
            if tasks is not None:   # new data drops the engine's task layout: put it back
                check(self.lib.gp_plan_set_tasks(self._h, _ptr(tasks[0]), _ptr(tasks[1]), tasks[2]))
                if getattr(self, "_task_covar", None) is not None:
                    bh = self._task_covar
                    check(self.lib.gp_plan_set_task_covar(self._h, (C.c_float * bh.numel())(*bh.reshape(-1).tolist()), tasks[2]))
        return self

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.gp_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- hyper-parameters --------------------------------------------------------------------
    def set_hypers(self, kind: str, lengthscale, outputscale: float = 1.0, noise: float = 0.0):
        ls = [float(v) for v in (lengthscale if hasattr(lengthscale, "__len__") else [lengthscale])]
        arr = (C.c_float * len(ls))(*ls)
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers(self._h, KIND[kind], arr, len(ls), float(outputscale), float(noise)))
        # recorded once the engine took them: bilinear_grad sizes its output by these lengthscales
        self.kind, self.lengthscale, self.outputscale, self.noise = kind, ls, float(outputscale), float(noise)
        self.alpha = None
        self.poly = None
        return self

    def set_hypers_poly(self, power: int, offset: float, outputscale: float = 1.0, noise: float = 0.0):
        """Polynomial kernel S (x.x' + c)^p over the raw inputs (gp_plan_set_hypers_poly): kind, integer power 1..8, offset c >= 0,
        outputscale and noise in one engine call.  bilinear_grad then returns [dc] and dF/dS (the power is not learned)."""
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers_poly(self._h, int(power), float(offset), float(outputscale), float(noise)))
        # recorded once the engine took them: bilinear_grad sizes its output by the kind
        self.kind, self.lengthscale, self.outputscale, self.noise = "poly", [], float(outputscale), float(noise)
        self.alpha = None
        self.poly = (int(power), float(offset))
        return self

    def set_hypers_pp(self, q: int, lengthscale, outputscale: float = 1.0, noise: float = 0.0):
        """Piecewise polynomial kernel S (1 - r)_+^(j+q) poly_q(r) on the compact-support backend (gp_plan_set_hypers_pp): q in
        {0, 1, 2, 3}, lengthscales (1 or d), outputscale and noise in one engine call.  bilinear_grad then returns [dl (1 or d)] and
        dF/dS; info() adds the evaluated and total tile pairs."""
        ls = [float(v) for v in (lengthscale if hasattr(lengthscale, "__len__") else [lengthscale])]
        arr = (C.c_float * len(ls))(*ls)
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers_pp(self._h, int(q), arr, len(ls), float(outputscale), float(noise)))
        self.kind, self.lengthscale, self.outputscale, self.noise = "ppoly", ls, float(outputscale), float(noise)
        self.alpha = None
        self.poly = None
        return self

    def set_hypers_rq(self, lengthscale, alpha: float, outputscale: float = 1.0, noise: float = 0.0):
        """Rational quadratic kernel S (1 + r^2 / (2 alpha))^-alpha (gp_plan_set_hypers_rq): kind, lengthscales (1 or d), alpha,
        outputscale and noise in one engine call.  bilinear_grad then returns [dl (1 or d) | dalpha] and dF/dS."""
        ls = [float(v) for v in (lengthscale if hasattr(lengthscale, "__len__") else [lengthscale])]
        arr = (C.c_float * len(ls))(*ls)
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers_rq(self._h, arr, len(ls), float(alpha), float(outputscale), float(noise)))
        # recorded once the engine took them: bilinear_grad sizes its output by the lengthscales and alpha
        self.kind, self.lengthscale, self.outputscale, self.noise = "rq", ls, float(outputscale), float(noise)
        self.alpha = float(alpha)
        self.poly = None
        return self

    def set_ski(self, grid_sizes, grid_lo, grid_step):
        """SKI / KISS-GP: the operator becomes W (T_0 x ... x T_{d-1}) W^T on a regular grid (first node grid_lo[i], spacing
        grid_step[i], grid_sizes[i] nodes per dimension).  Call before set_hypers."""
        d = len(grid_sizes)
        gs = (C.c_int * d)(*[int(v) for v in grid_sizes])
        lo = (C.c_float * d)(*[float(v) for v in grid_lo])
        st = (C.c_float * d)(*[float(v) for v in grid_step])
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_ski(self._h, gs, lo, st, d))
        self.grid_points = 1
        for v in grid_sizes:
            self.grid_points *= int(v)
        return self

    def _ski_block(self, a: torch.Tensor, grid_rows: bool, name: str):
        """a as a 2-D block with unit column stride, checked against the plan: [M, t] (grid_rows) or [n, t]."""
        _require_cuda_f32(a, name)
        if a.device != self.device:
            raise RuntimeError(f"{name} lives on {a.device}, the plan on {self.device}")
        if getattr(self, "grid_points", None) is None:
            raise RuntimeError("the plan has no SKI grid (set_ski)")
        rows = self.grid_points if grid_rows else self.n1
        vec = a.dim() == 1
        a2 = a.unsqueeze(-1) if vec else a
        if a2.dim() != 2 or a2.size(0) != rows:
            raise RuntimeError(f"{name} must be [{rows}] or [{rows}, t] (got {tuple(a.shape)})")
        if a2.stride(-1) != 1:
            a2 = a2.contiguous()
        return a2, vec

    def ski_grid_matmul(self, v: torch.Tensor) -> torch.Tensor:
        """s K_uu W^T v on the SKI grid: v [n] or [n, t] over the plan's points -> [M] or [M, t], M = prod(grid_sizes), rows in
        the reference's flat grid order (dimension 0 slowest)."""
        v2, vec = self._ski_block(v, False, "rhs")
        out = torch.empty(self.grid_points, v2.size(1), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self.lib.gp_ski_grid_matmul(self._h, _ptr(v2), v2.stride(0), v2.size(1), _ptr(out), out.stride(0)))
        return out.squeeze(-1) if vec else out

    def ski_interp_matmul(self, c: torch.Tensor) -> torch.Tensor:
        """W c: grid values c [M] or [M, t] interpolated to the plan's points -> [n] or [n, t] in the caller's row order."""
        c2, vec = self._ski_block(c, True, "grid matrix")
        out = torch.empty(self.n1, c2.size(1), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self.lib.gp_ski_interp_matmul(self._h, _ptr(c2), c2.stride(0), c2.size(1), _ptr(out), out.stride(0)))
        return out.squeeze(-1) if vec else out

    def ski_input_grad(self, left: torch.Tensor, right: torch.Tensor) -> torch.Tensor:
        """dF/dx [n, d] of F = sum(left * (K_ski @ right)) for left, right [n] or [n, t] over the plan's points: the input gradient
        of the interpolated operator (outputscale folded in, noise excluded; the grid covariance does not move with x)."""
        l2, _ = self._ski_block(left, False, "left")
        r2, _ = self._ski_block(right, False, "right")
        if l2.size(1) != r2.size(1):
            raise RuntimeError(f"ski_input_grad: left and right need the same columns (got {tuple(left.shape)}, {tuple(right.shape)})")
        out = torch.empty(self.n1, self.d, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(self.lib.gp_ski_input_grad(self._h, _ptr(l2), _ld(l2), _ptr(r2), _ld(r2), r2.size(1), _ptr(out), out.stride(0)))
        return out

    def set_sum(self, terms):
        """Kernel sum (AdditiveKernel): this plan's operator becomes sum_t K_t (+ its own noise).  `terms` are ready plans over
        the same rows (their own kind / lengthscales / outputscale / active dimensions); they must outlive this plan.  Call after
        set_hypers (only the noise of this plan is used)."""
        terms = list(terms)
        arr = (C.c_void_p * len(terms))(*[t._h.value for t in terms])
        self._terms = terms                       # keep them alive
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_sum(self._h, arr, len(terms)))
        return self

    def set_product(self, factors):
        """Kernel product (ProductKernel): this plan's operator becomes S prod_f K_f (+ its own noise), S the product of the
        factors' outputscales.  `factors` are 2 to 4 ready plain plans over the same rows (their own kind / lengthscales /
        outputscale / active dimensions); they must outlive this plan.  set_hypers on this plan supplies the noise only."""
        factors = list(factors)
        arr = (C.c_void_p * max(len(factors), 1))(*[f._h.value for f in factors])
        self._factors = factors                   # keep them alive
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_product(self._h, arr, len(factors)))
        return self

    def set_additive(self, max_degree: int | None, comp_scale=None):
        """Additive GP: this plan's operator becomes sum_{m=1}^{M} e_m(c_1 .. c_D), c_i = comp_scale[i] k(x_i, x'_i) over the D = d
        columns (e_m the elementary symmetric polynomials, M = min(max_degree, D)).  set_hypers gives D lengthscales; its
        outputscale is ignored.  max_degree None (or comp_scale None) clears it.  bilinear_grad then returns the D lengthscale
        gradients and the list of D component-scale gradients."""
        if max_degree is None or comp_scale is None:
            self._additive = None
            with torch.cuda.device(self.device):
                check(self.lib.gp_plan_set_additive(self._h, 0, None, 0))
            return self
        sc = [float(v) for v in comp_scale]
        arr = (C.c_float * len(sc))(*sc)
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_additive(self._h, int(max_degree), arr, len(sc)))
        self._additive = (int(max_degree), sc)
        return self

    def set_spectral(self, weights=None, means=None, scales=None):
        """Spectral mixture kernel: this plan's operator becomes S prod_d sum_q w_q exp(-2 pi^2 v_qd^2 tau_d^2) cos(2 pi mu_qd tau_d)
        over tau = x - x' (S the outputscale of set_hypers, whose kind and lengthscale are ignored).  weights [Q], means and scales
        [Q, d] (host sequences or tensors); weights None clears it.  bilinear_grad then returns the Q (1 + 2d) gradients
        [dw | dmu (row-major) | dv (row-major)] and dF/dS."""
        if weights is None:
            self._spectral = None
            with torch.cuda.device(self.device):
                check(self.lib.gp_plan_set_spectral(self._h, 0, None, None, None, 0))
            return self
        w = [float(v) for v in (weights.reshape(-1).tolist() if torch.is_tensor(weights) else weights)]
        mu = torch.as_tensor(means, dtype=torch.float64).reshape(len(w), -1)
        sc = torch.as_tensor(scales, dtype=torch.float64).reshape(len(w), -1)
        Q, d = mu.shape
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_spectral(self._h, Q, (C.c_float * Q)(*w), (C.c_float * (Q * d))(*mu.reshape(-1).tolist()),
                                                (C.c_float * (Q * d))(*sc.reshape(-1).tolist()), d))
        self._spectral = (Q, d)
        return self

    def set_periodic(self, period=None):
        """Periodic kernel: this plan's operator becomes S exp(-2 sum_d sin^2(pi tau_d / p_d) / l_d) over tau = x - x', with the
        lengthscales l, outputscale S and noise of set_hypers (kind "rbf").  period: 1 or d values (a host sequence or tensor);
        None clears it.  bilinear_grad then returns [dl (1 or d) | dp (1 or d)] and dF/dS."""
        if period is None:
            self._periodic = None
            with torch.cuda.device(self.device):
                check(self.lib.gp_plan_set_periodic(self._h, None, 0, 0))
            return self
        per = [float(v) for v in (period.reshape(-1).tolist() if torch.is_tensor(period) else period)]
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_periodic(self._h, (C.c_float * len(per))(*per), len(per), self.d))
        self._periodic = len(per)
        return self

    def set_noise_diag(self, diag: torch.Tensor | None):
        """Per-row noise variances (FixedNoiseGaussianLikelihood): K_hat = K + diag(d).  None restores the scalar noise."""
        if diag is None:
            self._noise_diag = None
            check(self.lib.gp_plan_set_noise_diag(self._h, _ptr(None), 0))
            return self
        _require_cuda_f32(diag, "noise diagonal")
        self._noise_diag = diag.contiguous()      # keep it alive: the engine holds the raw pointer
        check(self.lib.gp_plan_set_noise_diag(self._h, _ptr(self._noise_diag), self._noise_diag.numel()))
        return self

    def set_lowrank(self, u: torch.Tensor | None):
        """Low-rank correction: the operator becomes s K - U U^T (+ noise).  u [n, r], 1 <= r <= 128; None clears it."""
        if u is None or u.size(-1) == 0:
            self._lowrank = None
            check(self.lib.gp_plan_set_lowrank(self._h, _ptr(None), 0, 0))
            return self
        _require_cuda_f32(u, "low-rank factor")
        if u.device != self.device:
            raise RuntimeError(f"low-rank factor lives on {u.device}, the plan on {self.device}")
        if u.dim() != 2 or u.size(0) != self.n2:
            raise RuntimeError(f"low-rank factor must be [{self.n2}, r] (got {tuple(u.shape)})")
        if u.stride(-1) != 1:
            u = u.contiguous()
        self._lowrank = u                         # keep it alive: the engine holds the raw pointer
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_lowrank(self._h, _ptr(u), u.stride(0), u.size(1)))
        return self

    def set_tasks(self, task1: torch.Tensor | None, task2: torch.Tensor | None = None, num_tasks: int | None = None):
        """Hadamard multitask: the operator becomes s K(x, x') o B[t, t'] once set_task_covar supplies B.  task1 [n1] (task2 [n2] on
        a cross plan, None on a square one) integer task ids in [0, num_tasks); None clears them.  The engine copies the ids and
        sorts its packed rows and columns by task; refresh_data (new inputs) re-applies them."""
        if task1 is None:
            self._tasks = None
            with torch.cuda.device(self.device):
                check(self.lib.gp_plan_set_tasks(self._h, _ptr(None), _ptr(None), 0))
            return self
        t1 = task1.reshape(-1).to(device=self.device, dtype=torch.int32).contiguous()
        if t1.numel() != self.n1:
            raise RuntimeError(f"task1 must have {self.n1} entries (got {t1.numel()})")
        t2 = None
        if not self.same:
            if task2 is None:
                raise RuntimeError("a cross plan needs the task ids of both inputs")
            t2 = task2.reshape(-1).to(device=self.device, dtype=torch.int32).contiguous()
            if t2.numel() != self.n2:
                raise RuntimeError(f"task2 must have {self.n2} entries (got {t2.numel()})")
        T = int(num_tasks) if num_tasks is not None else int(max(t1.max().item(), -1 if t2 is None else t2.max().item())) + 1
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_tasks(self._h, _ptr(t1), _ptr(t2), T))
        self._tasks = (t1, t2, T)
        self.num_tasks = T
        return self

    def set_task_covar(self, b: torch.Tensor):
        """B [T, T] of the Hadamard operator (any device; copied to the host).  Call again whenever it changes."""
        T = getattr(self, "num_tasks", None)
        if (getattr(self, "_tasks", None) is None and getattr(self, "data", None) is None) or T is None:
            raise RuntimeError("set_task_covar: the plan has no task ids (set_tasks) and is no Kronecker plan")
        bh = b.detach().to(device="cpu", dtype=torch.float32).contiguous()
        if tuple(bh.shape) != (T, T):
            raise RuntimeError(f"task covariance must be [{T}, {T}] (got {tuple(b.shape)})")
        arr = (C.c_float * (T * T))(*bh.reshape(-1).tolist())
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_task_covar(self._h, arr, T))
        self._task_covar = bh
        return self

    def task_covar_grad(self, left: torch.Tensor, right: torch.Tensor) -> torch.Tensor:
        """d/dB [T, T] (float64, CPU) of sum(left * ((s K o B) @ right)) for left [n1, s], right [n2, s]."""
        T = getattr(self, "num_tasks", None)
        if (getattr(self, "_tasks", None) is None and getattr(self, "data", None) is None) or T is None:
            raise RuntimeError("task_covar_grad: the plan has no task ids (set_tasks) and is no Kronecker plan")
        if left.dim() != 2 or right.dim() != 2 or left.size(0) != self.n1 or right.size(0) != self.n2 \
                or left.size(1) != right.size(1) or left.size(1) < 1:
            raise RuntimeError(f"task_covar_grad: left must be [{self.n1}, s] and right [{self.n2}, s] "
                               f"(got {tuple(left.shape)}, {tuple(right.shape)})")
        _require_cuda_f32(left, "left")
        _require_cuda_f32(right, "right")
        left, right = _row_block(left), _row_block(right)
        out = (C.c_double * (T * T))()
        with torch.cuda.device(self.device):
            check(self.lib.gp_task_covar_grad(self._h, _ptr(left), _ld(left), _ptr(right), _ld(right), left.size(1), out))
        return torch.tensor([out[i] for i in range(T * T)], dtype=torch.float64).reshape(T, T)

    def info(self):
        b, s, k, m = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        check(self.lib.gp_plan_info(self._h, C.byref(b), C.byref(s), C.byref(k), C.byref(m)))
        out = {"backend": {1: "tcgen05", 2: "simt", 3: "ski", 4: "sum", 5: "kron", 6: "deriv", 7: "product", 8: "compact"}.get(b.value, "?"),
               "nsplit": s.value, "kpad": k.value, "n_sm": m.value}
        if b.value == _lib.GP_BACKEND_COMPACT:   # tile pairs of 128 rows x 64 columns: evaluated per K.V, and all of them
            ev, tot = C.c_int64(), C.c_int64()
            check(self.lib.gp_plan_tile_pairs(self._h, C.byref(ev), C.byref(tot)))
            out["tile_pairs"], out["tile_pairs_total"] = ev.value, tot.value
        return out

    def time_kmv_kernel(self, v: torch.Tensor, warmup: int = 3, reps: int = 20) -> float:
        """Average device time (ms) of ONE launch of the fused K.V kernel alone (CUDA events on the plan stream)."""
        v = v.contiguous()
        ms = C.c_float()
        check(self.lib.gp_time_kmv_kernel(self._h, _ptr(v), v.stride(0), v.size(1), warmup, reps, C.byref(ms)))
        return ms.value

    def launches(self) -> int:
        return int(self.lib.gp_kernel_launches(self._h))

    # ---- kernel seam -------------------------------------------------------------------------
    def kmv(self, v: torch.Tensor, add_noise: bool = False) -> torch.Tensor:
        """K(X1,X2) @ v (+ noise*v).  v [n2] or [n2, t]."""
        _require_cuda_f32(v, "rhs")
        vec = v.dim() == 1
        v2 = (v.unsqueeze(-1) if vec else v).contiguous()
        if v2.size(0) != self.n2:
            raise RuntimeError(f"Size mismatch: operator has {self.n2} columns, rhs has {v2.size(0)} rows")
        out = torch.empty(self.row_count, v2.size(1), device=self.device, dtype=torch.float32)
        check(self.lib.gp_kmv(self._h, _ptr(v2), _ld(v2), v2.size(1), _ptr(out), out.stride(0), int(add_noise)))
        return out.squeeze(-1) if vec else out

    def rows(self, idx: torch.Tensor) -> torch.Tensor:
        idx = idx.to(device=self.device, dtype=torch.int64).contiguous()
        out = torch.empty(idx.numel(), self.n2, device=self.device, dtype=torch.float32)
        check(self.lib.gp_krows(self._h, _ptr(idx), idx.numel(), _ptr(out), out.stride(0)))
        return out

    def diag(self) -> torch.Tensor:
        out = torch.empty(self.row_count, device=self.device, dtype=torch.float32)
        check(self.lib.gp_kdiag(self._h, _ptr(out)))
        return out

    def bilinear_grad(self, left: torch.Tensor, right: torch.Tensor):
        """(d/d lengthscale[*], d/d outputscale) of sum(left * (K @ right)) for left [row_count, s], right [n2, s].  On a kernel
        product: the factors' lengthscale gradients one after the other, and the gradient of the combined scale S.  On an additive
        plan: the D lengthscale gradients and the list of the D component-scale gradients.  On a spectral plan: the Q (1 + 2d)
        gradients [dw | dmu | dv] and dF/dS.  On a periodic plan: [dl | dp] and dF/dS.  On a rational quadratic plan: [dl | dalpha]
        and dF/dS.  On a polynomial plan: [dc] and dF/dS."""
        if left.dim() != 2 or right.dim() != 2 or left.size(0) != self.row_count or right.size(0) != self.n2 \
                or left.size(1) != right.size(1) or left.size(1) < 1:
            raise RuntimeError(f"bilinear_grad: left must be [{self.row_count}, s] and right [{self.n2}, s] with s >= 1 "
                               f"(got {tuple(left.shape)}, {tuple(right.shape)})")
        _require_cuda_f32(left, "left")
        _require_cuda_f32(right, "right")
        for t, name in ((left, "left"), (right, "right")):
            if t.device != self.device:
                raise RuntimeError(f"{name} lives on {t.device}, the plan on {self.device}")
        left, right = _row_block(left), _row_block(right)
        s = left.size(1)
        factors = getattr(self, "_factors", None)
        nls = sum(len(f.lengthscale) for f in factors) if factors else len(self.lengthscale)
        if not factors and getattr(self, "alpha", None) is not None:   # [dl | dalpha] and dF/dS
            nls += 1
        if not factors and getattr(self, "poly", None) is not None:    # [dc] and dF/dS
            nls = 1
        gl = (C.c_double * nls)()
        if getattr(self, "_spectral", None) is not None:   # [dw | dmu | dv] and dF/dS
            Q, d = self._spectral
            nls = Q * (1 + 2 * d)
            gl = (C.c_double * nls)()
        if getattr(self, "_periodic", None) is not None:   # [dl | dp] and dF/dS
            nls = len(self.lengthscale) + self._periodic
            gl = (C.c_double * (2 * self.d))()   # the engine writes at most d + d values, whatever this side recorded
        if getattr(self, "_additive", None) is not None:   # D component-scale gradients
            go = (C.c_double * len(self._additive[1]))()
            with torch.cuda.device(self.device):
                check(self.lib.gp_bilinear_grad(self._h, _ptr(left), _ld(left), _ptr(right), _ld(right), s, gl, go))
            return [gl[i] for i in range(nls)], list(go)
        go = C.c_double()
        with torch.cuda.device(self.device):
            check(self.lib.gp_bilinear_grad(self._h, _ptr(left), _ld(left), _ptr(right), _ld(right), s, gl, C.byref(go)))
        return [gl[i] for i in range(nls)], go.value

    def _grad_outputs(self, dx1: bool, dx2: bool):
        """The output blocks of an input gradient: on a square plan DX1 receives the total and DX2 is None."""
        o1 = torch.empty(self.n1, self.d, device=self.device, dtype=torch.float32) if dx1 else None
        o2 = torch.empty(self.n2, self.d, device=self.device, dtype=torch.float32) if (dx2 and not self.same) else None
        return o1, o2

    def kmv_input_grad(self, g: torch.Tensor, v: torch.Tensor, dx1: bool = True, dx2: bool = True):
        """(dF/dx1 [n1, d], dF/dx2 [n2, d]) of F = sum(g * (K @ v)) in raw input units (outputscale folded in, noise excluded);
        g [n1] or [n1, t], v [n2] or [n2, t].  On a square plan the first entry is the total gradient and the second is None;
        an entry not asked for is None."""
        _require_cuda_f32(g, "g")
        _require_cuda_f32(v, "v")
        g2 = g.unsqueeze(-1) if g.dim() == 1 else g
        v2 = v.unsqueeze(-1) if v.dim() == 1 else v
        if g2.dim() != 2 or v2.dim() != 2 or g2.shape != (self.row_count, v2.size(1)) or v2.size(0) != self.n2:
            raise RuntimeError(f"kmv_input_grad: g must be [{self.row_count}, t] and v [{self.n2}, t] (got {tuple(g.shape)}, {tuple(v.shape)})")
        g2 = g2 if g2.stride(-1) == 1 else g2.contiguous()
        v2 = v2 if v2.stride(-1) == 1 else v2.contiguous()
        o1, o2 = self._grad_outputs(dx1, dx2)
        with torch.cuda.device(self.device):
            check(self.lib.gp_kmv_input_grad(self._h, _ptr(g2), _ld(g2), _ptr(v2), _ld(v2), v2.size(1),
                                             _ptr(o1), self.d, _ptr(o2), self.d))
        return o1, o2

    def dense_input_grad(self, w: torch.Tensor, dx1: bool = True, dx2: bool = True):
        """(dF/dx1, dF/dx2) of F = sum(w * K) for w [n1, n2]: the input gradient of the block rows() returns (see kmv_input_grad)."""
        _require_cuda_f32(w, "w")
        if w.dim() != 2 or tuple(w.shape) != (self.row_count, self.n2):
            raise RuntimeError(f"dense_input_grad: w must be [{self.row_count}, {self.n2}] (got {tuple(w.shape)})")
        w = w if w.stride(-1) == 1 else w.contiguous()
        o1, o2 = self._grad_outputs(dx1, dx2)
        with torch.cuda.device(self.device):
            check(self.lib.gp_kdense_input_grad(self._h, _ptr(w), _ld(w), _ptr(o1), self.d, _ptr(o2), self.d))
        return o1, o2

    # ---- solver seam -------------------------------------------------------------------------
    def pivoted_cholesky(self, rank: int, error_tol: float = 1e-3):
        """Returns (Lt [m, n] (= L^T), pivots [m], status)."""
        rank = min(rank, self.n2)
        lt = torch.empty(rank, self.n2, device=self.device, dtype=torch.float32)
        piv = torch.empty(rank, device=self.device, dtype=torch.int64)
        r = C.c_int()
        st = check(self.lib.gp_pivoted_cholesky(self._h, rank, float(error_tol), _ptr(lt), _ptr(piv), C.byref(r)))
        return lt[: r.value], piv[: r.value], st

    def precond_build(self, lt: torch.Tensor):
        """W [n_local, k] with P^-1 v = (v - W W^T v)/noise, and log det P."""
        lt = lt.contiguous()
        k = lt.size(0)
        w = torch.empty(self.row_count, k, device=self.device, dtype=torch.float32)
        ld = C.c_double()
        st = check(self.lib.gp_precond_build(self._h, _ptr(lt), k, _ptr(w), C.byref(ld)))
        return w, ld.value, st

    def ciq_precond_build(self, lt: torch.Tensor):
        """U [n, k], tr(K - L L^T) and the status: the split factor of P = L L^T + D for ciq_sqrt_matmul(precond_u=U)."""
        lt = lt.contiguous()
        k = lt.size(0)
        u = torch.empty(self.n2, k, device=self.device, dtype=torch.float32)
        tr = C.c_double()
        st = check(self.lib.gp_ciq_precond_build(self._h, _ptr(lt), k, _ptr(u), C.byref(tr)))
        return u, tr.value, st

    def precond_probes(self, lt, eps1, eps2):
        lt = lt.contiguous(); eps1 = eps1.contiguous(); eps2 = eps2.contiguous()
        k, tp = lt.size(0), eps2.size(1)
        z = torch.empty(self.row_count, tp, device=self.device, dtype=torch.float32)
        check(self.lib.gp_precond_probes(self._h, _ptr(lt), k, _ptr(eps1), _ptr(eps2), tp, _ptr(z)))
        return z

    def mbcg(self, rhs: torch.Tensor, n_tridiag: int = 0, tolerance: float = 1.0, max_iter: int = 1000,
             max_tridiag_iter: int = 20, precond_w: torch.Tensor | None = None, warn: bool = True):
        """linear_cg on K + noise I.  rhs [n, t], t <= 16.  Returns (solves, t_mat | None, MbcgInfo)."""
        _require_cuda_f32(rhs, "rhs")
        rhs = rhs.contiguous()
        n, t = rhs.shape
        solves = torch.empty_like(rhs)
        mti = int(max_tridiag_iter)  # > max_iter is rejected by the engine like the reference does
        tmat = torch.zeros(max(n_tridiag, 1), min(mti, 4096), min(mti, 4096), device=self.device, dtype=torch.float32)
        it, js = C.c_int(), C.c_int()
        resid = (C.c_float * 16)()
        w = None if precond_w is None else precond_w.contiguous()
        st = self.lib.gp_mbcg(self._h, _ptr(rhs), rhs.stride(0), t, n_tridiag, float(tolerance), int(max_iter), int(mti),
                              _ptr(w), 0 if w is None else w.size(1), _ptr(solves), solves.stride(0), _ptr(tmat),
                              C.byref(it), C.byref(js), resid)
        check(st, warn=warn)
        info = MbcgInfo(it.value, js.value, [resid[i] for i in range(t)], st)
        tm = tmat[:n_tridiag, : js.value, : js.value] if n_tridiag else None
        return solves, tm, info

    def slq_logdet(self, tmat: torch.Tensor, n: int | None = None) -> float:
        tmat = tmat.contiguous()
        tp, j, _ = tmat.shape
        out = C.c_double()
        check(self.lib.gp_slq_logdet(self._h, _ptr(tmat), tp, j, j, int(n if n is not None else self.n2), C.byref(out)))
        return out.value

    def lanczos(self, init: torch.Tensor, max_iter: int, tol: float = 1e-5):
        """Returns (Q [n_local, J], T [J, J]); on a row-sharded plan init / Q hold this rank's rows."""
        init = init.contiguous()
        if init.numel() != self.row_count:
            raise RuntimeError(f"Lanczos start vector has {init.numel()} entries, the plan owns {self.row_count} rows")
        qt = torch.zeros(max_iter, self.row_count, device=self.device, dtype=torch.float32)
        tm = torch.zeros(max_iter, max_iter, device=self.device, dtype=torch.float32)
        j = C.c_int()
        check(self.lib.gp_lanczos(self._h, _ptr(init), int(max_iter), float(tol), _ptr(qt), _ptr(tm), C.byref(j)))
        return qt[: j.value].t(), tm[: j.value, : j.value]

    def ciq_sqrt_matmul(self, b: torch.Tensor, tau, w, tol: float = 1e-4, max_iter: int = 1000, warn: bool = True,
                        precond_u: torch.Tensor | None = None):
        """K_hat sum_q w_q (K_hat + tau_q I)^{-1} b ~= K_hat^{1/2} b by multi-shift MINRES (csrc/minres.cu); K_hat is this plan's
        operator with its noise.  b [n, t], t <= 16; tau / w host sequences of Q <= 32 floats.  Returns (out [n, t], CiqInfo).
        With precond_u = U [n, k] from ciq_precond_build: K_hat F^-T sum_q w_q (A + tau_q I)^{-1} b ~= F A^{1/2} b, A = F^-1 K_hat F^-T
        (tau / w then belong to A's spectrum)."""
        _require_cuda_f32(b, "rhs")
        vec = b.dim() == 1
        b2 = b.unsqueeze(-1) if vec else b
        if b2.stride(-1) != 1:
            b2 = b2.contiguous()
        n, t = b2.shape
        Q = len(tau)
        out = torch.empty(n, t, device=self.device, dtype=torch.float32)
        ta = (C.c_double * max(Q, 1))(*[float(v) for v in tau])
        wa = (C.c_double * max(Q, 1))(*[float(v) for v in w])
        it = C.c_int()
        resid = (C.c_float * max(Q * t, 1))()
        with torch.cuda.device(self.device):
            if precond_u is None:
                st = self.lib.gp_ciq_sqrt_matmul(self._h, _ptr(b2), b2.stride(0), t, ta, wa, Q, float(tol), int(max_iter),
                                                 _ptr(out), out.stride(0), C.byref(it), resid)
            else:
                u = precond_u.contiguous()
                st = self.lib.gp_ciq_sqrt_matmul_precond(self._h, _ptr(b2), b2.stride(0), t, _ptr(u), u.size(-1), ta, wa, Q,
                                                         float(tol), int(max_iter), _ptr(out), out.stride(0), C.byref(it), resid)
        if st == _lib.GP_E_NAN_MVM:
            raise _lib.NanError(_lib.last_error())
        check(st, warn=warn)
        info = CiqInfo(it.value, [[resid[q * t + c] for c in range(t)] for q in range(Q)], st,
                       0 if precond_u is None else precond_u.size(-1))
        return (out.squeeze(-1) if vec else out), info

    def mll(self, y_minus_mean, eps1, eps2, rademacher, num_probes=10, precond_rank=15, min_precond_size=2000,
            precond_tol=1e-3, cg_tol=1.0, max_cg_iter=1000, max_tridiag_iter=20, want_solve=False, warn=True):
        opts = MllOpts(num_probes, precond_rank, min_precond_size, precond_tol, cg_tol, max_cg_iter, max_tridiag_iter)
        res = MllResult()
        solve = torch.empty(self.row_count, device=self.device, dtype=torch.float32) if want_solve else None
        st = self.lib.gp_mll(self._h, _ptr(y_minus_mean.contiguous()), _ptr(eps1), _ptr(eps2), _ptr(rademacher),
                             C.byref(opts), _ptr(solve), C.byref(res))
        check(st, warn=warn)
        if res.status_flags & 6 and warn:   # bit 1: CG not converged, bit 2: SLQ eigen-solver not converged
            import warnings
            warnings.warn(_lib.last_error(), _lib.NumericalWarning)
        return res, solve


class _DataPlanOperator(Plan):
    """A plan whose operator is built on a ready data Plan (kept alive here): the engine reads the data plan's packed rows and
    hyper-parameters, and only the noise is this plan's own.  Subclasses attach the data plan through their C call."""

    def __init__(self, data: Plan, *args):
        self.lib = data.lib
        self.device = data.device
        self._h = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(self.lib.gp_plan_create(C.byref(self._h), self.device.index or 0, C.c_void_p(stream)))
        self.comm = None
        self.noise, self.outputscale = 0.0, 1.0
        self.attach(data, *args)

    def set_hypers(self, kind=None, lengthscale=None, outputscale: float = 1.0, noise: float = 0.0):
        """Only the noise is this plan's own: kind and lengthscales are the data plan's."""
        return self.set_noise(noise)

    def set_noise(self, noise: float):
        ls = list(self.data.lengthscale)
        arr = (C.c_float * len(ls))(*ls)
        self.kind, self.lengthscale, self.noise = self.data.kind, ls, float(noise)
        self.outputscale = self.data.outputscale
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers(self._h, KIND[self.kind], arr, len(ls), float(self.outputscale), float(noise)))
        return self


class KronPlan(_DataPlanOperator):
    """The Kronecker multitask operator (s K_data) (x) B over interleaved rows i T + a (gp_plan_set_kron): N1 T x N2 T, built on a
    ready data Plan (kept alive here).  set_noise supplies the noise; set_task_covar / task_covar_grad take B and its gradient,
    bilinear_grad returns the data kernel's (lengthscale, outputscale) gradients.  Every product, solve and sample call of Plan
    works on it."""

    def __init__(self, data: Plan, num_tasks: int):
        super().__init__(data, num_tasks)

    def attach(self, data: Plan, num_tasks: int):
        """(Re-)attach the data plan: validation and geometry only; a B of the same size stays set, and so does a mask of the same
        N1, N2 and T (set_observed)."""
        T = int(num_tasks)
        obs = getattr(self, "_observed", None)
        if obs is not None and (obs[2], obs[3], obs[4]) != (data.n1, data.n2, T):
            obs = None                    # the engine drops the mask with the sizes it was given for
        self._observed = obs
        self.data, self.num_tasks = data, T
        self.same, self.d = data.same, data.d
        self.n1 = data.n1 * T if obs is None or obs[0] is None else obs[0].numel()
        self.n2 = data.n2 * T if obs is None or obs[1] is None else obs[1].numel()
        self.row_begin, self.row_count = 0, self.n1
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_kron(self._h, data._h, T))
        return self

    def refresh_data(self):
        return self.attach(self.data, self.num_tasks)

    def set_observed(self, rows: torch.Tensor | None, cols: torch.Tensor | None):
        """Keep the interleaved rows `rows` and columns `cols` only (strictly increasing int64 indices; None: all), so the operator
        becomes P_r ((s K) (x) B) P_c^T (gp_plan_set_kron_observed).  rows = cols = None removes the mask.  The indices are copied
        to the host and from there to the device once.  On a square plan the two masks are equal: cols = None takes rows."""
        rh = None if rows is None else rows.detach().to(device="cpu", dtype=torch.int64).contiguous()
        ch = None if cols is None else cols.detach().to(device="cpu", dtype=torch.int64).contiguous()
        if self.same and ch is None:
            ch = rh
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_kron_observed(self._h, _ptr(rh), 0 if rh is None else rh.numel(),
                                                      _ptr(ch), 0 if ch is None else ch.numel()))
        T = self.num_tasks
        n1f, n2f = self.data.n1 * T, self.data.n2 * T
        rh = None if rh is None or rh.numel() == n1f else rh     # a list of every row is no mask (as in the engine)
        ch = None if ch is None or ch.numel() == n2f else ch
        self._observed = None if rh is None and ch is None else (rh, ch, self.data.n1, self.data.n2, T)
        self.n1 = n1f if rh is None else rh.numel()
        self.n2 = n2f if ch is None else ch.numel()
        self.row_count = self.n1
        if getattr(self, "_noise_diag", None) is not None and self._noise_diag.numel() != self.n1:
            self._noise_diag = None       # the engine dropped it with the old row count
        return self


class LcmPlan(_DataPlanOperator):
    """The linear model of coregionalisation sum_q (s_q K_q) (x) B_q over interleaved rows i T + a (gp_plan_set_kron_terms): N1 T x
    N2 T, built on Q = 1..4 ready data Plans over the same number of points (kept alive here), each with its own kind, lengthscales,
    outputscale s_q, backend and inputs.  set_noise supplies the noise; set_term_covars / terms_grad take the B_q and return every
    gradient.  Every product, solve and sample call of Plan works on it."""

    def __init__(self, datas, num_tasks: int):
        super().__init__(list(datas)[0], list(datas), num_tasks)

    def attach(self, first: Plan, datas, num_tasks: int):
        """(Re-)attach the data plans: validation and geometry only; B_q of the same Q and T stay set."""
        datas = list(datas)
        T = int(num_tasks)
        arr = (C.c_void_p * len(datas))(*[d._h.value for d in datas])
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_kron_terms(self._h, arr, len(datas), T))
        self.data, self.datas, self.num_tasks = datas[0], datas, T
        self.same, self.d = datas[0].same, datas[0].d
        self.n1, self.n2 = datas[0].n1 * T, datas[0].n2 * T
        self.row_begin, self.row_count = 0, self.n1
        return self

    def refresh_data(self):
        return self.attach(self.data, self.datas, self.num_tasks)

    def set_noise(self, noise: float):
        """The noise of this plan; each term keeps its own kind, lengthscales and outputscale."""
        arr = (C.c_float * 1)(1.0)
        self.kind, self.lengthscale, self.noise, self.outputscale = self.data.kind, [1.0], float(noise), 1.0
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_hypers(self._h, KIND[self.kind], arr, 1, 1.0, float(noise)))
        return self

    def set_term_covars(self, b: torch.Tensor):
        """B_q [Q, T, T] (any device; copied to the host).  Call again whenever one changes."""
        Q, T = len(self.datas), self.num_tasks
        bh = b.detach().to(device="cpu", dtype=torch.float32).contiguous()
        if tuple(bh.shape) != (Q, T, T):
            raise RuntimeError(f"the task covariances must be [{Q}, {T}, {T}] (got {tuple(b.shape)})")
        arr = (C.c_float * (Q * T * T))(*bh.reshape(-1).tolist())
        with torch.cuda.device(self.device):
            check(self.lib.gp_plan_set_kron_term_covars(self._h, arr, Q, T))
        return self

    def terms_grad(self, left: torch.Tensor, right: torch.Tensor):
        """([dl_q] per term, [ds_q], dB [Q, T, T] float64 on the CPU) of sum(left * (K @ right)), left [n1, s], right [n2, s]."""
        if left.dim() != 2 or right.dim() != 2 or left.size(0) != self.n1 or right.size(0) != self.n2 \
                or left.size(1) != right.size(1) or left.size(1) < 1:
            raise RuntimeError(f"terms_grad: left must be [{self.n1}, s] and right [{self.n2}, s] "
                               f"(got {tuple(left.shape)}, {tuple(right.shape)})")
        _require_cuda_f32(left, "left")
        _require_cuda_f32(right, "right")
        left, right = _row_block(left), _row_block(right)
        Q, T = len(self.datas), self.num_tasks
        nls = [len(d.lengthscale) for d in self.datas]
        gl, go, db = (C.c_double * sum(nls))(), (C.c_double * Q)(), (C.c_double * (Q * T * T))()
        with torch.cuda.device(self.device):
            check(self.lib.gp_kron_terms_grad(self._h, _ptr(left), _ld(left), _ptr(right), _ld(right), left.size(1), gl, go, db))
        out, o = [], 0
        for k in nls:
            out.append([gl[o + i] for i in range(k)])
            o += k
        return out, [go[q] for q in range(Q)], torch.tensor(list(db), dtype=torch.float64).reshape(Q, T, T)


class DerivPlan(_DataPlanOperator):
    """The value / gradient operator over interleaved rows i (d+1) + a: N1 (d+1) x N2 (d+1), built on a ready plain data Plan of
    covariance `kind` (kept alive here): "rbf" (gp_plan_set_deriv, RBFKernelGrad) or "matern52" (gp_plan_set_deriv_kind,
    Matern52KernelGrad).  set_noise supplies the noise; bilinear_grad returns the data kernel's (lengthscale, outputscale)
    gradients.  Every product, solve and sample call of Plan works on it; it has no task covariance."""

    def __init__(self, data: Plan, kind: str = "rbf"):
        if kind not in ("rbf", "matern52"):
            raise ValueError(f"derivative observations are available for the 'rbf' and 'matern52' kernels (got {kind!r})")
        super().__init__(data, kind)

    def attach(self, data: Plan, kind: str = "rbf"):
        """(Re-)attach the data plan: validation and geometry only.  A refused data plan leaves the operator as it was."""
        with torch.cuda.device(self.device):
            if kind == "rbf":
                check(self.lib.gp_plan_set_deriv(self._h, data._h))
            else:
                check(self.lib.gp_plan_set_deriv_kind(self._h, data._h, KIND[kind]))
        rw = data.d + 1
        self.data, self.num_outputs, self.deriv_kind = data, rw, kind
        self.same, self.d = data.same, data.d
        self.n1, self.n2 = data.n1 * rw, data.n2 * rw
        self.row_begin, self.row_count = 0, self.n1
        return self

    def refresh_data(self):
        return self.attach(self.data, self.deriv_kind)

    def set_task_covar(self, b):
        raise RuntimeError("a derivative-observation plan has no task covariance (its d + 1 outputs per point are fixed by the kernel)")

    def task_covar_grad(self, left, right):
        raise RuntimeError("a derivative-observation plan has no task covariance (its d + 1 outputs per point are fixed by the kernel)")
