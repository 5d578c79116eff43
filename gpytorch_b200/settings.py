"""Solver knobs with the reference's names and defaults (gpytorch/settings.py:6-31 re-exports the
linear_operator settings; own knobs :173-180, :261-269).  Class-level context managers, as in the
reference (settings.py:84-144): `with settings.cg_tolerance(1e-4): ...`, `settings.cg_tolerance.value()`.
"""
from __future__ import annotations

import logging


class _Knob:
    """One process-wide setting addressed through its class.  Entering `with knob(v):` pushes v on the class's override stack,
    leaving pops it; the innermost override wins, an empty stack means the default.  (The reference keeps a single global slot and
    saves / restores it in every instance, settings.py:84-144; the stack gives the same nesting semantics and makes the state
    of all knobs one list per class, which snapshot() below copies for worker threads.)"""

    _default = None
    _overrides: list = []

    def __init_subclass__(cls, **kwargs):
        super().__init_subclass__(**kwargs)
        cls._overrides = []          # every knob owns its stack

    def __init__(self, value):
        self._value = value

    def __enter__(self):
        type(self)._overrides.append(self._value)
        return self

    def __exit__(self, *exc):
        type(self)._overrides.pop()
        return False

    @classmethod
    def _current(cls):
        return cls._overrides[-1] if cls._overrides else cls._default


class _value_context(_Knob):
    """`knob.value()` / `with knob(v): ...`; subclasses give the reference's default as `_global_value`."""

    _global_value = None

    @classmethod
    def value(cls):
        return cls._overrides[-1] if cls._overrides else cls._global_value

    @classmethod
    def _set_value(cls, value):
        """Change the process-wide default (outside any `with`)."""
        cls._global_value = value


class _feature_flag(_Knob):
    """`flag.on()` / `flag.off()` / `with flag(True | False): ...`."""

    _default = False

    def __init__(self, state=True):
        super().__init__(bool(state))

    @classmethod
    def on(cls):
        return bool(cls._current())

    @classmethod
    def off(cls):
        return not cls.on()


class cg_tolerance(_value_context):
    _global_value = 1.0


class eval_cg_tolerance(_value_context):
    _global_value = 0.01  # gpytorch/settings.py:173-180


class max_cg_iterations(_value_context):
    _global_value = 1000


class max_cholesky_size(_value_context):
    _global_value = 800


class max_lanczos_quadrature_iterations(_value_context):
    _global_value = 20


class max_preconditioner_size(_value_context):
    _global_value = 15


class min_preconditioning_size(_value_context):
    _global_value = 2000


class num_trace_samples(_value_context):
    _global_value = 10


class preconditioner_tolerance(_value_context):
    _global_value = 1e-3


class max_root_decomposition_size(_value_context):
    _global_value = 100


class ciq_samples(_feature_flag):
    """Draw MultivariateNormal samples of an engine operator as K_hat^{1/2} xi by contour integral quadrature and multi-shift
    MINRES (linear_operator settings; off by default).  Off: Cholesky up to max_cholesky_size, a Lanczos root above it."""
    _default = False


class ciq_preconditioner(_feature_flag):
    """With ciq_samples on, run CIQ on A = F^-1 K_hat F^-T, F F^T = P the pivoted-Cholesky preconditioner of the solves (same knobs:
    max_preconditioner_size, min_preconditioning_size, preconditioner_tolerance), and return F A^{1/2} xi (off by default).
    msMINRES then needs about sqrt(kappa(A)) instead of sqrt(kappa(K_hat)) iterations.  The draw has the same distribution
    N(0, K_hat) but is a different root applied to the same xi: off, samples are K_hat^{1/2} xi, continuous in the
    hyper-parameters (common random numbers across a sweep); on, they jump where the pivot order changes.  No effect where the
    solves have no preconditioner (SKI without ski_preconditioner, no noise, n < min_preconditioning_size,
    max_preconditioner_size(0), a failed build)."""
    _default = False


class num_contour_quadrature(_value_context):
    """Quadrature points Q of the CIQ square root (linear_operator settings; default 15)."""
    _global_value = 15


class minres_tolerance(_value_context):
    """Relative residual at which msMINRES stops (linear_operator settings; default 1e-4)."""
    _global_value = 1e-4


class observation_nan_policy(_value_context):
    """NaN handling policy for observations (settings.py:407-450).

    * ``ignore``: do not check for NaN values (the default).
    * ``mask``: mask out NaN values during calculation: ExactMarginalLogLikelihood and the exact prediction strategy use the
      observed entries of the mean, the target and the covariance rows and columns (an entry that is NaN in one batch element is
      masked for the whole batch).  A Kronecker multitask model keeps one engine operator, P ((s K) (x) B + D) P^T over the
      observed interleaved rows.  With no NaN in the targets every call returns what ``ignore`` returns.
    * ``fill``: fill in NaN values with a dummy value for prediction; refused by ExactMarginalLogLikelihood.  Prediction gives
      the mean ``mask`` gives (the two are the same posterior; the engine never builds the dense masked kernel).

    Deviation: the reference's predictive covariance and LOVE cache solve with the full training covariance even under ``mask``;
    here both condition on the observed rows only, which is the posterior of the masked model."""

    _fill_value = -999.0
    _global_value = "ignore"

    def __init__(self, value):
        if value not in {"ignore", "mask", "fill"}:
            raise ValueError(f"NaN handling policy {value} not supported!")
        super().__init__(value)

    @staticmethod
    def _get_observed(observations, event_shape):
        """The mask over event_shape of the entries that are not NaN in any batch element (settings.py:428-440)."""
        import torch
        return ~torch.any(torch.isnan(observations.reshape(-1, *event_shape)), dim=0)

    @classmethod
    def _fill_tensor(cls, observations):
        """observations with every NaN replaced by _fill_value (settings.py:442-450)."""
        import torch
        return torch.nan_to_num(observations, nan=cls._fill_value)


class skip_logdet_forward(_feature_flag):
    _default = False


class fast_pred_var(_feature_flag):
    """LOVE predictive variances: K_hat^{-1} ~= R R^T from `max_root_decomposition_size` Lanczos steps
    (settings.py:183-222; models/exact_prediction_strategies.py:268-272, 464-478)."""
    _default = False


class fast_pred_samples(_feature_flag):
    """Fast predictive samples using Lanczos Variance Estimates (LOVE).
    Use this for improved performance when sampling from a predictive posterior matrix.

    As described in the paper: `Constant-Time Predictive Distributions for Gaussian Processes`_.

    (settings.py:225-243.)  Here: an exact GP's posterior in eval mode keeps its LOVE covariance K** - K*x R R^T Kx* lazy
    (operators.LowRankUpdatedKernelLinearOperator), so that variances, CIQ samples and log_prob at m test points never build an
    m x m matrix.  Off by default.

    .. _`Constant-Time Predictive Distributions for Gaussian Processes`:
        https://arxiv.org/abs/1803.06058
    """
    _default = False


class skip_posterior_variances(_feature_flag):
    """Return a zero predictive covariance (models/exact_prediction_strategies.py:432-433)."""
    _default = False


class _use_eval_tolerance(_feature_flag):
    _default = False


class terminate_cg_by_size(_feature_flag):
    """Cap the CG iterations at n for an n x n system (linear_operator settings; off by default as upstream)."""
    _default = False


class tridiagonal_jitter(_value_context):
    """Relative jitter upstream adds to the Lanczos tridiagonals before the eigendecomposition (default 1e-6).  Mirrored for API
    compatibility; the device QL iteration (csrc/slq.cu) works on the unjittered fp64 tridiagonal -- the difference is below
    the stochastic error of the trace estimate."""
    _global_value = 1e-6


class verbose_linalg(_feature_flag):
    """Log which solver path runs (dense Cholesky vs preconditioned CG, iteration counts) on the 'LinAlg (Verbose)' logger."""
    _default = False
    logger = logging.getLogger("LinAlg (Verbose)")


class deterministic_probes(_feature_flag):
    """Re-use ONE set of probe base samples for every log-det estimate while the flag is on (upstream: the probe vectors are
    stored on the class).  Here the class stores the seed the base samples are drawn from."""
    _default = False
    seed = None

    def __enter__(self):
        if self._value and deterministic_probes.seed is None:
            import torch
            deterministic_probes.seed = int(torch.randint(0, 2**31 - 1, (1,)).item())
        return super().__enter__()

    def __exit__(self, *exc):
        out = super().__exit__(*exc)
        if not deterministic_probes._overrides:
            deterministic_probes.seed = None
        return out


class fast_computations:
    """fast_computations(covar_root_decomposition=True, log_prob=True, solves=True): switch the Krylov paths off individually --
    with log_prob / solves off the dense Cholesky branch runs whatever the size (the reference's max_cholesky_size branch), with
    covar_root_decomposition off LOVE's Lanczos root is replaced by the Cholesky inverse root."""

    class covar_root_decomposition(_feature_flag):
        _default = True

    class log_prob(_feature_flag):
        _default = True

    class solves(_feature_flag):
        _default = True

    def __init__(self, covar_root_decomposition=True, log_prob=True, solves=True):
        self._ctx = (fast_computations.covar_root_decomposition(covar_root_decomposition), fast_computations.log_prob(log_prob),
                     fast_computations.solves(solves))

    def __enter__(self):
        for c in self._ctx:
            c.__enter__()
        return self

    def __exit__(self, *exc):
        for c in reversed(self._ctx):
            c.__exit__(*exc)
        return False


# ---- engine-specific knobs (no reference counterpart) ----
class backend(_value_context):
    """'auto' | 'tcgen05' | 'simt': which fused K.V kernel the engine runs."""
    _global_value = "auto"


class ski_preconditioner(_feature_flag):
    """Precondition solves of a SKI / KISS-GP operator (GridInterpolationKernel) with the pivoted-Cholesky preconditioner of the
    dense kernels (same knobs: max_preconditioner_size, min_preconditioning_size, preconditioner_tolerance).  The pivoted
    Cholesky reads exact entries of K_ski = s W K_uu W^T from its separable form (csrc/ski_rows.cuh); the N(0, P) probes, mBCG
    with the preconditioner, the prediction mean cache and, with ciq_preconditioner, the split-preconditioned CIQ sampler then
    pick it up as they do for dense kernels.  Off by default because turning it on changes results of existing SKI runs: the
    probe distribution and the log-det estimator of the MLL, and the root that preconditioned CIQ applies to xi.  Whether the
    reference preconditions interpolated operators by default is not established here."""
    _default = False


class ski_grid_prediction(_feature_flag):
    """Predict from a KISS-GP model (ScaleKernel(GridInterpolationKernel(...))) with caches kept on the grid, as the reference's
    InterpolatedPredictionStrategy does (models/exact_prediction_strategies.py:481-827): the mean is mu* + W* c with
    c = s K_uu W^T alpha, the LOVE covariance K**_test - U U^T with U = W* C, C = s K_uu W^T R.  The cost per test point is
    O(4^d J) and does not depend on the training-set size; the test prior is forward(test_x) alone, never the joint train + test
    operator (models._ski_grid_mode lists when it applies and what it falls back to).

    Off by default because a feature may not change existing results: with the flag off, SKI predictions keep the joint path bit
    for bit.  tools/ski_predict_bench.py measures both paths, so that a follow-up can make this path the default and delete the
    SKI branch of the joint path."""
    _default = False


class probe_seed(_value_context):
    """Seed of the base samples for the SLQ probes (None = draw from torch's global CUDA generator)."""
    _global_value = None


# ---- propagation into worker threads (operators.BatchLinearOperator) ----
# The knobs are process-wide class state (as in the reference), so worker threads already see what the calling thread's `with`
# blocks set; snapshot() / restore() make the hand-over explicit and testable: restore re-enters the captured overrides.
def _all_knobs():
    import sys
    seen, todo = [], list(vars(sys.modules[__name__]).values())
    while todo:
        obj = todo.pop()
        if isinstance(obj, type) and obj not in seen:
            if issubclass(obj, _Knob) and obj not in (_Knob, _value_context, _feature_flag):
                seen.append(obj)
            elif obj.__module__ == __name__:
                todo.extend(v for v in vars(obj).values() if isinstance(v, type))
    return seen


def snapshot():
    """{knob class: its current override stack (copied)}."""
    return {k: list(k._overrides) for k in _all_knobs()}


class restore:
    """`with restore(snap):` -- run with the captured overrides innermost, whatever the current thread has entered meanwhile."""

    def __init__(self, snap):
        self.snap = snap
        self._entered = []

    def __enter__(self):
        for knob, stack in self.snap.items():
            if stack:
                ctx = knob(stack[-1])
                # _Knob.__enter__ only (deterministic_probes must not draw a new seed in a worker)
                _Knob.__enter__(ctx)
                self._entered.append(ctx)
        return self

    def __exit__(self, *a):
        for ctx in reversed(self._entered):
            _Knob.__exit__(ctx)
        self._entered = []
        return False
