"""gpytorch_b200 -- H100-native BBMM exact-GP inference behind the gpytorch kernels / LinearOperator /
ExactMarginalLogLikelihood API surface.  The arithmetic lives in libgpbbmm.so (hand-written sm_90a CUDA,
C ABI in include/gp_bbmm.h); this package is the thin Python host mirroring the reference interface.
"""
from . import _lib, constraints, distributions, functions, kernels, likelihoods, means, mlls, models, operators, settings, utils  # noqa: F401
from ._lib import NanError, NotPSDError, NumericalWarning  # noqa: F401
from .engine import KronPlan, Plan  # noqa: F401
from .functions import inv_quad_logdet, linear_cg, pivoted_cholesky, root_decomposition, solve  # noqa: F401
from .mlls import ExactMarginalLogLikelihood  # noqa: F401

__version__ = "0.1.0"
