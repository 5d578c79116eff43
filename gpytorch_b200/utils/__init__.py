"""gpytorch.utils subset: grid helpers for KISS-GP models and sum_interaction_terms for additive GPs."""
from . import grid  # noqa: F401
from .interaction import sum_interaction_terms  # noqa: F401
