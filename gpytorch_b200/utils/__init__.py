"""gpytorch.utils subset: grid helpers for KISS-GP models."""
from . import grid  # noqa: F401
