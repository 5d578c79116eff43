"""gpytorch.utils.grid subset of the reference (utils/grid.py): ScaleToBounds (lines 11-54) keeps learned features inside a fixed
KISS-GP grid, choose_grid_size (lines 80-100) sizes a grid from the training set."""
import math

import torch


class ScaleToBounds(torch.nn.Module):
    """Maps its input affinely so that the training batch spans 95 % of [lower_bound, upper_bound]:
    y = (x - min) * 0.95 (upper - lower) / (max - min) + 0.95 lower, with one global min / max over all entries.

    In training mode min and max come from the current batch (gradients flow through them) and are stored; in eval mode the stored
    values are used and x is first clamped to [min, max], so test features never leave the grid.  Deep kernel learning puts it
    between the network and a GridInterpolationKernel with grid_bounds (lower, upper)."""

    def __init__(self, lower_bound, upper_bound):
        super().__init__()
        self.lower_bound = float(lower_bound)
        self.upper_bound = float(upper_bound)
        self.register_buffer("min_val", torch.tensor(lower_bound))
        self.register_buffer("max_val", torch.tensor(upper_bound))

    def forward(self, x):
        if self.training:
            lo, hi = x.min(), x.max()
            self.min_val.data = lo
            self.max_val.data = hi
        else:
            lo, hi = self.min_val, self.max_val
            x = x.clamp(lo, hi)
        span = 0.95 * (self.upper_bound - self.lower_bound)
        return (x - lo) * (span / (hi - lo)) + 0.95 * self.lower_bound


def choose_grid_size(train_inputs, ratio=1.0, kronecker_structure=True):
    """utils/grid.py:80-100 of the reference: a KISS-GP grid size for training inputs x ([n] or [..., n, d]).  With Kronecker
    structure (the default) every dimension gets int(ratio * n^(1/d)) nodes, so that the grid has about ratio * n nodes in all;
    without it, ratio * n.  The SKI backend accepts 4 to 131072 nodes per dimension."""
    num_data = train_inputs.numel() if train_inputs.dim() == 1 else train_inputs.size(-2)
    num_dim = 1 if train_inputs.dim() == 1 else train_inputs.size(-1)
    if kronecker_structure:
        return int(ratio * math.pow(num_data, 1.0 / num_dim))
    return ratio * num_data
