"""gpytorch.utils.grid.ScaleToBounds (utils/grid.py:11-54 of the reference): keeps learned features inside a fixed KISS-GP grid."""
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
