"""fp64 SKI products that scale to N = 10^6 points and M = 10^6 grid nodes, the launch geometry of csrc/ski.cu, and the cases of
tests/test_gpu_ski_scale.py (tests/test_ski_scale_host.py checks all three without a GPU).

Reference.  The pinned pieces of oracle/ski.py (`interpolate` through oracle.ski_predict._interp, `left_t_interp`, `left_interp`,
`kron_toeplitz_matmul`, `grid_toeplitz_columns`) run over row chunks, so that no n x 4^d index array or n x 4^d x t temporary is
formed for the whole point set; W^T V accumulates into the [M, t] grid block chunk by chunk.  Every product also comes as its
majorant: |W| for W, |V| for V, the support pattern S of W (ones on the 4^d nodes of a row) for the weight-error floor, and T_i
itself for |T_i| (all four kernel kinds give T_i >= 0).

Interpolation follows tests/test_gpu_ski_predict.py: the fp32 points are interpolated in fp32 on the fp32 grid axes the plan
is given (the same grid coordinate (x - u_0) / spacing, hence the same first nodes as the plan), then promoted to fp64.  The
Toeplitz factors are evaluated on the grid the plan evaluates them on: u_0 + j * spacing in fp64 from the fp32 first node and
spacing (`regular_axes`), not on the nodes of the fp32 linspace, which sit up to an ulp of 1 away from it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from functools import reduce
from operator import mul

import torch

from oracle import ski
from oracle import ski_predict as osp

ROWS = 65536                 # points per interpolation chunk
TEMP = 1 << 23               # elements of the largest n x 4^d x t (or M x t FFT) temporary

# ---- the chunked reference -----------------------------------------------------------------------------------------------------


def regular_axes(lo, step, sizes):
    """The grid the plan builds its Toeplitz factors on: lo_i + j step_i in fp64 (lo, step the fp32 values given to set_ski)."""
    return [float(a) + float(s) * torch.arange(g, dtype=torch.float64) for a, s, g in zip(lo, step, sizes)]


class Interp:
    """W over row chunks of the points x [n, d]: (first row, indices [r, 4^d], values [r, 4^d] fp64), interpolated in
    `interp_dtype` on the axes `axes` (fp32 by default, as the plan does)."""

    def __init__(self, axes, x, interp_dtype=torch.float32, rows=ROWS):
        self.M = reduce(mul, [int(a.numel()) for a in axes], 1)
        self.n = x.size(0)
        self.nnz = 4 ** x.size(1)
        ax = [a.double() for a in axes]
        self.chunks = [(r0, *osp._interp(ax, x[r0:r0 + rows].double(), interp_dtype)) for r0 in range(0, self.n, rows)]

    def _cols(self, rows, t):
        return max(1, min(t, TEMP // max(1, rows * self.nnz)))

    @staticmethod
    def _vals(val, mode):
        return val if mode == "w" else (val.abs() if mode == "abs" else torch.ones_like(val))

    def node_counts(self):
        """m_node [M]: how many points have the node among their 4^d interpolation nodes (one-hot rows count all 4^d)."""
        m = torch.zeros(self.M, dtype=torch.float64)
        for _, idx, _ in self.chunks:
            m += torch.bincount(idx.reshape(-1), minlength=self.M).double()
        return m

    def wt(self, V, mode="w"):
        """W^T V [M, t] (mode "w"), |W|^T V ("abs") or S^T V ("support") for V [n, t] fp64."""
        out = torch.zeros(self.M, V.size(1), dtype=torch.float64)
        for r0, idx, val in self.chunks:
            vv = self._vals(val, mode)
            c = self._cols(idx.size(0), V.size(1))
            for c0 in range(0, V.size(1), c):
                out[:, c0:c0 + c] += ski.left_t_interp(idx, vv, V[r0:r0 + idx.size(0), c0:c0 + c], self.M)
        return out

    def w(self, Cg, mode="w"):
        """W Cg [n, t] (mode "w"), |W| Cg ("abs") or S Cg ("support") for grid values Cg [M, t] fp64."""
        out = torch.empty(self.n, Cg.size(1), dtype=torch.float64)
        for r0, idx, val in self.chunks:
            vv = self._vals(val, mode)
            c = self._cols(idx.size(0), Cg.size(1))
            for c0 in range(0, Cg.size(1), c):
                out[r0:r0 + idx.size(0), c0:c0 + c] = ski.left_interp(idx, vv, Cg[:, c0:c0 + c])
        return out


def toeplitz_columns(kind, axes, lengthscale, deriv_dim=None):
    """First columns of T_0 .. T_{d-1} (oracle.ski.grid_toeplitz_columns); with deriv_dim = i the factor of dimension i is
    l dT_i/dl (the derivative factor the plan's hyper-parameter gradient sweeps), by automatic differentiation in fp64."""
    ls = torch.as_tensor(lengthscale, dtype=torch.float64).reshape(-1)
    cols = ski.grid_toeplitz_columns(kind, axes, ls if ls.numel() > 1 else ls[0])
    if deriv_dim is None:
        return cols
    i = deriv_dim
    li = ls[0] if ls.numel() == 1 else ls[i]
    # T_i depends on l_i alone: l_i dT_i/dl_i = d/de T_i(l_i e^e) at e = 0 (reverse mode, one pass per entry)
    cols[i] = torch.autograd.functional.jacobian(lambda e: ski.grid_toeplitz_columns(kind, [axes[i]], li * torch.exp(e))[0],
                                                 torch.zeros((), dtype=torch.float64))
    return cols


def kuu(cols, Z):
    """(T_0 x ... x T_{d-1}) Z for grid blocks Z [M, t] (oracle.ski.kron_toeplitz_matmul over column groups)."""
    M = Z.size(0)
    c = max(1, TEMP // (4 * M))
    return torch.cat([ski.kron_toeplitz_matmul(cols, Z[:, c0:c0 + c]) for c0 in range(0, Z.size(1), c)], 1)


def ski_matmul(kind, x, axes, toeplitz_axes, lengthscale, outputscale, V, interp_dtype=torch.float32):
    """(s W K_uu W^T V, s |W| K_uu |W|^T |V|) over row chunks, both fp64."""
    W = Interp(axes, x, interp_dtype)
    cols = toeplitz_columns(kind, toeplitz_axes, lengthscale)
    V = V.double()
    out = W.w(kuu(cols, W.wt(V)))
    mag = W.w(kuu([c.abs() for c in cols], W.wt(V.abs(), "abs")), "abs")
    return outputscale * out, outputscale * mag


# ---- launch geometry of csrc/ski.cu (ski_bucket_points, ski_tiled_pass, ski_mode_products, ski_mode_kernel) ---------------------
EDGE_BY_D = {1: 64, 2: 16, 3: 4, 4: 2}


def cdiv(a, b):
    return -(-a // b)


def tile_geometry(sizes):
    """(tile edge in cells, tiles per dimension) of the point bucketing."""
    E = EDGE_BY_D[len(sizes)]
    return E, [max(1, cdiv(g - 3, E)) for g in sizes]


def launch_geometry(sizes, n, n_sm):
    """What one product launches: tiles, parts per tile, work items and grid of the tiled passes, largest tile block, and per
    mode the slab count, the mode kernel's grid and its 16-row tiles (nmt)."""
    E, nt = tile_geometry(sizes)
    ntiles = math.prod(nt)
    parts = min(1024, max(1, cdiv(n // ntiles, 256)))
    items = ntiles * parts
    M = math.prod(sizes)
    modes = []
    for g in sizes:
        total = M // g * 16
        modes.append(dict(G=g, nslab=cdiv(total, 64), tail=total % 64, grid=min(cdiv(total, 64), 2 * n_sm), nmt=cdiv(g, 16),
                          GK=cdiv(g, 8) * 8))
    return dict(E=E, nt=nt, ntiles=ntiles, parts=parts, items=items, grid=min(items, 16 * n_sm),
                block_nodes=math.prod(min(E + 3, g) for g in sizes), modes=modes)


def first_nodes(x, lo, step, sizes):
    """The plan's first interpolation node per point and dimension (ski_axis_weights: fp32 grid coordinate, one-hot cells
    clamped to 0 / G - 4), int64 [n, d]."""
    xs = x.float()
    f = []
    for i, g in enumerate(sizes):
        t = (xs[:, i] - torch.tensor(lo[i], dtype=torch.float32)) / torch.tensor(step[i], dtype=torch.float32)
        f.append((torch.floor(t).long() - 1).clamp(0, g - 4))
    return torch.stack(f, 1)


def tile_counts(x, lo, step, sizes):
    """Points per tile, in the plan's tile order (dimension 0 slowest)."""
    E, nt = tile_geometry(sizes)
    f = first_nodes(x, lo, step, sizes)
    t = torch.zeros(x.size(0), dtype=torch.long)
    for i in range(len(sizes)):
        t = t * nt[i] + f[:, i] // E
    return torch.bincount(t, minlength=math.prod(nt))


def empty_parts(counts, parts):
    """Work items (tile, part) whose point range [p0, p1) is empty (ski_work_range)."""
    k = torch.arange(parts)
    p0 = counts.unsqueeze(1) * k // parts
    p1 = counts.unsqueeze(1) * (k + 1) // parts
    return int((p0 == p1).sum())


# ---- the cases ------------------------------------------------------------------------------------------------------------------
def bench_grid(sizes):
    """GridInterpolationKernel(grid_size, grid_bounds=[(0, 1)]^d) as bench.py builds it for the plan: fp32 linspace axes extended
    by one cell, the plan given the first node and the fp32 spacing of the first cell."""
    axes = [torch.linspace(0.0 - 1.0 / (g - 2), 1.0 + 1.0 / (g - 2), g) for g in sizes]
    return axes, [float(a[0]) for a in axes], [float(a[1] - a[0]) for a in axes]


@dataclass
class Case:
    name: str
    sizes: list
    n: int
    kind: str
    ls: float
    reaches: list                       # paths of launch_geometry this case must reach (test_ski_scale_host.py)
    points: str = "uniform"
    t: list = field(default_factory=lambda: [2])
    grads: bool = False                 # also bilinear_grad and ski_input_grad
    seed: int = 0
    outputscale: float = 1.25


CASES = [
    Case("c5", [100, 100, 100], 1_000_000, "rbf", 0.2, ["scan_carry", "cta_reuse", "slab_stride", "mode_pairs", "last_pair_single"],
         outputscale=1.0),
    Case("g100_matern", [100, 100, 100], 200_000, "matern52", 0.15,
         ["scan_carry", "cta_reuse", "slab_stride", "mode_pairs", "last_pair_single", "v16_chunks"], t=[1, 16, 17, 33], grads=True,
         seed=1),
    Case("g65_97_7", [65, 97, 7], 200_000, "matern32", 0.2, ["mode_pairs", "slab_tails", "parts"], t=[3], seed=2),
    Case("g128_d2", [128, 128], 1_000_000, "rbf", 0.1, ["g128", "cta_reuse_parts"], seed=3),
    Case("g128x4_crowded", [128, 4], 200_000, "matern12", 0.3, ["g128", "g4", "parts"], t=[5], seed=4),
    Case("g128_d1_crowded", [128], 600_000, "rbf", 0.05, ["g128", "parts_cap"], t=[2], seed=5),
    Case("g20_d4", [20, 20, 20, 20], 200_000, "rbf", 0.3, ["d4", "cta_reuse", "slab_stride"], t=[2], grads=True, seed=6),
    Case("g4_d4", [4, 4, 4, 4], 1000, "matern52", 0.5, ["d4"], t=[3], seed=7),
    Case("clustered_d2", [128, 128], 200_000, "matern52", 0.1, ["g128", "empty_tiles", "one_point_tiles", "empty_parts"],
         points="clustered", t=[3], grads=True, seed=8),
    Case("clustered_d3", [100, 100, 100], 100_000, "rbf", 0.2, ["empty_tiles", "one_point_tiles", "cta_reuse"], points="clustered",
         t=[2], seed=9),
    Case("tile_edges_d2", [70, 70], 20_000, "rbf", 0.1, ["tile_edges"], points="tile_edges", t=[3], seed=10),
    Case("tile_edges_d3", [38, 38, 38], 20_000, "matern32", 0.2, ["tile_edges"], points="tile_edges", t=[3], seed=11),
    Case("tile_edges_d4", [12, 12, 12, 12], 20_000, "rbf", 0.4, ["tile_edges", "d4"], points="tile_edges", t=[3], seed=12),
]


def case_points(case):
    """(x fp32 [n, d], fp32 axes, lo, step) of a case, all points inside [0, 1)^d: never in the one-hot first / last cells."""
    axes, lo, step = bench_grid(case.sizes)
    d, n = len(case.sizes), case.n
    g = torch.Generator().manual_seed(case.seed)
    if case.points == "uniform":
        return torch.rand(n, d, generator=g), axes, lo, step
    E, nt = tile_geometry(case.sizes)
    st = torch.tensor(step, dtype=torch.float64)
    lo_t = torch.tensor(lo, dtype=torch.float64)

    def in_cells(cells, frac):   # points in grid cells `cells` [m, d] (first node = cell - 1) at fractions frac of a cell
        return (lo_t + (cells.double() + frac) * st).float()

    if case.points == "clustered":
        # all but 40 points in the tile (2, .., 2); single points and pairs in distant tiles; every other tile empty
        base = torch.tensor([2 * E + 1] * d)                 # first node 2 E: tile 2 in every dimension
        x = in_cells(base + torch.randint(0, E, (n, d), generator=g), 0.05 + 0.9 * torch.rand(n, d, generator=g, dtype=torch.float64))
        cluster = sum(2 * math.prod(nt[i + 1:]) for i in range(d))
        tiles = [t for t in torch.randperm(math.prod(nt), generator=g).tolist() if t != cluster][:20]
        far = []
        for t in tiles:                                      # tile index -> first node k E of its tile in every dimension
            c = []
            for m in reversed(nt):
                c.append(t % m * E + 1)
                t //= m
            far.append(c[::-1])
        far = torch.tensor(far)
        far = torch.cat([far, far[:10]], 0)                  # ten of the 20 tiles hold two points, the others one
        x[:30] = in_cells(far, 0.05 + 0.9 * torch.rand(30, d, generator=g, dtype=torch.float64))
        return x, axes, lo, step
    # tile_edges: every coordinate in a cell whose first node is k E - 1 or k E (the cells on both sides of a tile boundary)
    cells = []
    for i, m in enumerate(case.sizes):
        ks = torch.arange(1, nt[i] + 1) * E
        cand = torch.cat([ks - 1, ks])                       # first nodes k E - 1, k E
        cand = cand[cand <= m - 4]                           # first node G - 3 is the one-hot last cell
        cells.append(cand[torch.randint(0, cand.numel(), (n,), generator=g)] + 1)
    return in_cells(torch.stack(cells, 1), 0.02 + 0.96 * torch.rand(n, d, generator=g, dtype=torch.float64)), axes, lo, step
