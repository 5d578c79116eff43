"""KISS-GP grids over 128 nodes per dimension (csrc/ski.cu, ski_mode_banded_kernel): an fp64 Toeplitz product from the generating
column, the band end of the fp32 column, the launch geometry of the banded mode kernel, and the cases of
tests/test_gpu_ski_large_grid.py (tests/test_ski_large_grid_host.py checks all of it without a GPU).

The factor T_i[a][b] = t_i[|a - b|] is applied from its first column by a direct banded sum (`toeplitz_apply`: only the offsets
where t is non-zero) and, as a cross-check, by an fp64 FFT (`toeplitz_apply_fft`).  The plan evaluates t in fp32; entries at
|a - b| >= band are exactly 0.0f there (expf underflows), and the banded kernel skips the k-chunks made of such entries only.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

import ski_scale_oracle as so

DENSE_G = 128        # ski_mode_kernel up to here, ski_mode_banded_kernel above
MAX_G = 131072
BR = 128             # SKI_BR: output rows per work item
KC = 32              # SKI_KC: k rows per chunk
MT = 64              # SKI_MT: positions per slab
U = 2.0 ** -24


def toeplitz_apply(col, Z):
    """T Z for T[a][b] = col[|a - b|] (fp64 col [G], Z [G, t]) as a direct sum over the offsets with col != 0."""
    G = col.numel()
    out = col[0] * Z.clone()
    for dl in torch.nonzero(col[1:] != 0).flatten().add(1).tolist():
        out[dl:] += col[dl] * Z[:G - dl]
        out[:G - dl] += col[dl] * Z[dl:]
    return out


def toeplitz_apply_fft(col, Z):
    """T Z through a circulant embedding of length 2 G and an fp64 FFT."""
    G = col.numel()
    c = torch.cat([col, col.new_zeros(1), col[1:].flip(0)])
    f = torch.fft.rfft(c)
    zp = torch.cat([Z, Z.new_zeros(G, Z.size(1))], 0)
    return torch.fft.irfft(f.unsqueeze(1) * torch.fft.rfft(zp, dim=0), n=2 * G, dim=0)[:G]


def column_fp32(kind, G, step, ls, deriv=False):
    """The plan's generating column in fp32, the expression of ski_toeplitz_entry (host expf: the band ends agree with the device's
    wherever the underflow is not decided by the last ulp of the argument)."""
    k = torch.arange(G, dtype=torch.float32)
    r = k * torch.tensor(step, dtype=torch.float32) * torch.tensor(1.0 / ls, dtype=torch.float32)
    if kind == "rbf":
        v = torch.exp(-0.5 * r * r)
        return v * (r * r) if deriv else v
    nu2 = {"matern12": 1.0, "matern32": 3.0, "matern52": 5.0}[kind]
    rho = math.sqrt(nu2) * r
    ex = torch.exp(-rho)
    if kind == "matern12":
        return rho * ex if deriv else ex
    if kind == "matern32":
        return rho * rho * ex if deriv else (1 + rho) * ex
    return (1 + rho) * rho * rho * (1.0 / 3.0) * ex if deriv else (1 + rho + rho * rho * (1.0 / 3.0)) * ex


def band_end(col):
    """1 + the last index with col != 0 (0 if none): the device's band index."""
    nz = torch.nonzero(col != 0).flatten()
    return int(nz[-1]) + 1 if nz.numel() else 0


def underflow_band(kind, G, step, ls):
    """Where fp32 expf underflows to 0 (argument below log(2^-150)): the first k whose exponent argument is past it, from the
    closed form of the argument (-r^2 / 2 for RBF, -sqrt(nu2) r for the Materns, r = k step / l)."""
    x0 = 150 * math.log(2.0)
    if kind == "rbf":
        kmin = math.sqrt(2 * x0) * ls / step
    else:
        nu2 = {"matern12": 1.0, "matern32": 3.0, "matern52": 5.0}[kind]
        kmin = x0 / math.sqrt(nu2) * ls / step
    return min(G, math.floor(kmin) + 1)


def banded_geometry(G, band, outer_inner, n_sm):
    """One banded mode product: work items (slab, row block), the k-chunks each row block runs, and the paths it reaches.
    outer_inner = M / G * 16 positions."""
    nrb = so.cdiv(G, BR)
    nslab = so.cdiv(outer_inner, MT)
    runs, skipped = [], 0
    for rb in range(nrb):
        r0, r1 = rb * BR, min(G, rb * BR + BR)
        klo, khi = max(0, r0 - band + 1), (min(G, r1 + band - 1) if band > 0 else 0)
        ch = list(range(klo // KC * KC, khi, KC)) if klo < khi else []
        runs.append(len(ch))
        skipped += so.cdiv(G, KC) - len(ch)
    return dict(nrb=nrb, nslab=nslab, items=nslab * nrb, grid=min(nslab * nrb, 4 * n_sm), runs=runs, skipped_chunks=skipped,
                partial_chunk=G % KC != 0, partial_rows=G % BR != 0, slab_tail=outer_inner % MT != 0)


def k_active(G, band):
    """Most k rows one output row accumulates over in the banded kernel (the k-chunks that meet [r0 - band + 1, r1 + band - 1))."""
    return min(G, BR + 2 * max(band - 1, 0) + 2 * KC)


# ---- the cases ------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    sizes: list
    n: int
    kind: str
    ls: float
    reaches: list                 # "skip", "partial_chunk", "partial_rows", "no_skip", "dense_mode", "slab_stride"
    t: list = field(default_factory=lambda: [2])
    grads: bool = False
    seed: int = 0
    outputscale: float = 1.25


CASES = [
    Case("g129_rbf", [129], 200_000, "rbf", 0.02, ["skip", "partial_chunk", "partial_rows"], t=[3], grads=True, seed=1),
    Case("g192_m12_noskip", [192], 200_000, "matern12", 0.5, ["no_skip", "partial_rows"], t=[2], seed=2),
    Case("g193_m32", [193], 200_000, "matern32", 0.005, ["skip", "partial_chunk", "partial_rows"], t=[17], seed=3),
    Case("g1000_rbf", [1000], 1_000_000, "rbf", 0.06, ["skip", "partial_chunk", "partial_rows"], t=[2], grads=True, seed=4),
    Case("g4097_m12", [4097], 1_000_000, "matern12", 0.002, ["skip", "partial_chunk", "partial_rows"], t=[2], seed=5),
    Case("g131072_rbf", [131072], 1_000_000, "rbf", 1e-5, ["skip", "slab_stride"], t=[2], grads=True, seed=6),
    Case("g1000sq_m52", [1000, 1000], 1_000_000, "matern52", 0.01, ["skip", "partial_chunk", "partial_rows", "slab_stride"], t=[2],
         seed=7, outputscale=1.0),
    Case("g129x4_m12", [129, 4], 200_000, "matern12", 0.3, ["no_skip", "partial_chunk", "partial_rows", "dense_mode"], t=[5],
         grads=True, seed=8),
    Case("g256x256x64_rbf", [256, 256, 64], 200_000, "rbf", 0.02, ["skip", "dense_mode", "slab_stride"], t=[2],
         seed=9),
    Case("g130x8x8x8_m32", [130, 8, 8, 8], 200_000, "matern32", 0.1, ["no_skip", "partial_chunk", "partial_rows", "dense_mode"],
         t=[2], grads=True, seed=10),
]


def case_grid(case):
    """(x fp32 [n, d] uniform in [0, 1)^d, fp32 axes, lo, step) as bench.py builds a grid over [0, 1]^d."""
    axes, lo, step = so.bench_grid(case.sizes)
    g = torch.Generator().manual_seed(case.seed)
    return torch.rand(case.n, len(case.sizes), generator=g), axes, lo, step


def case_paths(case, n_sm=132):
    """The paths of the mode products one product of the case reaches."""
    _, _, step = so.bench_grid(case.sizes)
    M = math.prod(case.sizes)
    got = set()
    for G, s in zip(case.sizes, step):
        if G <= DENSE_G:
            got.add("dense_mode")
            continue
        b = band_end(column_fp32(case.kind, G, s, case.ls))
        geo = banded_geometry(G, b, M // G * 16, n_sm)
        got.add("skip" if geo["skipped_chunks"] else "no_skip")
        if geo["partial_chunk"]:
            got.add("partial_chunk")
        if geo["partial_rows"]:
            got.add("partial_rows")
        if geo["items"] > geo["grid"]:
            got.add("slab_stride")
    return got
