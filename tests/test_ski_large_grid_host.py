"""CPU checks of the large-grid SKI pieces (tests/ski_large_grid_oracle.py): the fp64 Toeplitz product from the generating column
against the dense oracle, the band ends of the fp32 columns against where expf underflows, the banded mode kernel's launch geometry
and the paths the GPU cases reach, the kernel's machine code, and utils.grid.choose_grid_size."""
import math
import os
import shutil
import subprocess

import pytest
import torch

import ski_large_grid_oracle as lo
from oracle import ski

KINDS = ["rbf", "matern12", "matern32", "matern52"]


@pytest.mark.parametrize("G", [4, 129, 193, 300])
@pytest.mark.parametrize("kind", KINDS)
def test_generating_column_product_matches_dense_oracle(G, kind):
    axis = torch.linspace(-0.1, 1.1, G, dtype=torch.float64)
    col = ski.grid_toeplitz_columns(kind, [axis], 0.07)[0]
    Z = torch.randn(G, 3, generator=torch.Generator().manual_seed(G), dtype=torch.float64)
    dense = torch.stack([col[(torch.arange(G) - a).abs()] for a in range(G)])
    ref = dense @ Z
    for got in (lo.toeplitz_apply(col, Z), lo.toeplitz_apply_fft(col, Z), ski.kron_toeplitz_matmul([col], Z)):
        assert float((got - ref).abs().max()) <= 1e-12 * float((dense.abs() @ Z.abs()).max())


def test_banded_sum_skips_exact_zeros_only():
    col = torch.tensor([1.0, 0.5, 0.0, 0.25, 0.0, 0.0], dtype=torch.float64)
    Z = torch.randn(6, 2, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    assert torch.allclose(lo.toeplitz_apply(col, Z), lo.toeplitz_apply_fft(col, Z), rtol=0, atol=1e-14)
    assert lo.band_end(col) == 4 and lo.band_end(torch.zeros(5)) == 0
    assert lo.band_end(torch.tensor([1.0, float("nan"), 0.0])) == 2    # NaN counts as non-zero: nothing is skipped around it


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("G,ls", [(1000, 0.01), (4097, 0.002), (131072, 1e-4), (200, 5.0)])
def test_band_end_is_where_fp32_expf_underflows(kind, G, ls):
    step = 1.0 / (G - 3)
    col = lo.column_fp32(kind, G, step, ls)
    b = lo.band_end(col)
    assert (col[b:] == 0).all() and (b == 0 or col[b - 1] != 0)
    ub = lo.underflow_band(kind, G, step, ls)
    assert abs(b - ub) <= 1, (b, ub)                 # the last ulp of the argument decides the boundary entry
    db = lo.band_end(lo.column_fp32(kind, G, step, ls, deriv=True))
    assert db <= b                                   # l dt/dl = (polynomial in r) * the same exponential: zero where t is


def test_banded_geometry_formulas():
    g = lo.banded_geometry(4097, 852, 16, 132)
    assert g["nrb"] == 33 and g["nslab"] == 1 and g["items"] == 33 and g["grid"] == 33
    assert g["partial_chunk"] and g["partial_rows"] and g["slab_tail"]   # d = 1: 16 positions in a 64-wide slab
    # row block 0 runs k in [0, 128 + 851): chunks 0 .. 30; the middle blocks 2 * ceil(851 / 32) + 4 or 5 chunks
    assert g["runs"][0] == math.ceil((128 + 851) / 32)
    assert g["skipped_chunks"] == sum(math.ceil(4097 / 32) - r for r in g["runs"])
    full = lo.banded_geometry(192, 192, 16, 132)
    assert full["skipped_chunks"] == 0 and full["runs"] == [6, 6]
    none = lo.banded_geometry(300, 0, 16, 132)
    assert none["runs"] == [0, 0, 0]                 # band 0: every row written as 0, no chunk runs
    assert lo.banded_geometry(1000, 464, 1000 * 16, 132)["items"] == 250 * 8
    assert lo.k_active(131072, 19) == 128 + 36 + 64 and lo.k_active(200, 200) == 200


@pytest.mark.parametrize("case", lo.CASES, ids=lambda c: c.name)
def test_gpu_cases_reach_their_paths(case):
    got = lo.case_paths(case)
    assert set(case.reaches) <= got, (case.name, sorted(got))
    assert all(4 <= g <= lo.MAX_G for g in case.sizes) and math.prod(case.sizes) * 16 < 2 ** 31


def test_gpu_cases_cover_every_path():
    reached = set().union(*(lo.case_paths(c) for c in lo.CASES))
    assert {"skip", "no_skip", "partial_chunk", "partial_rows", "dense_mode", "slab_stride"} <= reached
    bands = {c.name: lo.band_end(lo.column_fp32(c.kind, c.sizes[0], lo.so.bench_grid(c.sizes)[2][0], c.ls)) for c in lo.CASES}
    assert bands["g131072_rbf"] < lo.KC                                  # the band inside one chunk
    assert abs(bands["g1000sq_m52"] - 500) < 50                          # about G / 2
    assert bands["g192_m12_noskip"] == 192                               # no skip at all, Matern-1/2 tail


LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpytorch_b200", "lib", "libgpbbmm.so")


def _cuobjdump(*args):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(LIB):
        pytest.skip("libgpbbmm.so not built (python -m gpytorch_b200.build)")
    r = subprocess.run([tool, *args, LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def test_banded_mode_kernel_is_3xtf32_mma_without_local_memory():
    body, keep = [], False
    for line in _cuobjdump("-sass").splitlines():
        if "Function :" in line:
            keep = "ski_mode_banded_kernel" in line
        elif keep:
            body.append(line)
    assert "HMMA.1688.F32.TF32" in "\n".join(body)
    res = _cuobjdump("-res-usage").splitlines()
    for name in ("ski_mode_banded_kernel", "ski_toeplitz_col_kernel", "ski_krows_kernel", "ski_kdiag_kernel"):
        i = next(k for k, line in enumerate(res) if name in line)
        assert "STACK:0" in res[i + 1] and "LOCAL:0" in res[i + 1], (name, res[i + 1])


def test_choose_grid_size_matches_the_reference_formula():
    from gpytorch_b200.utils.grid import choose_grid_size

    assert choose_grid_size(torch.zeros(1000)) == 1000
    assert choose_grid_size(torch.zeros(100_000, 1)) == 100_000
    assert choose_grid_size(torch.zeros(10 ** 6, 2)) == int(math.pow(10 ** 6, 0.5))
    assert choose_grid_size(torch.zeros(3, 500, 3), ratio=2.0) == int(2.0 * math.pow(500, 1 / 3))
    assert choose_grid_size(torch.zeros(400, 2), ratio=0.5, kronecker_structure=False) == 200.0
    for n, d in [(123, 1), (4567, 2), (89_000, 3), (10 ** 5, 4)]:
        assert choose_grid_size(torch.zeros(n, d)) == int(1.0 * math.pow(n, 1.0 / d))
