"""CPU checks of tests/ski_scale_oracle.py: the chunked fp64 SKI reference against oracle.ski.ski_matmul and a dense
W K_uu W^T, its majorant and node counts against their dense forms, and that every case of tests/test_gpu_ski_scale.py reaches
the csrc/ski.cu paths it is listed for, on 132 SMs (H100 SXM) and on 114 (H100 PCIe)."""
import math
from functools import reduce
from operator import mul

import pytest
import torch

import ski_scale_oracle as so
from oracle import ski


def _dense(axes, x, kind, ls, toeplitz_axes):
    idx, val = ski.interpolate(axes, x)
    M = reduce(mul, [int(a.numel()) for a in axes], 1)
    W = torch.zeros(x.size(0), M, dtype=torch.float64).scatter_add(1, idx, val)
    S = torch.zeros(x.size(0), M, dtype=torch.float64).scatter_add(1, idx, torch.ones_like(val))
    K = torch.ones(1, 1, dtype=torch.float64)
    for c in so.toeplitz_columns(kind, toeplitz_axes, ls):
        g = c.numel()
        K = torch.kron(K, c[(torch.arange(g).unsqueeze(1) - torch.arange(g)).abs()])
    return W, S, K


@pytest.mark.parametrize("d,sizes,kind", [(1, [37], "rbf"), (2, [19, 11], "matern12"), (3, [9, 12, 7], "matern52"),
                                          (4, [6, 5, 7, 5], "matern32")])
def test_chunked_reference_matches_the_oracle_and_the_dense_operator(monkeypatch, d, sizes, kind):
    monkeypatch.setattr(so, "TEMP", 3000)            # several column groups per chunk and per Kronecker product
    g = torch.Generator().manual_seed(d)
    n, t, ls, s = 700, 5, 0.3, 1.7
    lo = [-1.0 / (m - 2) for m in sizes]
    step = [1.0 / (m - 2) for m in sizes]
    axes = so.regular_axes(lo, step, sizes)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    x[:5] = torch.tensor(lo, dtype=torch.float64) + 0.4 * torch.tensor(step, dtype=torch.float64)   # one-hot first cell
    V = torch.randn(n, t, generator=g, dtype=torch.float64)
    W = so.Interp(axes, x, torch.float64, rows=97)
    assert len(W.chunks) == math.ceil(n / 97)
    out, mag = so.ski_matmul(kind, x, axes, axes, ls, s, V, interp_dtype=torch.float64)
    ref = ski.ski_matmul(kind, x, axes, ls, s, V)
    assert float((out - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    Wd, Sd, K = _dense(axes, x, kind, ls, axes)
    dense = s * Wd @ K @ Wd.T @ V
    assert float((out - dense).abs().max()) <= 1e-12 * float(dense.abs().max())
    dmag = s * Wd.abs() @ K @ Wd.abs().T @ V.abs()
    assert float((mag - dmag).abs().max()) <= 1e-12 * float(dmag.abs().max())
    assert (mag >= out.abs() * (1 - 1e-12)).all()
    # the grid-side pieces the GPU bounds use
    assert torch.allclose(W.wt(V.abs(), "support"), Sd.T @ V.abs(), rtol=1e-12, atol=0)
    C = torch.randn(Wd.size(1), 3, generator=g, dtype=torch.float64)
    assert torch.allclose(W.w(C), Wd @ C, rtol=1e-12, atol=1e-12 * float(C.abs().max()))
    assert torch.allclose(W.w(C.abs(), "support"), Sd @ C.abs(), rtol=1e-12, atol=0)
    assert torch.equal(W.node_counts(), torch.bincount(ski.interpolate(axes, x)[0].reshape(-1), minlength=Wd.size(1)).double())


@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32", "matern52"])
def test_derivative_factor_is_l_dT_dl(kind):
    axes = so.regular_axes([-0.1, -0.2], [0.1, 0.2], [12, 9])
    ls, h = 0.35, 1e-6
    for i in range(2):
        dc = so.toeplitz_columns(kind, axes, ls, i)[i]
        fd = (so.toeplitz_columns(kind, axes, ls * (1 + h))[i] - so.toeplitz_columns(kind, axes, ls * (1 - h))[i]) / (2 * h)
        assert torch.allclose(dc, fd, rtol=1e-6, atol=1e-9)
        assert (dc >= 0).all()
    r = (axes[0] - axes[0][0]) / ls
    if kind == "rbf":
        assert torch.allclose(so.toeplitz_columns(kind, axes, ls, 0)[0], r * r * torch.exp(-0.5 * r * r), rtol=1e-13, atol=0)


def test_fp32_interpolation_picks_the_plans_first_nodes():
    """The reference interpolates the fp32 points in fp32 on the axes the plan is given: its first nodes are the plan's."""
    for case in so.CASES[:3] + so.CASES[-3:]:
        x, axes, lo, step = so.case_points(case)
        sel = torch.randperm(case.n, generator=torch.Generator().manual_seed(0))[:5000]
        W = so.Interp(axes, x[sel])
        d = len(case.sizes)
        strides = [math.prod(case.sizes[i + 1:]) for i in range(d)]
        first = sum(so.first_nodes(x[sel], lo, step, case.sizes)[:, i] * strides[i] for i in range(d))
        assert torch.equal(W.chunks[0][1][:, 0], first), case.name


def _reaches(case, n_sm):
    geo = so.launch_geometry(case.sizes, case.n, n_sm)
    modes = geo["modes"]
    x, axes, lo, step = so.case_points(case)
    counts = so.tile_counts(x, lo, step, case.sizes)
    f = so.first_nodes(x, lo, step, case.sizes)
    got = {
        "scan_carry": geo["ntiles"] > 1024,
        "cta_reuse": geo["items"] > geo["grid"],
        "cta_reuse_parts": geo["parts"] > 1 and geo["items"] > geo["grid"],
        "slab_stride": any(m["nslab"] > m["grid"] for m in modes),
        "mode_pairs": any(m["nmt"] >= 5 for m in modes),                       # warps 4..7: row-tile pairs mp = 2, 3
        "last_pair_single": any(m["nmt"] == 7 for m in modes),                 # mp = 3 without its second row tile
        "slab_tails": {48, 16} <= {m["tail"] for m in modes},
        "parts": geo["parts"] > 1,
        "parts_cap": geo["parts"] == 1024 and case.n // geo["ntiles"] > 1024 * 256,
        "g128": any(m["G"] == 128 and m["nmt"] == 8 and m["GK"] == 128 for m in modes),
        "g4": 4 in case.sizes,
        "d4": len(case.sizes) == 4 and geo["block_nodes"] * 32 * 4 <= 96 * 1024,
        "v16_chunks": 1 in case.t and max(case.t) > 32 and any(16 < t < 32 for t in case.t),
        "empty_tiles": bool((counts == 0).any()),
        "one_point_tiles": bool((counts == 1).any()),
        "empty_parts": so.empty_parts(counts[counts > 0], geo["parts"]) > 0,
        "tile_edges": all(bool((f[:, i] == k * geo["E"] - 1).any()) and bool((f[:, i] == k * geo["E"]).any())
                          for i, g in enumerate(case.sizes) for k in range(1, geo["nt"][i]) if k * geo["E"] <= g - 4),
    }
    return geo, got


@pytest.mark.parametrize("case", so.CASES, ids=lambda c: c.name)
def test_cases_reach_their_paths(case):
    for n_sm in (132, 114):
        geo, got = _reaches(case, n_sm)
        missing = [r for r in case.reaches if not got[r]]
        assert not missing, (case.name, n_sm, missing, geo)


def test_c5_geometry_is_the_benchmarks():
    c5 = so.CASES[0]
    assert (c5.sizes, c5.n, c5.kind, c5.ls, c5.outputscale) == ([100, 100, 100], 1_000_000, "rbf", 0.2, 1.0)
    geo = so.launch_geometry(c5.sizes, c5.n, 132)
    assert geo["ntiles"] == 15625 and geo["parts"] == 1 and geo["grid"] == 2112
    assert [m["nslab"] for m in geo["modes"]] == [2500] * 3 and [m["nmt"] for m in geo["modes"]] == [7] * 3
    axes, lo, step = so.bench_grid(c5.sizes)
    ref = [torch.linspace(0.0 - 1.0 / 98, 1.0 + 1.0 / 98, 100)] * 3
    assert all(torch.equal(a, b) for a, b in zip(axes, ref))
