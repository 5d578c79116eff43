"""Host checks of the fused K.V kernels' oracle (tests/kmv_oracle.py): the fp64 product against oracle.kernels and against the
reference's own matrices (tests/golden/kernels_golden.npz); the geometry mirror against DESIGN's ring-depth table, and every case
of test_gpu_kmv.py still reaching its edge on 132 SMs (H100 SXM) and 114 SMs (H100 PCIe); and the bound tight enough that
deliberately wrong engines, built in fp64 on the GPU test's own cases, fall outside it in at least one entry."""
import pytest
import torch

import bilinear_oracle as bo
import kmv_oracle as ko
from oracle import kernels as ok

KINDS = list(bo.KINDS)
N_SMS = (132, 114)
GOLD_NAMES = {"rbf": "rbf", "matern12": "mat12", "matern32": "mat32", "matern52": "mat52"}


# ---- the fp64 product ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("geom", ["cross", "square", "shard"])
def test_exact_matches_dense_kernel_matrix(kind, geom):
    g = torch.Generator().manual_seed(7 + KINDS.index(kind))
    x1, x2 = torch.rand(90, 4, generator=g), torch.rand(70, 4, generator=g)
    same = geom != "cross"
    rb, rc = (17, 40) if geom == "shard" else (0, None)
    cols = x1 if same else x2
    V = torch.randn(cols.size(0), 5, generator=g, dtype=torch.float64)
    ls, os_, nz = float(bo.f32(0.55)), float(bo.f32(1.3)), float(bo.f32(0.1))
    K = ok.kernel_matrix(kind, x1.double(), cols.double(), ls, os_, same)
    want = K @ V + (nz * V if same else 0)
    got = ko.exact(kind, x1, None if same else x2, 0.55, 1.3, 0.1, V, same=same, row_begin=rb, row_count=rc)
    torch.testing.assert_close(got, want[rb:rb + (rc or 90)], rtol=1e-12, atol=1e-12)


def test_exact_matches_reference_goldens(golden):
    """V = I: the reference's own fp64 kernel matrices, outputscale 1.  The oracle holds the lengthscale in fp32 as the engine
    does, 3e-8 relative from the golden's fp64 value, which moves an entry by at most m 6e-8 of it."""
    for tag in "abcd":
        x1 = torch.from_numpy(golden[f"{tag}_f64_x1"]); x2 = torch.from_numpy(golden[f"{tag}_f64_x2"])
        same = bool(golden[f"{tag}_f64_same"])
        ls = float(golden[f"{tag}_f64_ls"])
        I = torch.eye(x2.size(0), dtype=torch.float64)
        for kind, nk in GOLD_NAMES.items():
            want = torch.from_numpy(golden[f"{tag}_f64_{nk}"])
            got = ko.exact(kind, x1, None if same else x2, ls, 1.0, 0.0, I, same=same)
            torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-7, msg=f"{tag} {kind}")


# ---- geometry -----------------------------------------------------------------------------------------------------------------
def test_ring_depth_table():
    """DESIGN section 4.1: 12 stages at KP <= 32, 11 at 40, 8 at 64, 4 at 128."""
    assert {kp: ko.ring_depth(kp) for kp in ko.KP_D} == {8: 12, 16: 12, 24: 12, 32: 12, 40: 11, 64: 8, 96: 5, 128: 4}
    assert all(bo.kp_of(d) == kp for kp, d in ko.KP_D.items())
    assert [bo.dp_of(d) for d in ko.SIMT_D] == [4, 8, 12, 16, 24, 32, 48, 64, 96, 128]


@pytest.mark.parametrize("n_sm", N_SMS)
def test_gpu_cases_reach_their_edges(n_sm):
    # ring depths: one split of exactly T tiles, T at every edge of the NS-deep ring
    for d, T, n1, n2 in ko.ring_cases() + ko.large_row_cases():
        geo = ko.geometry(n1, n2, d, "tcgen05", n_sm)
        assert (geo["nsplit"], geo["T"]) == (1, T), (d, T, n1, n2, geo)
    seen = {(ko.geometry(n1, n2, d, "tcgen05", n_sm)["KP"], T) for d, T, n1, n2 in ko.ring_cases()}
    assert seen == {(kp, T) for kp in ko.RING_KP for T in ko.ring_T(ko.ring_depth(kp))}
    for d, T, n1, n2 in ko.large_row_cases():   # several waves of CTAs
        assert ko.geometry(n1, n2, d, "tcgen05", n_sm)["ntile_i"] > 2 * n_sm
    # a square plan with several splits and a shorter last one
    n, d = ko.SPLIT_SQUARE
    geo = ko.geometry(n, n, d, "tcgen05", n_sm)
    assert geo["nsplit"] > 1 and geo["T_last"] < geo["T"], geo
    # SIMT: the last split of the cps edge holds one column
    n1, n2, d = ko.CPS_EDGE
    geo = ko.geometry(n1, n2, d, "simt", n_sm)
    assert geo["nsplit"] > 1 and n2 % geo["cps"] == 1, geo
    # shards: the diagonal crosses 64-column tiles, and on two of them the start of a split with jt0 != 0
    crossing = 0
    for rb, rc in ko.SHARDS:
        geo = ko.geometry(ko.SHARD_N, ko.SHARD_N, 3, "tcgen05", n_sm, rc)
        starts = [s * geo["T"] * ko.TILE_J for s in range(1, geo["nsplit"])]
        crossing += any(rb < c < rb + rc for c in starts)
        assert rb // 64 != (rb + rc - 1) // 64 or rc <= 64
    assert crossing >= 2
    # row edges: rows n1 <= 64 leave consumer 1 only padding rows; every column edge is one partial tile
    assert all(ko.geometry(n1, 65, 3, "tcgen05", n_sm)["rows_pad"] == 256 for n1 in ko.N1_EDGES[:3])
    assert all(ko.geometry(64, n2, 3, "tcgen05", n_sm)["nsplit"] == 1 for n2 in ko.N2_EDGES)


# ---- the bound has teeth ------------------------------------------------------------------------------------------------------
def _outside(kind, x1, x2, ls, os_, noise, V, path, geo, same=False, rb=0, rc=None, **mut):
    true = ko.exact(kind, x1, x2, ls, os_, noise, V, same=same, row_begin=rb, row_count=rc)
    wrong = ko.exact(kind, x1, x2, ls, os_, noise, V, same=same, row_begin=rb, row_count=rc, **mut)
    bnd = ko.bound(kind, x1, x2, ls, os_, noise, V, path, geo["nsplit"], geo["T"], same=same, row_begin=rb, row_count=rc)
    return bool(((true - wrong).abs() > bnd).any())


def _ring_case(kp, T, kind):
    """test_gpu_kmv.test_ring_edges_within_bound's inputs for (KP, T)."""
    d, T, n1, n2 = next(c for c in ko.ring_cases() if c[0] == ko.KP_D[kp] and c[1] == T)
    x1, x2 = ko.points(n1, d, 10 + T), ko.points(n2, d, 20 + T)
    V = torch.randn(n2, 17, generator=torch.Generator().manual_seed(T))
    return (kind, x1, x2, 0.5 * d ** 0.5, 1.3, 0.1, V), ko.geometry(n1, n2, d, "tcgen05")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mutant", ["p_lo", "v_lo", "order", "os_twice", "noise_cross"])
def test_arithmetic_mutants_are_outside_the_bound(kind, mutant):
    args, geo = _ring_case(8, 13, kind)
    arg = 0.1 if mutant == "noise_cross" else None
    assert _outside(*args, "tc", geo, mutant=mutant, mutant_arg=arg)


@pytest.mark.parametrize("kp", ko.RING_KP)
@pytest.mark.parametrize("factor", [0.0, 2.0])
def test_skipped_or_doubled_ring_tile_on_one_cta_is_outside_the_bound(kp, factor):
    """A stage read one phase late drops a tile or counts one twice: the first tile of the second ring pass, in row tile 1 only."""
    NS = ko.ring_depth(kp)
    args, geo = _ring_case(kp, NS + 1, KINDS[kp % 4])
    assert _outside(*args, "tc", geo, mutant="tile", mutant_arg=(1, NS, factor))


def _shard_args(rb, rc, kind, t=17):
    x = ko.points(ko.SHARD_N, 3, 5)
    V = torch.randn(ko.SHARD_N, t, generator=torch.Generator().manual_seed(rb))
    return (kind, x, None, 0.5, 1.3, 0.1, V), ko.geometry(ko.SHARD_N, ko.SHARD_N, 3, "tcgen05", 132, rc)


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("kind", KINDS)
def test_wrong_diagonal_masks_and_noise_are_outside_the_bound(path, kind):
    for rb, rc in ko.SHARDS[1:]:
        args, geo = _shard_args(rb, rc, kind)
        kw = dict(same=True, rb=rb, rc=rc)
        assert _outside(*args, path, geo, **kw, mutant="diag_shift"), (rb, rc)
        assert _outside(*args, path, geo, **kw, mutant="diag_local"), (rb, rc)
        assert _outside(*args, path, geo, **kw, mutant="noise_twice"), (rb, rc)


def test_missing_mask_on_a_later_split_is_outside_the_bound_on_matern12():
    """The unmasked diagonal of the tensor-core path: a_ii from the 3xTF32 GEMM, off from 0 by up to the bound's own da, which
    Matern-1/2 turns into sqrt(da).  With V = identity columns on the diagonal (test_gpu_kmv's single-entry case) one entry is
    the pair, and the bound catches it for Matern-1/2.  For RBF the change is ln2 da, inside the bound: the exactness check
    there (a diagonal entry equals fp32(outputscale) bit for bit) is what catches a missing mask."""
    rb, rc = 400, 300
    x = ko.points(ko.SHARD_N, 3, 5)
    geo = ko.geometry(ko.SHARD_N, ko.SHARD_N, 3, "tcgen05", 132, rc)
    first = geo["T"] * ko.TILE_J                                     # first column of split 1 (jt0 != 0)
    V, cols = ko.identity_cols(ko.SHARD_N, [first, first + 1, first + 63, first + 64, rb + rc - 1])
    args = ("matern12", x, None, 0.6, 1.2, 0.0, V)
    assert _outside(*args, "tc", geo, same=True, rb=rb, rc=rc, mutant="diag_da", mutant_arg=first)
    # the same mutant on the same entries stays inside the RBF bound: the bit-exact diagonal check is needed there
    args = ("rbf", x, None, 0.6, 1.2, 0.0, V)
    assert not _outside(*args, "tc", geo, same=True, rb=rb, rc=rc, mutant="diag_da", mutant_arg=first)


@pytest.mark.parametrize("kind", KINDS)
def test_dropped_n_lo_on_spread_inputs_is_outside_the_bound(kind):
    """test_gpu_kmv's spread 1-D case: |z|^2 up to 4e3, where n_lo carries up to 2^-11 |n| ~ 1 of the argument."""
    x = ko.spread_points(1500, 1, kind, 3, 4e3)
    V = torch.randn(1500, 3, generator=torch.Generator().manual_seed(4))
    geo = ko.geometry(1500, 1500, 1, "tcgen05", 132)
    assert _outside(kind, x, None, 1.0, 1.0, 0.0, V, "tc", geo, same=True, mutant="n_lo")


def test_spread_inputs_reach_the_stated_norms():
    for kind in KINDS:
        for d, z2 in ((1, 4e3), (3, 4e3), (41, 1e3)):
            x = ko.spread_points(1000, d, kind, 3, z2)
            z = (x.double() - x.double().mean(0)) * (bo._C[kind] ** 0.5)
            assert 0.5 * z2 < (z * z).sum(1).max() < 2.5 * z2, (kind, d)
