"""Host checks of tests/multitask_oracle.py: the layout mirrors of tasks.cu and kron.cu against hand-computed layouts on 132 SMs
(H100 SXM) and 114 SMs (H100 PCIe), every case of test_gpu_multitask_edges.py still reaching its edge, the fp64 results
against the dense oracles (tests/hadamard_oracle.py, tests/kron_oracle.py, autograd), and the bounds tight enough that
deliberately wrong layouts, built in fp64 on the GPU test's own inputs, fall outside them in at least one entry."""
import pytest
import torch

import hadamard_oracle as ho
import kmv_oracle as ko
import kron_oracle as kro
import multitask_oracle as mo

N_SMS = (132, 114)


# ---- layout mirrors -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_sm", N_SMS)
def test_segment_splits_by_hand(n_sm):
    """3000 rows (24 row tiles, one wave): 897 columns (15 tiles) is the first segment with 2 splits, 8 + 7; 1025 gives 9 + 8;
    1536 gives 3 x 8.  896 columns (14 tiles) stays one split: two splits of 7 tiles are below the 8-tile minimum."""
    for tc in (True, False):
        assert mo.segment_split(3000, 896, tc, n_sm) == (14, 1)
        assert mo.segment_split(3000, 897, tc, n_sm) == (8, 2)
        assert mo.segment_split(3000, 1025, tc, n_sm) == (9, 2)
        assert mo.segment_split(3000, 1536, tc, n_sm) == (8, 3)
        assert mo.segment_split(3000, 1, tc, n_sm) == (1, 1)


def test_segment_split_depends_on_the_sm_count():
    """30720 rows are 240 row tiles: one wave of 2 CTAs per SM on 132 SMs (one split is best), two waves on 114 SMs, where
    two splits of 8 tiles fill the third wave better."""
    assert mo.segment_split(30720, 1024, True, 132) == (16, 1)
    assert mo.segment_split(30720, 1024, True, 114) == (8, 2)


def test_task_layout_by_hand():
    t = torch.tensor([2, 0, 2, 1, 0, 2])
    off, perm = mo.sort_by_task(t, 4)
    assert off == [0, 2, 3, 6, 6] and perm.tolist() == [1, 4, 3, 0, 2, 5]
    lay = mo.task_layout(t, None, 4, "tcgen05")
    assert lay["seg"] == [0, 64, 128, 192, 192] and lay["nsplit"] == [1, 1, 1, 0] and lay["slot0"] == [0, 1, 2, 3, 3]
    assert lay["slot_task"] == [0, 1, 2] and lay["nslot"] == 3
    assert lay["map2"].tolist() == [1, 4] + [-1] * 62 + [3] + [-1] * 63 + [0, 2, 5] + [-1] * 61
    simt = mo.task_layout(t, None, 4, "simt")
    assert simt["seg"] == [0, 2, 3, 6, 6] and simt["map2"].tolist() == [1, 4, 3, 0, 2, 5]
    assert [c.tolist() for c in simt["slots"]] == [[1, 4], [3], [0, 2, 5]]


def test_reduction_chunks_by_hand():
    lay = mo.task_layout(mo.task_ids(mo.RED_CASES["n4200_straddle"], 1), None, 6, "tcgen05")
    assert mo.dB_chunks(lay) == [(0, 0, 2048, 0, 1), (1, 2048, 4096, 1, 4), (2, 4096, 4200, 4, 5)]


def test_kron_layout_by_hand():
    lay = mo.kron_layout(1450, 1450, 5, 7, 7, "tcgen05", 132)
    assert (lay["nsplit"], lay["T"], lay["T_last"], lay["nchunk"], lay["npad"], lay["nred"]) == (3, 8, 7, 4, 1472, 1)
    assert mo.kron_layout(1450, 1450, 5, 7, 7, "simt", 132)["npad"] == 1450


@pytest.mark.parametrize("n_sm", N_SMS)
def test_gpu_cases_reach_their_edges(n_sm):
    for backend in ("tcgen05", "simt"):
        # products: multi-split segments with a shorter last split, one-column and empty tasks, nslot beyond one slot per task
        for name in ("square", "cross"):
            _, _, t1, t2, T, _ = mo.hadamard_case(name, 0)
            lay = mo.task_layout(t1, t2, T, backend, n_sm)
            assert [lay["nsplit"][b] for b in (0, 1, 2, 3, 4, 5)] == [2, 1, 0, 1, 2, 1], lay["nsplit"]
            assert lay["tps"][0] * ko.TILE_J < 897 < 2 * lay["tps"][0] * ko.TILE_J and lay["tps"][4] == 9
            assert lay["nslot"] > T
            if name == "cross":
                assert lay["off1"][3] == lay["off1"][4] and lay["off2"][3] < lay["off2"][4]   # task 3: columns, no rows
                assert lay["off1"][2] < lay["off1"][3] and lay["off2"][2] == lay["off2"][3]   # task 2: rows, no columns
        # reductions
        edges = {}
        for name, sizes in mo.RED_CASES.items():
            T = len(mo.sizes_list(sizes))
            lay = mo.task_layout(mo.task_ids(sizes, 0), None, T, backend, n_sm)
            ch = mo.dB_chunks(lay)
            off = lay["off1"]
            edges[name] = {
                "straddle": [a for a in range(T) if any(off[a] < r < off[a + 1] for r in (2048, 4096))],
                "starts": [off[a] for a in range(T) if off[a] < off[a + 1] and off[a] in (2048, 4096)],
                "single": [z for z, _, _, lo, hi in ch if lo == hi],
                "nchunk": len(ch), "split": max(lay["nsplit"])}
        assert edges["n2048"]["nchunk"] == 1 and mo.task_layout(mo.task_ids(mo.RED_CASES["n2048"]), None, 5, backend,
                                                                n_sm)["n1"] == 2048
        assert edges["n2049"]["nchunk"] == 2 and edges["n2049"]["straddle"] == [1] and edges["n2049"]["single"] == [1]
        assert edges["n4200_starts"]["starts"] == [2048, 4096] and edges["n4200_starts"]["nchunk"] == 3
        assert edges["n4200_straddle"]["straddle"] == [1, 4]
        assert edges["T32"]["single"] == [1, 2] and edges["T32"]["starts"] == [2048, 4096]
        assert all(e["split"] >= 2 for e in edges.values())
        # Kronecker: 3 splits with a shorter last one, 1 / 2 / 4 / 2 / 1 chunks, dB over 1 / 2 / 3 chunks with 2 splits
        n, d = mo.KRON_SPLIT
        geo = mo.kron_layout(n, n, d, 1, 16, backend, n_sm)
        assert geo["nsplit"] == 3 and geo["T_last"] < geo["T"]
        assert [mo.kron_layout(n, n, d, T, t, backend, n_sm)["nchunk"] for T, t in mo.KRON_TT] == [1, 2, 4, 2, 1]
        assert any((T * t) % 16 for T, t in mo.KRON_TT)
        assert [mo.kron_layout(n1, n2, 3, 3, 6, backend, n_sm)["nred"] for n1, n2 in mo.KRON_RED] == [1, 2, 3]
        assert all(mo.kron_layout(n1, n2, 3, 3, 6, backend, n_sm)["nsplit"] == 2 for n1, n2 in mo.KRON_RED)


def test_tf32_split_keeps_every_nan():
    """The tensor-core V split (tf32_hi, mirrored by kmv_oracle._tf32_round) keeps a NaN.  The rule without the NaN case adds
    half a tf32 ulp to the bits, which carries the payload of CUDA's canonical NaN 0x7fffffff (what kron_mix_kernel's fmaf
    returns for a NaN in V) into the sign bit: -0, so the NaN vanished from the Kronecker product on tensor cores."""
    bits = torch.tensor([0x7FFFFFFF, 0x7FC00000, 0x7F800001, -1, -0x400000], dtype=torch.int32)
    assert torch.isnan(ko._tf32_round(bits.view(torch.float32))).all()
    without = ((bits + 0x1000) & -8192).view(torch.float32)
    assert without[0].item() == 0.0 and torch.signbit(without[0]) and without[3].item() == 0.0
    finite = torch.randn(1000, generator=torch.Generator().manual_seed(1)).float()
    assert torch.equal(ko._tf32_round(finite), ((finite.view(torch.int32) + 0x1000) & -8192).view(torch.float32).double())


# ---- fp64 results against the dense oracles -----------------------------------------------------------------------------------
def _small_hadamard(cross, backend):
    g = torch.Generator().manual_seed(3 + cross)
    n1, n2, T, d = 150, (170 if cross else 150), 4, 3
    x1 = torch.rand(n1, d, generator=g)
    x2 = torch.rand(n2, d, generator=g) if cross else None
    t1 = torch.randint(0, T, (n1,), generator=g)
    t2 = torch.randint(0, T, (n2,), generator=g) if cross else None
    B = mo.random_B(T, 5)
    lay = mo.task_layout(t1, t2, T, backend)
    return x1, x2, t1, t2, T, B, lay, g


@pytest.mark.parametrize("cross", [False, True])
@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32", "matern52"])
def test_hadamard_exact_matches_dense(cross, kind):
    x1, x2, t1, t2, T, B, lay, g = _small_hadamard(cross, "tcgen05")
    xc, tc2 = (x2, t2) if cross else (x1, t1)
    V = torch.randn(xc.size(0), 5, generator=g, dtype=torch.float64)
    nd = torch.rand(x1.size(0), dtype=torch.float64) if not cross else None
    ls, os_ = 0.4, 1.3
    K = ho.hadamard_matrix(kind, x1.double(), xc.double(), t1, tc2, float(ko.bo.f32(ls)), float(ko.bo.f32(os_)), B.double(),
                           not cross)
    want = K @ V + (nd[:, None] * V if nd is not None else 0)
    torch.testing.assert_close(mo.hadamard_exact(kind, x1, x2, B, ls, os_, V, lay, noise_diag=nd), want, rtol=1e-12, atol=1e-12)
    # dB and the hyper-parameter gradients against autograd of the dense form
    L = torch.randn(x1.size(0), 3, generator=g, dtype=torch.float64)
    R = torch.randn(xc.size(0), 3, generator=g, dtype=torch.float64)
    lsv = torch.tensor([float(ko.bo.f32(ls))], dtype=torch.float64, requires_grad=True)
    osv = torch.tensor(float(ko.bo.f32(os_)), dtype=torch.float64, requires_grad=True)
    Bv = B.double().clone().requires_grad_(True)
    F = (L * (ho.hadamard_matrix(kind, x1.double(), xc.double(), t1, tc2, lsv[0], osv, Bv, not cross) @ R)).sum()
    F.backward()
    torch.testing.assert_close(mo.hadamard_dB(kind, x1, x2, ls, os_, L, R, lay), Bv.grad, rtol=1e-10, atol=1e-10)
    gl, gs = mo.hadamard_grad(kind, x1, x2, B, ls, os_, L, R, lay)
    torch.testing.assert_close(gl, lsv.grad, rtol=1e-9, atol=1e-9)
    assert abs(gs - float(osv.grad)) <= 1e-9 * abs(float(osv.grad))


@pytest.mark.parametrize("cross", [False, True])
def test_kron_exact_matches_dense(cross):
    g = torch.Generator().manual_seed(9)
    N1, N2, T, t, d = 40, (30 if cross else 40), 3, 5, 2
    x1 = torch.rand(N1, d, generator=g)
    x2 = torch.rand(N2, d, generator=g) if cross else None
    xc = x2 if cross else x1
    B = mo.random_B(T, 6)
    ls, os_ = float(ko.bo.f32(0.5)), float(ko.bo.f32(1.2))
    V = torch.randn(N2 * T, t, generator=g, dtype=torch.float64)
    K = kro.kron_matrix("matern52", x1.double(), xc.double(), ls, os_, B.double(), not cross)
    want = K @ V + (float(ko.bo.f32(0.1)) * V if not cross else 0)
    torch.testing.assert_close(mo.kron_exact("matern52", x1, x2, B, ls, os_, V, T, t, noise=0.1), want, rtol=1e-12, atol=1e-12)
    L = torch.randn(N1 * T, t, generator=g, dtype=torch.float64)
    lsv = torch.tensor([ls], dtype=torch.float64, requires_grad=True)
    osv = torch.tensor(os_, dtype=torch.float64, requires_grad=True)
    Bv = B.double().clone().requires_grad_(True)
    F = (L * (kro.kron_matrix("matern52", x1.double(), xc.double(), lsv[0], osv, Bv, not cross) @ V)).sum()
    F.backward()
    torch.testing.assert_close(mo.kron_dB("matern52", x1, x2, ls, os_, L, V, T, t), Bv.grad, rtol=1e-10, atol=1e-10)
    gl, gs = mo.kron_grad("matern52", x1, x2, B, ls, os_, L, V, T, t)
    torch.testing.assert_close(gl, lsv.grad, rtol=1e-9, atol=1e-9)
    assert abs(gs - float(osv.grad)) <= 1e-9 * abs(float(osv.grad))


# ---- the bounds have teeth ----------------------------------------------------------------------------------------------------
LS, OS = 0.5, 1.3


def _outside(true, wrong, bnd):
    return bool(((true - wrong).abs() > bnd).any())


def _prod(name, backend, kind):
    x1, x2, t1, t2, T, V = mo.hadamard_case(name, 0)
    B = mo.random_B(T, 1)
    lay = mo.task_layout(t1, t2, T, backend)
    true = mo.hadamard_exact(kind, x1, x2, B, LS, OS, V, lay)
    bnd = mo.hadamard_bound(kind, x1, x2, B, LS, OS, V, lay)
    return (x1, x2, B, V, lay), true, bnd


@pytest.mark.parametrize("backend,kind", [("tcgen05", "rbf"), ("simt", "matern12"), ("tcgen05", "matern32"),
                                          ("simt", "matern52")])
def test_hadamard_layout_mutants_are_outside_the_bound(backend, kind):
    """On the square product case: the last (shorter) split slot of the 897-column segment dropped; that segment read one
    tile late (it loses its first tile and gains the one-column task's); the one-column task's slot weighted by the next B
    column; on tensor cores the one-column task's first padding column carrying its V row."""
    (x1, x2, B, V, lay), true, bnd = _prod("square", backend, kind)
    run = lambda m, a: mo.hadamard_exact(kind, x1, x2, B, LS, OS, V, lay, mutant=m, mutant_arg=a)
    assert _outside(true, run("drop_slot", lay["slot0"][0] + lay["nsplit"][0] - 1), bnd)
    assert _outside(true, run("tile_late", 0), bnd)
    assert _outside(true, run("slot_task", lay["slot0"][1]), bnd)
    if backend == "tcgen05":
        assert _outside(true, run("pad_v", 1), bnd)


def test_hadamard_cross_mutant_is_outside_the_bound():
    (x1, x2, B, V, lay), true, bnd = _prod("cross", "tcgen05", "matern52")
    wrong = mo.hadamard_exact("matern52", x1, x2, B, LS, OS, V, lay, mutant="drop_slot", mutant_arg=lay["slot0"][4] + 1)
    assert _outside(true, wrong, bnd)


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_dB_losing_a_straddling_row_is_outside_the_bound(backend):
    """n1 = 2049: task 1 straddles row 2048 with one row in chunk 1; that one row lost from dB[1, :]."""
    x1, _, t1, _, T, _ = mo.hadamard_case("n2049", 0)
    lay = mo.task_layout(t1, None, T, backend)
    g = torch.Generator().manual_seed(4)
    L = torch.randn(x1.size(0), 4, generator=g)
    R = torch.randn(x1.size(0), 4, generator=g)
    true = mo.hadamard_dB("rbf", x1, None, LS, OS, L, R, lay)
    wrong = mo.hadamard_dB("rbf", x1, None, LS, OS, L, R, lay, drop_rows=lay["perm1"][2048:])
    assert (wrong - true)[[0, 2]].abs().max() == 0 and (wrong - true)[1].abs().max() > 0
    assert _outside(true, wrong, mo.hadamard_dB_bound("rbf", x1, None, LS, OS, L, R, lay))


@pytest.mark.parametrize("backend,kind", [("tcgen05", "matern32"), ("simt", "rbf")])
def test_kron_mutants_are_outside_the_bound(backend, kind):
    """N = 1450 (3 splits), T = 3, t = 6 (2 chunks): the scatter reading chunk 0's last split slot from chunk 1, and the mix
    leaving out its smallest B term."""
    n, d = mo.KRON_SPLIT
    T, t = 3, 6
    x = ko.points(n, d, 7)
    B = mo.random_B(T, 8)
    V = torch.randn(n * T, t, generator=torch.Generator().manual_seed(9))
    geo = mo.kron_layout(n, n, d, T, t, backend)
    true = mo.kron_exact(kind, x, None, B, LS, OS, V, T, t)
    bnd = mo.kron_bound(kind, x, None, B, LS, OS, V, T, t, geo)
    wrong = mo.kron_exact(kind, x, None, B, LS, OS, V, T, t, geo=geo, mutant="scatter_chunk", mutant_arg=(0, geo["nsplit"] - 1))
    assert _outside(true, wrong, bnd)
    a, b = divmod(int(B.abs().argmin()), T)
    assert _outside(true, mo.kron_exact(kind, x, None, B, LS, OS, V, T, t, mutant="mix_drop", mutant_arg=(a, b)), bnd)
