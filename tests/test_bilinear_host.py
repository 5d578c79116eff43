"""Host checks of the hyper-parameter gradient's oracle (tests/bilinear_oracle.py): the fp64 closed form against fp64 autograd
through oracle.kernels and against the reference's own backward (tests/golden/kernels_golden.npz); the fp32 bound is tight enough
that deliberately wrong engines fall outside it on the GPU test's own cases; and Plan.bilinear_grad checks its operands before
it reaches the engine."""
import numpy as np
import pytest
import torch

import bilinear_oracle as bo
from oracle import kernels as ok

KINDS = list(bo.KINDS)


def _autograd(kind, x1, x2, ls, s, L, R, same):
    lsp = bo.f32(ls).reshape(-1 if bo.f32(ls).numel() > 1 else ()).clone().requires_grad_()
    osp = bo.f32(s)[0].clone().requires_grad_()
    K = ok.kernel_matrix(kind, x1.double(), (x1 if same else x2).double(), lsp, osp, same)
    ((L @ R.t()) * K).sum().backward()
    return lsp.grad.reshape(-1), osp.grad.item()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("geom", ["square", "cross", "cross_coinciding"])
def test_closed_form_matches_fp64_autograd(kind, ard, geom):
    g = torch.Generator().manual_seed(3 + KINDS.index(kind) + 10 * ard)
    n1, n2, d, s = 11, 9, 4, 5
    x1 = torch.rand(n1, d, generator=g).float()
    x2 = torch.rand(n2, d, generator=g).float()
    if geom == "cross_coinciding":
        x2 = torch.cat([x1[:4], x2[4:]])          # four pairs at distance 0 in a cross plan
    if geom == "square":
        n2, x2 = n1, None
    ls = [0.4, 0.6, 0.9, 1.3] if ard else 0.55
    L = torch.randn(n1, s, generator=g, dtype=torch.float64)
    R = torch.randn(n2, s, generator=g, dtype=torch.float64)
    rl, ro = _autograd(kind, x1, x2, ls, 1.3, L, R, geom == "square")
    cl, co = bo.closed_form(kind, x1, x2, ls, 1.3, L, R, same=geom == "square")
    torch.testing.assert_close(cl, rl, rtol=1e-11, atol=1e-12)
    assert co == pytest.approx(ro, rel=1e-12, abs=1e-12)


def test_closed_form_matches_reference_goldens(golden):
    """left = W, right = I: dF/dl of sum(W * K) from the reference's RBFCovariance / MaternCovariance backward (outputscale 1).
    The oracle holds the lengthscale in fp32 as the engine does, 3e-8 relative from the golden's fp64 value."""
    names = {"rbf": "rbf", "matern12": "mat12", "matern32": "mat32", "matern52": "mat52"}
    for tag in "abcd":
        x1 = torch.from_numpy(golden[f"{tag}_f64_x1"]); x2 = torch.from_numpy(golden[f"{tag}_f64_x2"])
        same = bool(golden[f"{tag}_f64_same"])
        ls = float(golden[f"{tag}_f64_ls"])
        W = torch.from_numpy(golden[f"{tag}_f64_rbf_W"])
        for kind, nk in names.items():
            want = float(golden[f"{tag}_f64_{nk}_dls"].reshape(-1)[0])
            got = bo.closed_form(kind, x1, None if same else x2, ls, 1.0, W, torch.eye(x2.size(0), dtype=torch.float64), same=same)[0]
            assert got.item() == pytest.approx(want, rel=1e-6), (tag, kind, got.item(), want)


# ---- the bound has teeth: wrong engines land outside it on the GPU test's own cases --------------------------------------------
def _paths_case(kind, ard):
    """test_gpu_bilinear.test_paths_and_kinds_within_bound: n = 257, d = 5, s = 17."""
    g = torch.Generator().manual_seed(1 + KINDS.index(kind))
    x = torch.rand(257, 5, generator=g)
    L, R = torch.randn(257, 17, generator=g), torch.randn(257, 17, generator=g)
    ls = [float(v) for v in torch.linspace(0.5, 1.5, 5)] if ard else 0.8
    return (kind, x, None, ls, 1.3, L.double(), R.double())


def _shard_case():
    """test_gpu_bilinear.test_row_shards_within_bound_and_sum_to_the_full_gradient: the shard rows [129, 329) of n = 1000."""
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1000, 4, generator=g)
    L, R = 0.1 + torch.rand(1000, 17, generator=g), 0.1 + torch.rand(1000, 17, generator=g)
    return ("matern12", x, None, 0.6, 1.4, L[129:329].double(), R.double()), 129


def _small_square_case():
    """test_gpu_bilinear.test_small_square_psd_weights_within_bound, Matern-1/2: n = 64, distinct points, L = R."""
    g = torch.Generator().manual_seed(61)
    x = torch.rand(64, 4, generator=g)
    L = 0.1 + torch.rand(64, 16, generator=g)
    return ("matern12", x, None, 0.6, 1.2, L.double(), L.double())


def _outside(true, wrong, bnd):
    (tl, to), (wl, wo), (bl, bob) = true, wrong, bnd
    return bool(((tl - wl).abs() > bl).any()) or abs(to - wo) > bob


@pytest.mark.parametrize("path", ["tc", "simt"])
def test_mask_ignoring_row_begin_is_outside_the_bound(path):
    args, b = _shard_case()
    true = bo.closed_form(*args, same=True, row_begin=b)
    wrong = bo.closed_form(*args, same=True, row_begin=b, diag_offset=0)
    assert _outside(true, wrong, bo.bound(*args, path, same=True, row_begin=b))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path", ["tc", "simt"])
def test_dropped_last_column_chunk_is_outside_the_bound(kind, path):
    args = _paths_case(kind, False)
    true = bo.closed_form(*args, same=True)
    wrong = bo.closed_form(*args[:5], args[5][:, :16], args[6][:, :16], same=True)
    assert _outside(true, wrong, bo.bound(*args, path, same=True))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mutation", [{"ard_no_r2": True}, {"ard_shift": 1}])
def test_wrong_ard_factor_is_outside_the_bound(kind, mutation):
    args = _paths_case(kind, True)
    true = bo.closed_form(*args, same=True)
    wrong = bo.closed_form(*args, same=True, **mutation)
    bl, _ = bo.bound(*args, "simt", same=True)
    assert ((true[0] - wrong[0]).abs() > bl).all()


def test_unmasked_diagonal_on_matern12_is_outside_the_tensor_core_bound():
    """Without the diagonal mask the tensor-core path evaluates a_ii from the 3xTF32 GEMM, off from 0 by up to the bound's own
    da, and Matern-1/2's g = rho e turns that into sqrt(da) per diagonal pair."""
    args = _small_square_case()
    kind, x, _, ls, os_, L, R = args
    sc = (2.0 ** 0.5) / 0.6
    z = (x.double() - x.double().mean(0)) * sc
    da = (1 + bo.kp_of(4) / 4) * 2.0 ** -21 * 2 * (z * z).sum(1)
    true = bo.closed_form(*args, same=True)
    wrong = bo.closed_form(*args, same=True, diag_m=da)
    assert _outside(true, wrong, bo.bound(*args, "tc", same=True))


# ---- Plan.bilinear_grad operand checks ----------------------------------------------------------------------------------------
def _fake_plan(row_count, n2):
    from gpytorch_b200.engine import Plan

    p = Plan.__new__(Plan)
    p.row_count, p.n2, p.lengthscale, p.device = row_count, n2, [0.5], torch.device("cpu")
    p._h = None
    return p


@pytest.mark.parametrize("left,right", [((5, 3), (7, 4)), ((4, 3), (7, 3)), ((5, 3), (6, 3)), ((5,), (7,)), ((5, 0), (7, 0))])
def test_bilinear_grad_rejects_bad_shapes_before_the_engine(left, right):
    p = _fake_plan(5, 7)
    with pytest.raises(RuntimeError, match="bilinear_grad: left must be"):
        p.bilinear_grad(torch.zeros(left), torch.zeros(right))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("host", ["left", "right"])
def test_bilinear_grad_rejects_host_operands(dtype, host):
    """Right shapes, but an operand in host memory (float32 or float64) never reaches the engine; the dtype refusal of a
    device operand is tested on the GPU (test_gpu_bilinear.py)."""
    p = _fake_plan(5, 7)
    with pytest.raises(RuntimeError, match="CUDA device"):
        if host == "left":
            p.bilinear_grad(torch.zeros(5, 3, dtype=dtype), torch.zeros(7, 3))
        else:
            p.bilinear_grad(torch.zeros(5, 3), torch.zeros(7, 3, dtype=dtype))


def test_bilinear_grad_copies_only_blocks_it_cannot_stride():
    """An expanded [n, s] block (row stride 0) or a transposed one is copied before the engine sees it; a padded or one-row
    block is passed as is, and its leading dimension (_ld) is >= s."""
    from gpytorch_b200.engine import _ld, _row_block

    for t in (torch.zeros(1, 3).expand(5, 3), torch.zeros(3, 5).t(), torch.zeros(5, 6)[:, ::2]):
        c = _row_block(t)
        assert c.data_ptr() != t.data_ptr() and c.is_contiguous() and _ld(c) == 3
    for t in (torch.zeros(7, 9)[:, :3], torch.zeros(1, 3).expand(1, 3), torch.zeros(4, 3)):
        assert _row_block(t) is t and _ld(t) >= 3


def test_one_row_block_leading_dimension():
    from gpytorch_b200.engine import _ld

    row = torch.zeros(1, 6).as_strided((1, 6), (0, 1))
    assert _ld(row) == 6 and _ld(torch.zeros(4, 6)[:, :3]) == 6
