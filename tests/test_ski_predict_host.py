"""CPU checks of KISS-GP prediction on the grid (settings.ski_grid_prediction): the fp64 identities the grid caches rest on, the
eligibility / precedence of models._ski_grid_mode, the flag's default, and the resources of the new kernels in the built library."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import ski, ski_predict

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpytorch_b200", "lib", "libgpbbmm.so")


@pytest.mark.parametrize("d,sizes,kind", [(1, [30], "rbf"), (2, [14, 11], "matern52"), (3, [9, 8, 7], "rbf")])
def test_grid_caches_reproduce_the_joint_cross_covariance(d, sizes, kind):
    """W* (s K_uu W^T alpha) = K_ski(test, train) alpha and W* (s K_uu W^T R) = K_ski(test, train) R in fp64, with K_ski the
    oracle's interpolated product on the joint point set (what the joint prediction path slices)."""
    g = torch.Generator().manual_seed(d)
    n, m, J = 200, 37, 6
    axes = ski.create_grid(sizes, [(0.0, 1.0)] * d, dtype=torch.float64)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    xt = torch.rand(m, d, generator=g, dtype=torch.float64)
    xt[0] = torch.stack([a[0] for a in axes])          # first node: one-hot weights
    xt[1] = torch.stack([a[-1] for a in axes])         # last node
    alpha = torch.randn(n, 1, generator=g, dtype=torch.float64)
    R = torch.randn(n, J, generator=g, dtype=torch.float64)
    ls, osc = 0.3, 1.3
    xj = torch.cat([x, xt])
    for v in (alpha, R):
        pad = torch.cat([v, torch.zeros(m, v.size(1), dtype=torch.float64)])
        joint = ski.ski_matmul(kind, xj, axes, ls, osc, pad)[n:]
        grid = ski_predict.interp_matmul(axes, xt, ski_predict.grid_matmul(kind, x, axes, ls, osc, v))
        assert float((grid - joint).abs().max()) <= 1e-12 * float(joint.abs().max())
    # the strategy itself: mean = K*x alpha, covar = K** - (K*x R)(K*x R)^T
    y = torch.randn(n, generator=g, dtype=torch.float64)
    out = ski_predict.interpolated_prediction(kind, x, xt, y, axes, ls, osc, 0.2, R)
    Kj = ski.ski_matmul(kind, xj, axes, ls, osc, torch.eye(n + m, dtype=torch.float64))
    Kj = 0.5 * (Kj + Kj.T)
    alpha_ref = torch.linalg.solve(Kj[:n, :n] + 0.2 * torch.eye(n, dtype=torch.float64), y)
    assert torch.allclose(out["mean"], Kj[n:, :n] @ alpha_ref, rtol=0, atol=1e-10 * float((Kj[n:, :n] @ alpha_ref).abs().max()))
    U = Kj[n:, :n] @ R
    assert torch.allclose(out["covar"], Kj[n:, n:] - U @ U.T, rtol=0, atol=1e-10 * float(U.abs().max() ** 2 + Kj.abs().max()))


def _ops():
    from gpytorch_b200.operators import BatchLinearOperator, KernelLinearOperator, SKIKernelLinearOperator

    x, xt = torch.rand(50, 2), torch.rand(30, 2)
    ls, os_ = torch.tensor(0.5), torch.tensor(1.0)
    grid = ((16, 16), (0.0, 0.0), (0.1, 0.1))
    train = SKIKernelLinearOperator(x, "rbf", ls, os_, *grid)
    test = SKIKernelLinearOperator(xt, "rbf", ls.clone(), os_.clone(), *grid)
    others = {
        "plain": KernelLinearOperator(xt, xt, "rbf", ls, os_),
        "batch": BatchLinearOperator([test, test]),
        "other_grid": SKIKernelLinearOperator(xt, "rbf", ls, os_, (16, 17), (0.0, 0.0), (0.1, 0.1)),
        "other_kind": SKIKernelLinearOperator(xt, "matern52", ls, os_, *grid),
        "other_ls": SKIKernelLinearOperator(xt, "rbf", torch.tensor(0.6), os_, *grid),
        "other_os": SKIKernelLinearOperator(xt, "rbf", ls, torch.tensor(2.0), *grid),
    }
    return train, test, others


def test_ski_grid_mode_eligibility_and_precedence():
    from gpytorch_b200 import settings
    from gpytorch_b200.models import SKI_GRID_LOVE_MAX_BYTES, _ski_grid_mode
    from gpytorch_b200.operators import BatchLinearOperator

    train, test, others = _ops()
    assert _ski_grid_mode(train, test) is None                     # flag off: today's joint path
    with settings.fast_pred_var(True):
        assert _ski_grid_mode(train, test, 10) is None
    with settings.ski_grid_prediction(True):
        assert _ski_grid_mode(train, test) == "exact"
        for name, op in others.items():                            # ineligible test priors fall back
            assert _ski_grid_mode(train, op) is None, name
        assert _ski_grid_mode(BatchLinearOperator([train, train]), test) is None
        assert _ski_grid_mode(others["plain"], test) is None
        sharded = type(train)(train.x1, "rbf", train.lengthscale, train.outputscale, train.grid_sizes, train.grid_lo, train.grid_step)
        sharded._row_count = 25
        assert _ski_grid_mode(sharded, test) is None and _ski_grid_mode(train, sharded) is None
        for flag in (settings.fast_pred_var, settings.fast_pred_samples):
            with flag(True):
                assert _ski_grid_mode(train, test) == "love"       # J not known yet
                assert _ski_grid_mode(train, test, 1) == "lazy_love"
                assert _ski_grid_mode(train, test, 128) == "lazy_love"
                assert _ski_grid_mode(train, test, 129) == "dense_love"
                with settings.skip_posterior_variances(True):
                    assert _ski_grid_mode(train, test, 10) == "skip"
        with settings.skip_posterior_variances(True):
            assert _ski_grid_mode(train, test) == "skip"
        # the M J fp32 ceiling of the grid LOVE cache (M = 256 here)
        with settings.fast_pred_var(True):
            j_max = SKI_GRID_LOVE_MAX_BYTES // (4 * 256)
            assert _ski_grid_mode(train, test, j_max) == "dense_love"
            assert _ski_grid_mode(train, test, j_max + 1) == "joint_love"
        big = type(train)(train.x1, "rbf", train.lengthscale, train.outputscale, (128,) * 4, (0.0,) * 4, (0.01,) * 4)
        big_t = type(train)(test.x1, "rbf", train.lengthscale, train.outputscale, (128,) * 4, (0.0,) * 4, (0.01,) * 4)
        with settings.fast_pred_samples(True):
            assert _ski_grid_mode(big, big_t, 100) == "joint_love"      # 128^4 x 100 fp32 = 100 GB


def test_flag_default_and_snapshot():
    from gpytorch_b200 import settings

    assert settings.ski_grid_prediction.off()
    assert settings.ski_grid_prediction in settings.snapshot()
    with settings.ski_grid_prediction(True):
        assert settings.snapshot()[settings.ski_grid_prediction] == [True]


def test_lowrank_on_ski_is_a_separate_constructor_on_its_slot_key():
    from gpytorch_b200.operators import LowRankUpdatedKernelLinearOperator, _slot

    train, test, others = _ops()
    assert not LowRankUpdatedKernelLinearOperator.supports(test)
    with pytest.raises(RuntimeError):
        LowRankUpdatedKernelLinearOperator(test, torch.zeros(30, 3))
    op = LowRankUpdatedKernelLinearOperator.on_ski(test, torch.zeros(30, 3))
    assert op.shape == (30, 30) and op.base._plan_slot == _slot("plain", "lowrank") and test._plan_slot == _slot("plain", "own")
    with pytest.raises(RuntimeError):
        LowRankUpdatedKernelLinearOperator.on_ski(others["plain"], torch.zeros(30, 3))
    with pytest.raises(RuntimeError):
        LowRankUpdatedKernelLinearOperator.on_ski(test, torch.zeros(30, 129))


def test_ski_predict_kernels_are_spill_free():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = {"ski_interp_tiled_kernel": 0, "ski_grid_export_kernel": 0}
    for i, line in enumerate(lines):
        if "Function" not in line:
            continue
        for key in seen:
            if key in line:
                usage = lines[i + 1]
                assert int(re.search(r"STACK:(\d+)", usage).group(1)) == 0, f"{line.strip()}: local memory"
                assert int(re.search(r"REG:(\d+)", usage).group(1)) <= 80, f"{line.strip()}: {usage.strip()}"
                seen[key] += 1
    assert seen == {"ski_interp_tiled_kernel": 4, "ski_grid_export_kernel": 1}, seen
