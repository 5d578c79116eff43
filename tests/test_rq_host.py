"""CPU checks of the rational quadratic kernel: the fp64 oracle against the reference's own RQKernel (golden file), mutants of the
device formulas that must fall outside the oracle's bound, the RQKernel class surface, the operator wrappers that must keep
alpha, the refusals, the header and the compiled kernels (no local memory in the new K.V instantiations, unserialised wgmma
chains, the existing kinds' kernels unchanged in name and number)."""
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import rq_oracle as ro  # noqa: E402
from gpytorch_b200 import kernels, operators  # noqa: E402

GOLD = os.path.join(HERE, "golden", "rq_golden.npz")
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")


def _cases():
    z = np.load(GOLD)
    for ci in range(int(z["ncases"])):
        yield ci, {k[len(f"c{ci}_"):]: z[k] for k in z.files if k.startswith(f"c{ci}_")}


def test_oracle_matches_the_reference_class():
    for ci, c in _cases():
        d, ard, n1, n2, B = (int(v) for v in c["meta"])
        for b in range(max(B, 1)):
            sl = (lambda a: a[b]) if B else (lambda a: a)
            x1, x2 = torch.from_numpy(sl(c["x1"])), torch.from_numpy(sl(c["x2"]))
            ls, al = torch.from_numpy(sl(c["ls"])).reshape(-1), float(sl(c["alpha"]).reshape(-1)[0])
            K = ro.kernel(x1, x2, ls, al)
            assert torch.allclose(K, torch.from_numpy(sl(c["K"])), rtol=1e-12, atol=1e-14), ci
            assert torch.allclose(ro.kernel(x1, x1, ls, al), torch.from_numpy(sl(c["Kxx"])), rtol=1e-12, atol=1e-14), ci
            assert np.allclose(sl(c["diag"]), 1.0), ci
            gl, ga, _ = ro.grads(x1, x2, ls if ard else ls[:1], al, torch.from_numpy(sl(c["W"])))
            assert torch.allclose(gl.reshape(-1), torch.from_numpy(sl(c["gls"])).reshape(-1), rtol=1e-10, atol=1e-12), ci
            assert math.isclose(float(ga), float(sl(c["galpha"]).reshape(-1)[0]), rel_tol=1e-10, abs_tol=1e-12), ci


def _pair(r, alpha, path="simt"):
    x1 = torch.zeros(1, 1, dtype=torch.float64)
    x2 = torch.tensor([[r]], dtype=torch.float64)
    V = torch.ones(1, 1)
    return ro.kernel(x1, x2, 1.0, alpha)[0, 0].item(), ro.kmv_bound(x1, x2, 1.0, alpha, V, 1.0, path, 1, 1)[0, 0].item()


def test_bound_does_not_grow_with_alpha():
    for r in (0.3, 1.0, 3.0):
        bounds = [_pair(r, a)[1] for a in (0.5, 2.0, 50.0, 1e4, 1e6)]
        assert max(bounds) < 2e-6, (r, bounds)
        assert bounds[-1] <= 4 * min(bounds), (r, bounds)


def test_naive_lg2_mutant_falls_outside_the_bound():
    """lg2(fp32(1 + t)) multiplied by alpha = 1e4 at r = 1: the rounding of 1 + t alone moves k far beyond the bound."""
    alpha = 1e4
    k, b = _pair(1.0, alpha)
    t = 0.5 / alpha
    mutant = 2.0 ** (-alpha * math.log2(float(np.float32(1.0 + np.float32(t)))))
    assert abs(mutant - k) > 50 * b, (mutant, k, b)
    engine = 2.0 ** (-alpha * float(ro.lg2_1p_f32(t)))
    assert abs(engine - k) < b, (engine, k, b)


def test_dropped_one_plus_t_in_the_lengthscale_derivative_is_caught():
    """l dk/dl = r^2 k / (1 + t); the mutant r^2 k differs from the fp64 gradient far beyond the gradients' rtol 2e-4."""
    x1 = torch.zeros(1, 1, dtype=torch.float64)
    x2 = torch.tensor([[1.0]], dtype=torch.float64)
    W = torch.ones(1, 1, dtype=torch.float64)
    for alpha in (0.5, 2.0, 50.0):
        gl, _, _ = ro.grads(x1, x2, torch.tensor([1.0]), alpha, W)
        k = ro.kernel(x1, x2, 1.0, alpha)[0, 0].item()
        t = 0.5 / alpha
        assert math.isclose(float(gl), 1.0 * k / (1 + t), rel_tol=1e-12)   # dk/dl = r^2 k / ((1 + t) l), r = l = 1
        assert abs(1.0 * k - float(gl)) > 2e-4 * abs(float(gl)) * 10


def test_phi_is_formed_without_cancellation():
    """The device phi stays within 2^-18 relative over [0, 4]; the plain fp32 difference is off by far more at t ~ 1e-3."""
    worst = 0.0
    for t in np.concatenate([np.geomspace(1e-7, 0.124, 400), np.linspace(0.125, 4.0, 400)]):
        t = float(np.float32(t))
        ex = ro.phi_exact(t)
        worst = max(worst, abs(float(ro.phi_f32(t)) - ex) / ex)
    assert worst < 2.0 ** -18, worst
    t = float(np.float32(1e-3))
    naive = np.float32(np.log1p(np.float32(t)) - np.float32(np.float32(t) / np.float32(1 + np.float32(t))))
    assert abs(float(naive) - ro.phi_exact(t)) / ro.phi_exact(t) > 2.0 ** -14


def test_lg2_polynomial_is_absolutely_accurate():
    for t in np.geomspace(1e-9, 0.0624, 300):
        t = float(np.float32(t))
        assert abs(float(ro.lg2_1p_f32(t)) - math.log2(1 + t)) <= 8 * 2.0 ** -24 * math.log2(1 + t) + 1e-30, t


# ---- the class surface --------------------------------------------------------------------------------------------------------
def test_class_surface():
    k = kernels.RQKernel()
    assert tuple(k.raw_alpha.shape) == (1,) and tuple(k.raw_lengthscale.shape) == (1, 1)
    kb = kernels.RQKernel(ard_num_dims=3, batch_shape=torch.Size([4]))
    assert tuple(kb.raw_alpha.shape) == (4, 1) and tuple(kb.raw_lengthscale.shape) == (4, 1, 3)
    k.alpha = 2.5
    assert torch.allclose(k.alpha, torch.tensor([2.5]))
    k.initialize(raw_alpha=torch.tensor([0.0]))
    assert torch.allclose(k.alpha, torch.nn.functional.softplus(torch.tensor([0.0])))
    assert k.kind == "rq" and isinstance(k, kernels._StationaryKernel)
    with pytest.raises(NotImplementedError):
        kernels.RQKernel(lengthscale_prior=object())
    with pytest.raises(NotImplementedError):
        kernels.RQKernel(alpha_prior=object())
    assert "RQKernel" in kernels.__doc__


def test_kernel_level_refusals():
    rq = kernels.RQKernel()
    with pytest.raises(NotImplementedError, match="RQ"):
        kernels.ProductKernel(kernels.RBFKernel(), rq)
    with pytest.raises(NotImplementedError, match="RQ"):
        kernels.ProductKernel(kernels.ScaleKernel(rq), kernels.RBFKernel())
    with pytest.raises(NotImplementedError, match="RQ"):
        kernels.GridInterpolationKernel(rq, grid_size=16, num_dims=1)
    mk = kernels.MultitaskKernel(kernels.ScaleKernel(kernels.RQKernel()), num_tasks=2)
    with pytest.raises(NotImplementedError, match="RQ"):
        mk.forward(torch.zeros(3, 1), torch.zeros(3, 1))


# ---- wrappers keep alpha (CPU tensors: no plan is touched) -------------------------------------------------------------------
def _rq_op(n1=5, n2=None, alpha=3.0):
    x1 = torch.randn(n1, 2)
    x2 = None if n2 is None else torch.randn(n2, 2)
    return operators.RQKernelLinearOperator(x1, x2, torch.tensor(0.7), torch.tensor(alpha), torch.tensor(1.5))


def _is_rq_with(o, alpha):
    return isinstance(o, operators.RQKernelLinearOperator) and float(o.alpha) == alpha


def test_every_wrapper_method_keeps_alpha():
    op = _rq_op(5, 4)
    assert [t is u for t, u in zip(op.hyper_tensors(), [op.lengthscale, op.alpha, op.outputscale])] == [True] * 3
    assert _is_rq_with(op.t(), 3.0) and _is_rq_with(op.mT, 3.0) and _is_rq_with(op.transpose(-1, -2), 3.0)
    assert _is_rq_with(op.detach(), 3.0)
    assert _is_rq_with(op[1:3, :], 3.0) and _is_rq_with(op[:, 0:2], 3.0)
    w = op.with_outputscale(torch.tensor(2.0))
    assert _is_rq_with(w, 3.0) and float(w.outputscale) == 2.0
    sq = _rq_op(5)
    s = sq + operators.KernelLinearOperator(sq.x1, None, "rbf", torch.tensor(1.0))
    assert isinstance(s, operators.SumKernelLinearOperator) and _is_rq_with(s.ops[0], 3.0)
    # the RQ term takes the plain first-term slot, the plain term the second
    assert [o._plan_slot for o in s.ops] == [operators._slot("plain", "sum_term", 0), operators._slot("plain", "sum_term", 1)]
    assert len(s.hyper_tensors()) == 5
    lr = operators.LowRankUpdatedKernelLinearOperator(sq, torch.randn(5, 2))
    assert _is_rq_with(lr.base, 3.0)


def test_scale_kernel_folding_keeps_alpha():
    x = torch.randn(6, 2)
    rq = kernels.RQKernel()
    rq.alpha = 4.0
    for k in (kernels.ScaleKernel(rq), kernels.ScaleKernel(kernels.ScaleKernel(rq))):
        op = k(x)
        assert isinstance(op, operators.RQKernelLinearOperator) and math.isclose(float(op.alpha.detach()), 4.0, rel_tol=1e-6)
    s = kernels.ScaleKernel(kernels.ScaleKernel(kernels.RBFKernel()) + kernels.ScaleKernel(rq))(x)
    assert isinstance(s, operators.SumKernelLinearOperator)
    assert any(isinstance(t, operators.RQKernelLinearOperator) and math.isclose(float(t.alpha.detach()), 4.0, rel_tol=1e-6) for t in s.ops)
    kb = kernels.ScaleKernel(kernels.RQKernel(batch_shape=torch.Size([2])))
    bop = kb(torch.randn(2, 5, 1))
    assert all(isinstance(o, operators.RQKernelLinearOperator) for o in bop.ops)


def test_operator_level_refusals():
    op = _rq_op(5)
    plain = operators.KernelLinearOperator(op.x1, None, "rbf", torch.tensor(1.0))
    with pytest.raises(NotImplementedError, match="RQ"):
        op.mul(plain)
    with pytest.raises(NotImplementedError, match="RQ"):
        plain.mul(op)
    with pytest.raises(NotImplementedError, match="RQ"):
        operators.ProductKernelLinearOperator([plain, op])
    with pytest.raises(NotImplementedError, match="RQ"):
        operators.RQKernelLinearOperator(op.x1, None, torch.tensor(1.0), torch.tensor(1.0), row_begin=1, row_count=2)
    with pytest.raises(NotImplementedError, match="RQ"):
        operators._additive_components([op], "additive")


def test_plan_resends_when_alpha_changes():
    """Operators on one plan that differ in alpha alone re-send their hyper-parameters (set_hypers_rq(ls, al, os_, nz)); equal
    ones do not."""
    calls = []

    class _P:
        def set_hypers_rq(self, *args):
            calls.append(args)

    plan, x = _P(), torch.zeros(4, 1)
    for al in (1.0, 1.0, 2.0):
        op = operators.RQKernelLinearOperator(x, None, torch.tensor(0.5), torch.tensor(al), torch.tensor(1.5))
        op._plan = plan      # an existing plan, as the cache hands out: sent only when its key differs
        op.plan(0.25)
    assert calls == [([0.5], 1.0, 1.5, 0.25), ([0.5], 2.0, 1.5, 0.25)]


# ---- header, C ABI, compiled kernels ------------------------------------------------------------------------------------------
def test_header_and_settings_table_document_the_call():
    h = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert "GP_RQ = 4" in h
    assert re.search(r"int gp_plan_set_hypers_rq\(gp_plan\* plan, const float\* lengthscale, int n_ls, float alpha,", h)
    doc = h[h.index("Rational quadratic kernels"):h.index("int gp_plan_set_hypers_rq")]
    for call in ("gp_plan_set_sum", "gp_kmv_input_grad", "[dF/dl (n_ls) | dF/dalpha]"):
        assert call in doc, call
    # the calls an RQ plan refuses: an x in the rq column of the plan-settings table
    table = h[h.index("Plan settings."):h.index("*/", h.index("Plan settings."))]
    head = next(ln for ln in table.splitlines() if ln.rstrip().endswith("rq  ply"))
    col = head.index(" rq ") + 1
    refusing = {ln[5:col].split("  ")[0].strip() for ln in table.splitlines() if len(ln) > col and ln[col] == "x"}
    for call in ("gp_plan_set_tasks", "gp_plan_set_kron", "gp_plan_set_deriv", "gp_plan_set_deriv_kind", "gp_plan_set_product",
                 "gp_plan_set_ski", "gp_plan_set_additive", "gp_plan_set_spectral", "gp_plan_set_periodic",
                 "gp_plan_set_comm with more than one rank", "gp_plan_set_kron (as the data plan)", "gp_plan_set_deriv (as the data plan)",
                 "gp_plan_set_product, a factor"):
        assert call in refusing, call


def _tool(name):
    t = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return t if os.path.exists(t) else None


def test_new_kernels_have_no_local_memory_and_old_ones_keep_their_count():
    tool = _tool("cuobjdump")
    if not tool or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available")
    r = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    seen = {"rq_tc_kernel": 0, "rq_simt_kernel": 0, "kmv_tc_kernelILi": 0}
    for i, line in enumerate(lines):
        if "Function" not in line:
            continue
        for key in seen:
            if key in line:
                seen[key] += 1
                if key != "kmv_tc_kernelILi":
                    stack = int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1))
                    local = int(re.search(r"LOCAL:(\d+)", lines[i + 1]).group(1))
                    assert stack == 0 and local == 0, line
    assert seen == {"rq_tc_kernel": 3, "rq_simt_kernel": 10, "kmv_tc_kernelILi": 8}, seen


def test_rq_wgmma_chains_are_not_serialised(tmp_path):
    nvcc = os.environ.get("NVCC") or _tool("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "gpytorch_b200", "csrc", "kmv_tc.cu")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v",
           "-cubin", src, "-o", str(tmp_path / "kmv_tc.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert "rq_tc_kernel" in log
    assert not [ln for ln in log.splitlines() if re.search(r"\(C751[125]\)", ln)]
    tool = _tool("cuobjdump")
    sass = subprocess.run([tool, "-sass", str(tmp_path / "kmv_tc.cubin")], capture_output=True, text=True, timeout=300).stdout
    bodies, cur = [], None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = [] if "rq_tc_kernel" in line else None
            if cur is not None:
                bodies.append(cur)
        elif cur is not None:
            cur.append(line)
    assert len(bodies) == 3
    for body in bodies:
        ops = [ln for ln in body if re.search(r"HGMMA\.64x(32|16)x8\.F32\.TF32|WARPGROUP\.DEPBAR", ln)]
        starts = [i for i, ln in enumerate(ops) if re.search(r"HGMMA\.64x32x8\.F32\.TF32 .*RZ, !UPT", ln)]
        assert starts
        for i in starts:
            assert all("HGMMA" in ln for ln in ops[i:i + 16]) and len(ops[i:i + 16]) == 16
