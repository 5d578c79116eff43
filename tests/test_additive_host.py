"""Additive GPs without a GPU: the fp64 oracle against the reference's own sum_interaction_terms (golden), brute force and the
product identity; the dense sum_interaction_terms; dispatch of .sum(dim=-3) / sum_interaction_terms to the engine operator, the
broadcasting of shared hyper-parameters and the splitting of the engine's gradients; the refusals; the new C ABI; and the machine
code of csrc/additive.cu (no local memory, one MUFU.EX2 per component per pair)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import additive_oracle as ao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
SRC = os.path.join(ROOT, "gpytorch_b200", "csrc", "additive.cu")
KINDS = ["rbf", "matern12", "matern32", "matern52"]


def test_oracle_matches_reference_golden():
    z = np.load(os.path.join(ROOT, "tests", "golden", "additive_golden.npz"))
    ncase = len([k for k in z.files if k.endswith("_meta")])
    assert ncase >= 7
    for ci in range(ncase):
        k, D, M = (int(v) for v in z[f"c{ci}_meta"])
        K = ao.additive_dense(KINDS[k], torch.tensor(z[f"c{ci}_X1"]), torch.tensor(z[f"c{ci}_X2"]), z[f"c{ci}_ls"].tolist(),
                              z[f"c{ci}_sc"].tolist(), M)
        ref = torch.tensor(z[f"c{ci}_K"])
        assert (K - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


@pytest.mark.parametrize("D", [1, 2, 4, 6])
def test_recurrence_matches_brute_force_newton_girard_and_product_identity(D):
    g = torch.Generator().manual_seed(D)
    cs = [torch.rand(5, 4, generator=g, dtype=torch.float64) * 2 for _ in range(D)]
    for M in range(1, D + 1):
        e = ao.esym_sum(cs, M)
        assert torch.allclose(e, ao.brute_force(cs, M), rtol=1e-13, atol=0)
        assert torch.allclose(e, ao.newton_girard(cs, M), rtol=1e-10, atol=0)
    prod = torch.ones_like(cs[0])
    for c in cs:
        prod = prod * (1 + c)
    assert torch.allclose(ao.esym_sum(cs, D), prod - 1, rtol=1e-13, atol=0)
    assert torch.equal(ao.esym_sum(cs, D + 3), ao.esym_sum(cs, D))   # degrees above D add nothing


def test_dense_sum_interaction_terms():
    from gpytorch_b200.utils import sum_interaction_terms

    g = torch.Generator().manual_seed(3)
    c = torch.rand(2, 5, 6, 6, generator=g, dtype=torch.float64)   # [..., D, N, N]
    for M in (1, 2, 3, 5, 9):
        ref = torch.stack([ao.brute_force(list(c[b]), M) for b in range(2)])
        assert torch.allclose(sum_interaction_terms(c, max_degree=M), ref, rtol=1e-13, atol=0)
    assert torch.allclose(sum_interaction_terms(c), torch.stack([ao.brute_force(list(c[b]), 5) for b in range(2)]), rtol=1e-13)
    assert torch.allclose(sum_interaction_terms(c.movedim(1, 0), max_degree=2, dim=-4), sum_interaction_terms(c, max_degree=2))
    with pytest.raises(ValueError, match="negative"):
        sum_interaction_terms(c, dim=1)
    with pytest.raises(ValueError, match="max_degree"):
        sum_interaction_terms(c, max_degree=0)


def _batched(D, n=7, kind="rbf", shared=False):
    from gpytorch_b200 import kernels

    X = torch.rand(n, D)
    base = (kernels.RBFKernel if kind == "rbf" else kernels.MaternKernel)(**({} if shared else {"batch_shape": torch.Size([D])}),
                                                                           ard_num_dims=1)
    k = kernels.ScaleKernel(base, **({"batch_shape": torch.Size([D])} if shared else {}))
    return k, X, k(X.mT.unsqueeze(-1))


@pytest.mark.parametrize("shared", [False, True])
def test_sum_and_interaction_terms_dispatch_and_broadcast(shared):
    from gpytorch_b200.operators import AdditiveKernelLinearOperator, BatchLinearOperator
    from gpytorch_b200.utils import sum_interaction_terms

    D = 5
    k, X, b = _batched(D, shared=shared)
    assert isinstance(b, BatchLinearOperator)
    op = b.sum(dim=-3)
    assert isinstance(op, AdditiveKernelLinearOperator) and op.max_degree == 1 and tuple(op.shape) == (7, 7)
    assert torch.equal(op.x1, X) and op.same
    assert isinstance(b.sum(dim=0), AdditiveKernelLinearOperator)
    op2 = sum_interaction_terms(b, max_degree=3)
    assert isinstance(op2, AdditiveKernelLinearOperator) and op2.max_degree == 3
    assert sum_interaction_terms(b).max_degree == D and sum_interaction_terms(b, max_degree=50).max_degree == D
    ls, sc, _, _ = op._host_hypers()
    want_ls = k.base_kernel.lengthscale.detach().reshape(-1).tolist()
    assert ls == pytest.approx(want_ls * D if shared else want_ls)
    assert sc == pytest.approx(k.outputscale.detach().reshape(-1).tolist())
    # the hyper-parameter tensors are the components' own slices: autograd reaches the batched / shared parameters
    hs = op.hyper_tensors()
    assert len(hs) == 2 * D
    sum(h.sum() for h in hs).backward()
    g = k.base_kernel.raw_lengthscale.grad
    assert g is not None and g.numel() == (1 if shared else D)


def test_gradient_splitting_sums_shared_parameters(monkeypatch):
    from gpytorch_b200 import operators

    D = 4
    for shared in (False, True):
        k, X, b = _batched(D, shared=shared)
        op = b.sum(dim=-3)

        class FakePlan:
            def bilinear_grad(self, left, right):
                return [1.0, 2.0, 3.0, 4.0], [10.0, 20.0, 30.0, 40.0]

        monkeypatch.setattr(operators.AdditiveKernelLinearOperator, "plan", lambda self, noise=0.0: FakePlan())
        grads = op._bilinear_derivative_list(None, None)
        assert [float(g) for g in grads] == [1.0, 10.0, 2.0, 20.0, 3.0, 30.0, 4.0, 40.0]
        hs = op.hyper_tensors()
        torch.autograd.backward(hs, grads)
        ls_grad = k.base_kernel.raw_lengthscale.grad
        if shared:   # one shared lengthscale: the engine's D gradients are summed (through the constraint's chain rule)
            assert ls_grad.numel() == 1
        else:
            assert ls_grad.numel() == D
        monkeypatch.undo()


def test_stacked_inputs_are_shared_while_equal_and_the_cache_is_bounded():
    from gpytorch_b200 import operators

    operators._ADDITIVE_X.clear()
    D = 3
    _, X, b = _batched(D, n=40)
    op1 = b.sum()
    op2 = operators.BatchLinearOperator(b.ops).sum()
    assert op2.x1 is op1.x1                       # equal inputs: one buffer, so one engine plan without a re-pack
    for n in range(2, 2 + 2 * operators._ADDITIVE_X_ROLES):
        operators.BatchLinearOperator([type(o)(o.x1[:n], None, o.kind, o.lengthscale, o.outputscale) for o in b.ops]).sum()
    assert len(operators._ADDITIVE_X) == operators._ADDITIVE_X_ROLES
    assert all(len(v) <= 2 for v in operators._ADDITIVE_X.values())
    op3 = b.sum()
    assert op3.x1 is not op1.x1 and torch.equal(op3.x1, op1.x1)   # its role was evicted: stacked anew
    operators._ADDITIVE_X.clear()


def test_refusals():
    from gpytorch_b200 import kernels
    from gpytorch_b200.operators import AdditiveKernelLinearOperator, BatchLinearOperator, KernelLinearOperator
    from gpytorch_b200.utils import sum_interaction_terms

    D = 3
    _, X, b = _batched(D)
    with pytest.raises(NotImplementedError, match=r"BatchLinearOperator.sum\(dim=-2\)"):
        b.sum(dim=-2)
    with pytest.raises(NotImplementedError, match="only its batch dimension"):
        sum_interaction_terms(b, dim=-4)
    mixed = BatchLinearOperator([b.ops[0], KernelLinearOperator(b.ops[1].x1, None, "matern52", b.ops[1].lengthscale)])
    with pytest.raises(NotImplementedError, match="share one RBF / Matern kind"):
        mixed.sum(dim=-3)
    wide = kernels.RBFKernel(batch_shape=torch.Size([2]))(torch.rand(2, 5, 3))
    with pytest.raises(NotImplementedError, match=r"one input dimension \(\[n, 1\] inputs\)"):
        wide.sum(dim=-3)
    with pytest.raises(NotImplementedError, match="1 to 32 components"):
        BatchLinearOperator([b.ops[0]] * 33).sum()
    with pytest.raises(NotImplementedError, match="up to degree 8"):
        AdditiveKernelLinearOperator([b.ops[0]] * 10, max_degree=9)
    with pytest.raises(NotImplementedError, match="not AdditiveKernelLinearOperator"):
        BatchLinearOperator([b.sum(), b.sum()]).sum()
    xg = torch.rand(5, 1, requires_grad=True)
    with pytest.raises(NotImplementedError, match="gradients with respect to the inputs"):
        AdditiveKernelLinearOperator([KernelLinearOperator(xg, None, "rbf", torch.tensor(1.0))])
    op = b.sum()
    with pytest.raises(NotImplementedError, match="adds a \\(Constant\\)DiagLinearOperator only"):
        op + op
    # an additive operator is never re-wrapped as a plain term of a kernel sum, in either order
    plain = KernelLinearOperator(X, None, "rbf", torch.tensor(0.7))
    with pytest.raises(NotImplementedError, match="sums that contain additive operators"):
        plain + op
    with pytest.raises(NotImplementedError, match="adds a \\(Constant\\)DiagLinearOperator only"):
        op + plain
    from gpytorch_b200.operators import SumKernelLinearOperator
    with pytest.raises(NotImplementedError, match="sums that contain additive operators"):
        SumKernelLinearOperator([plain, op])
    with pytest.raises(NotImplementedError, match="products that contain an additive operator"):
        op * op
    with pytest.raises(NotImplementedError, match="inputs of an additive operator"):
        op._input_grad_list(None, None, [True])
    with pytest.raises(NotImplementedError, match="takes a BatchLinearOperator"):
        sum_interaction_terms([1, 2])


def test_c_abi_declares_set_additive():
    hdr = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert re.search(r"int gp_plan_set_additive\(gp_plan\* plan, int max_degree, const float\* comp_scale, int n_comp\);", hdr)
    from gpytorch_b200 import _lib

    assert _lib.PROTOTYPES["gp_plan_set_additive"][1][1:] == [_lib._I, _lib.C.POINTER(_lib._F), _lib._I]


def _tool():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available (python -m gpytorch_b200.build)")
    return tool


def test_ptxas_reports_no_spills_for_any_instantiation():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"additive_ptxas_{os.getpid()}.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas",
                        "-v", "-c", SRC, "-o", out], capture_output=True, text=True, timeout=900)
    if os.path.exists(out):
        os.remove(out)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) >= 2 * 5 * 6 + 2 * 6 and len(spills) == len(entries)
    assert all(s == ("0", "0", "0") for s in spills)


def test_kmv_sass_has_one_ex2_per_component_per_pair():
    r = subprocess.run([_tool(), "-sass", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    seen = 0
    for f in funcs:
        name = f.split("\n", 1)[0].strip()
        m = re.match(r"_ZN2gp19additive_kmv_kernelILb(\d)ELi(\d)ELi(\d+)EEEv", name)
        if not m:
            continue
        seen += 1
        DP = int(m.group(3))
        ex2 = len(re.findall(r"MUFU\.EX2", f))
        # the pair loop is unrolled twice over DP statically unrolled components: one ex2 each, nothing else calls MUFU.EX2
        assert ex2 == 2 * DP, (name, ex2)
        if m.group(1) == "1":
            assert "MUFU.SQRT" not in f and "MUFU.RSQ" not in f, name
    assert seen == 60
