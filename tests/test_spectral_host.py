"""Host-side tests of the spectral mixture kernel: the fp64 oracle against the reference's own covariances and gradients, the
kernel's parameters and initialisation, dispatch and refusals of the operator, the C ABI, and the compiled code of
csrc/spectral.cu (no local memory, 2 Q d MUFU operations per pair)."""
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import spectral_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpytorch_b200", "lib", "libgpbbmm.so")
SRC = os.path.join(ROOT, "gpytorch_b200", "csrc", "spectral.cu")
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "spectral_golden.npz"))
NCASES = len([k for k in GOLD.files if k.endswith("_shape")])


def _case(ci):
    g = {k[len(f"c{ci}_"):]: torch.from_numpy(GOLD[k]) for k in GOLD.files if k.startswith(f"c{ci}_")}
    return g


@pytest.mark.parametrize("ci", range(NCASES))
def test_oracle_matches_reference_golden(ci):
    g = _case(ci)
    Q, d = g["shape"].tolist()
    assert so.covariance(g["x1"], g["x2"], g["w"], g["mu"], g["v"]).sub(g["K12"]).abs().max() < 1e-12
    assert so.covariance(g["x1"], g["x1"], g["w"], g["mu"], g["v"]).sub(g["K11"]).abs().max() < 1e-12
    assert so.covariance(g["x1"], g["x1"], g["w"], g["mu"], g["v"], diag=True).sub(g["diag"]).abs().max() < 1e-12
    m = g["diag12"].numel()
    assert so.covariance(g["x1"][:m], g["x2"][:m], g["w"], g["mu"], g["v"], diag=True).sub(g["diag12"]).abs().max() < 1e-12
    # the square diagonal is the constant (sum_q w_q)^d
    assert torch.allclose(g["diag"], g["w"].sum().pow(d).expand_as(g["diag"]), rtol=1e-14, atol=0)
    # the oracle's gradients (fp64 autograd through the same covariance) match the reference's
    w, mu, v = (t.clone().requires_grad_(True) for t in (g["w"], g["mu"], g["v"]))
    K = so.covariance_torch(g["x1"], g["x2"], w, mu, v)
    assert K.detach().sub(g["K12"]).abs().max() < 1e-12
    (K * g["W"]).sum().backward()
    for got, ref in ((w.grad, g["gw"]), (mu.grad, g["gmu"]), (v.grad, g["gv"])):
        assert got.shape == ref.shape and (got - ref).abs().max() <= 1e-12 * max(1.0, ref.abs().max().item())


def test_oracle_matches_batched_golden():
    K = torch.from_numpy(GOLD["b_K"])
    for b in range(2):
        x = torch.from_numpy(GOLD["b_x"][b])
        ref = so.covariance(x, x, GOLD["b_w"][b], GOLD["b_mu"][b], GOLD["b_v"][b])
        assert (ref - K[b]).abs().max() < 1e-12


def test_entry_bound_does_not_grow_with_x():
    w, mu, v = [0.7, 0.4], [[0.49], [0.13]], [[0.02], [0.05]]
    x = torch.arange(0, 64, dtype=torch.float64).reshape(-1, 1)
    far = x + 99_000.0
    b0 = so.entry_bound(x, x, w, mu, v)
    b1 = so.entry_bound(far, far, w, mu, v)
    assert torch.allclose(b0, b1, rtol=1e-12, atol=0)
    assert b0.max() < 1e-5


def test_parameters_constraints_setters_and_error_texts():
    from gpytorch_b200 import constraints, kernels

    with pytest.raises(RuntimeError, match="num_mixtures is a required argument"):
        kernels.SpectralMixtureKernel()
    k = kernels.SpectralMixtureKernel(num_mixtures=4, ard_num_dims=3)
    assert k.raw_mixture_weights.shape == (4,)
    assert k.raw_mixture_means.shape == (4, 1, 3) and k.raw_mixture_scales.shape == (4, 1, 3)
    for name in ("raw_mixture_weights", "raw_mixture_means", "raw_mixture_scales"):
        assert isinstance(getattr(k, name + "_constraint"), constraints.Positive)
    kb = kernels.SpectralMixtureKernel(num_mixtures=2, ard_num_dims=1, batch_shape=torch.Size([3]))
    assert kb.raw_mixture_weights.shape == (3, 2) and kb.raw_mixture_means.shape == (3, 2, 1, 1)
    k.mixture_weights = torch.tensor([0.5, 1.0, 1.5, 2.0])
    k.mixture_means = 0.25
    k.mixture_scales = torch.full((4, 1, 3), 0.125)
    assert torch.allclose(k.mixture_weights, torch.tensor([0.5, 1.0, 1.5, 2.0]), rtol=1e-6)
    assert torch.allclose(k.mixture_means, torch.full((4, 1, 3), 0.25), rtol=1e-6)
    assert torch.allclose(k.mixture_scales, torch.full((4, 1, 3), 0.125), rtol=1e-6)
    k.initialize(mixture_weights=3.0)
    assert torch.allclose(k.mixture_weights, torch.full((4,), 3.0), rtol=1e-6)
    with pytest.raises(RuntimeError, match=r"The SpectralMixtureKernel expected the input to have 3 dimensionality \(based on the "
                                           r"ard_num_dims argument\). Got 2\."):
        k(torch.rand(5, 2))
    with pytest.raises(RuntimeError, match="train_x and train_y should be tensors"):
        k.initialize_from_data([1.0], torch.ones(1))
    custom = constraints.GreaterThan(1e-4)
    assert kernels.SpectralMixtureKernel(num_mixtures=1, mixture_means_constraint=custom).raw_mixture_means_constraint is custom


@pytest.mark.parametrize("ii", range(3))
def test_initialize_from_data_matches_reference(ii):
    from gpytorch_b200 import kernels

    Q, d, n, b = GOLD[f"i{ii}_cfg"].tolist()
    k = kernels.SpectralMixtureKernel(num_mixtures=Q, ard_num_dims=d, batch_shape=torch.Size([b]) if b else None)
    torch.manual_seed(100 + ii)
    k.initialize_from_data(torch.from_numpy(GOLD[f"i{ii}_x"]), torch.from_numpy(GOLD[f"i{ii}_y"]))
    for name in ("w", "mu", "v"):
        got = {"w": k.mixture_weights, "mu": k.mixture_means, "v": k.mixture_scales}[name].detach()
        ref = torch.from_numpy(GOLD[f"i{ii}_{name}"])
        assert got.shape == ref.shape
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-7), name


def test_initialize_from_data_empspect():
    if importlib.util.find_spec("sklearn") is None:
        pytest.skip("scikit-learn is not installed")
    from gpytorch_b200 import kernels

    x = torch.linspace(0, 1, 200)
    y = torch.sin(2 * torch.pi * 12 * x) + 0.5 * torch.sin(2 * torch.pi * 40 * x)
    np.random.seed(0)
    k = kernels.SpectralMixtureKernel(num_mixtures=2)
    k.initialize_from_data_empspect(x, y)
    assert k.mixture_means.shape == (2, 1, 1) and k.mixture_scales.shape == (2, 1, 1)
    assert torch.isfinite(k.mixture_means).all() and (k.mixture_weights > 0).all()
    # the fitted frequencies (in cycles per sample of the 200-point grid) sit at the two spectral peaks
    f = sorted((k.mixture_means.reshape(-1) * 199).tolist())
    assert abs(f[0] - 12) < 3 and abs(f[1] - 40) < 3


def _params(k, b=None):
    w, mu, v = k.mixture_weights, k.mixture_means, k.mixture_scales
    return (w, mu, v) if b is None else (w[b], mu[b], v[b])


def test_dispatch_plain_scaled_batched_and_active_dims():
    from gpytorch_b200 import kernels
    from gpytorch_b200.operators import BatchLinearOperator, SpectralMixtureKernelLinearOperator

    x = torch.rand(7, 2)
    k = kernels.SpectralMixtureKernel(num_mixtures=3, ard_num_dims=2)
    op = k(x)
    assert isinstance(op, SpectralMixtureKernelLinearOperator) and op.same and op.shape == (7, 7)
    assert len(op.hyper_tensors()) == 3 and all(torch.equal(a, b) for a, b in zip(op.hyper_tensors(), _params(k)))
    op2 = k(x, torch.rand(4, 2))
    assert not op2.same and op2.shape == (7, 4)
    assert op2._transpose_nonbatch().shape == (4, 7)
    sk = kernels.ScaleKernel(kernels.SpectralMixtureKernel(num_mixtures=3, ard_num_dims=2))
    sop = sk(x)
    assert isinstance(sop, SpectralMixtureKernelLinearOperator)
    assert len(sop.hyper_tensors()) == 4 and torch.equal(sop.hyper_tensors()[3], sk.outputscale)
    kb = kernels.ScaleKernel(kernels.SpectralMixtureKernel(num_mixtures=2, ard_num_dims=1, batch_shape=torch.Size([2])))
    bop = kb(torch.rand(2, 5, 1))
    assert isinstance(bop, BatchLinearOperator) and len(bop.ops) == 2
    for b, o in enumerate(bop.ops):
        w, mu, v = _params(kb.base_kernel, b)
        assert torch.equal(o.weights, w) and torch.equal(o.means, mu) and torch.equal(o.scales, v)
        assert torch.equal(o.outputscale, kb.outputscale[b])
    ka = kernels.SpectralMixtureKernel(num_mixtures=2, ard_num_dims=1, active_dims=[2])
    x3 = torch.rand(6, 3)
    aop = ka(x3)
    assert aop.x1.shape == (6, 1) and torch.equal(aop.x1[:, 0], x3[:, 2])
    sub = op[2:5, 0:3]
    assert isinstance(sub, SpectralMixtureKernelLinearOperator) and sub.shape == (3, 3) and not sub.same
    assert op.detach().hyper_tensors()[0].requires_grad is False


def test_refusals():
    from gpytorch_b200 import kernels
    from gpytorch_b200.operators import (AddedDiagLinearOperator, ConstantDiagLinearOperator, KernelLinearOperator,
                                         SpectralMixtureKernelLinearOperator)

    x = torch.rand(6, 1)
    k = kernels.SpectralMixtureKernel(num_mixtures=2)
    with pytest.raises(NotImplementedError, match="sums that contain spectral mixture operators"):
        (k + kernels.RBFKernel())(x)
    with pytest.raises(NotImplementedError, match="sums that contain spectral mixture operators"):
        (kernels.RBFKernel() + k)(x)
    with pytest.raises(NotImplementedError, match="ProductKernel factors"):
        k * kernels.RBFKernel()
    with pytest.raises(NotImplementedError, match="SpectralMixtureKernel base kernel of a GridInterpolationKernel"):
        kernels.GridInterpolationKernel(k, grid_size=16, num_dims=1)
    with pytest.raises(NotImplementedError, match="inputs of a spectral mixture operator"):
        k(x.clone().requires_grad_(True))
    op = k(x)
    plain = KernelLinearOperator(x, None, "rbf", torch.tensor(1.0))
    with pytest.raises(NotImplementedError, match="sums that contain spectral mixture operators"):
        op + plain
    with pytest.raises(NotImplementedError, match="sums that contain spectral mixture operators"):
        plain + op
    with pytest.raises(NotImplementedError, match="products that contain a spectral mixture operator"):
        op.mul(plain)
    with pytest.raises(NotImplementedError, match="IndexKernel operator only"):
        plain.mul(op)
    with pytest.raises(NotImplementedError, match="inputs of a spectral mixture operator"):
        op._input_grad_list(None, None, [True])
    with pytest.raises(NotImplementedError, match="inputs of a spectral mixture operator"):
        op._dense_input_grad_list(None, [True])
    with pytest.raises(NotImplementedError, match="num_mixtures <= 16"):
        kernels.SpectralMixtureKernel(num_mixtures=17)(x)
    with pytest.raises(NotImplementedError, match="num_mixtures \\* d <= 32"):
        kernels.SpectralMixtureKernel(num_mixtures=9, ard_num_dims=4)(torch.rand(5, 4))
    with pytest.raises(NotImplementedError, match="d <= 8"):
        kernels.SpectralMixtureKernel(num_mixtures=1, ard_num_dims=9)(torch.rand(5, 9))
    assert isinstance(op + ConstantDiagLinearOperator(torch.tensor(0.1), 6), AddedDiagLinearOperator)
    assert isinstance(op, SpectralMixtureKernelLinearOperator)


class _FakePlan:
    def __init__(self, gl, go):
        self.gl, self.go = gl, go

    def bilinear_grad(self, left, right):
        return self.gl, self.go


@pytest.mark.parametrize("scaled", [False, True])
def test_gradient_vectors_split_onto_parameter_shapes(scaled):
    from gpytorch_b200 import kernels

    Q, d = 3, 2
    k = kernels.SpectralMixtureKernel(num_mixtures=Q, ard_num_dims=d, batch_shape=torch.Size([2]))
    sk = kernels.ScaleKernel(k) if scaled else k
    op = sk(torch.rand(2, 5, d)).ops[1]
    gl = [float(i) for i in range(Q * (1 + 2 * d))]
    op.plan = lambda noise=0.0: _FakePlan(gl, 99.0)
    out = op._bilinear_derivative_list(None, None)
    assert len(out) == (4 if scaled else 3)
    assert out[0].shape == (Q,) and out[0].tolist() == gl[:Q]
    assert out[1].shape == (Q, 1, d) and out[1].reshape(-1).tolist() == gl[Q:Q + Q * d]
    assert out[2].shape == (Q, 1, d) and out[2].reshape(-1).tolist() == gl[Q + Q * d:]
    if scaled:
        assert out[3].shape == () and out[3].item() == 99.0
    # autograd takes them through the batch element's slices back to the [2, ...] parameters
    for t, gr in zip(op.hyper_tensors(), out):
        assert t.shape == gr.shape


class _SlotPlan:
    def set_hypers(self, *args):
        return self

    def set_spectral(self, *args):
        return self


def test_plan_slots_keep_low_rank_spectral_plans_apart(monkeypatch):
    """An ordinary spectral operator, the spectral base of a low-rank (LOVE) operator and a plain low-rank base ask the plan cache
    for three different slots: a plan carrying U never serves an ordinary spectral operator, and a spectral plan never serves a
    plain one."""
    from gpytorch_b200 import kernels, operators

    slots = []

    def fake_get_plan(x1, x2, backend, row_begin, row_count, comm, slot=0, owner=None):
        slots.append(slot)
        return _SlotPlan()

    monkeypatch.setattr(operators, "_get_plan", fake_get_plan)
    x = torch.rand(6, 1)
    k = kernels.ScaleKernel(kernels.SpectralMixtureKernel(num_mixtures=2))
    U = torch.rand(6, 2)
    k(x).plan()
    operators.LowRankUpdatedKernelLinearOperator(k(x), U).base.plan()
    operators.LowRankUpdatedKernelLinearOperator(operators.KernelLinearOperator(x, None, "rbf", torch.tensor(1.0)), U).base.plan()
    assert slots == [operators._SPECTRAL_SLOT, operators._SPECTRAL_LOWRANK_SLOT, operators._LOWRANK_SLOT]
    assert len(set(slots)) == 3


def test_c_abi_declares_set_spectral_and_every_refusal():
    hdr = open(os.path.join(ROOT, "include", "gp_bbmm.h")).read()
    assert re.search(r"int gp_plan_set_spectral\(gp_plan\* plan, int Q, const float\* weights, const float\* means, "
                     r"const float\* scales, int d\);", hdr)
    from gpytorch_b200 import _lib

    F = _lib.C.POINTER(_lib._F)
    assert _lib.PROTOTYPES["gp_plan_set_spectral"] == (_lib._I, [_lib._P, _lib._I, F, F, F, _lib._I])
    src = "".join(open(os.path.join(ROOT, "gpytorch_b200", "csrc", f)).read()
                  for f in ("api.cu", "xgrad.cu", "tasks.cu", "kron.cu", "deriv.cu", "sum.cu", "product.cu", "ski.cu", "additive.cu"))
    for call in ("gp_plan_set_backend", "gp_plan_set_tasks", "gp_plan_set_kron", "gp_plan_set_sum", "gp_plan_set_product",
                 "gp_plan_set_ski", "gp_plan_set_additive"):
        assert f'GP_REFUSE_SPECTRAL(p, "{call}")' in src, call
    assert src.count("GP_REFUSE_SPECTRAL(p, what)") == 2   # the input-gradient calls and gp_plan_set_deriv(_kind)
    assert "gp_plan_set_comm with more than one rank is not available on a spectral mixture plan" in src
    assert "a spectral mixture plan as a term is not available" in src and "a spectral mixture plan as a factor is not available" in src
    assert 'GP_REFUSE_SPECTRAL(data, "gp_plan_set_kron (as the data plan)")' in src
    assert "(as the data plan) is not available on a spectral mixture plan" in src


def test_ptxas_reports_no_spills_for_any_instantiation():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"spectral_ptxas_{os.getpid()}.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas",
                        "-v", "-c", SRC, "-o", out], capture_output=True, text=True, timeout=900)
    if os.path.exists(out):
        os.remove(out)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert sum("spectral_kmv_kernel" in e for e in entries) == 22 and sum("spectral_bilinear_kernel" in e for e in entries) == 22
    assert len(spills) == len(entries)
    assert all(s == ("0", "0", "0") for s in spills)


def test_kmv_sass_has_one_ex2_and_one_cos_per_component_dimension_and_pair():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libgpbbmm.so not available (python -m gpytorch_b200.build)")
    r = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0
    seen = 0
    for f in re.split(r"\n\s*Function : ", r.stdout):
        name = f.split("\n", 1)[0].strip()
        m = re.match(r"_ZN2gp19spectral_kmv_kernelILi(\d)ELi(\d+)EEEv", name)
        if not m:
            continue
        seen += 1
        D, QM = int(m.group(1)), int(m.group(2))
        # the pair loop is unrolled twice over QM x D statically unrolled terms: one ex2 and one cos each, run for q < Q only
        assert len(re.findall(r"MUFU\.EX2", f)) == 2 * QM * D, name
        assert len(re.findall(r"MUFU\.COS", f)) == 2 * QM * D, name
        assert "MUFU.SIN" not in f, name
    assert seen == 22
