"""CPU checks of the linear model of coregionalisation (LCMKernel, gp_plan_set_kron_terms): the fp64 oracle against a hand-built
matrix, against the Kronecker oracle at Q = 1 and against the identity sum_q K (x) B_q = K (x) sum_q B_q; its bounds catching the
mutants; LCMKernel's parameter tree and refusals; the exported C symbols and the new kernels' resources."""
import os
import re
import subprocess

import pytest
import torch

import kmv_oracle as ko
import kron_oracle as kr
import lcm_oracle as lo
import multitask_oracle as mo
from oracle import kernels as ok

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _terms(Q, T, n=40, d=3, cross=False, seed=0):
    kinds = ["rbf", "matern52", "matern12", "matern32"]
    x = ko.points(n, d, seed)
    x2 = ko.points(n + 7, d, seed + 1) if cross else None
    out = []
    for q in range(Q):
        dims = [c for c in range(d) if c != q % d] if q else list(range(d))   # different active dimensions per term
        out.append(lo.term(kinds[q % 4], x[:, dims], None if x2 is None else x2[:, dims], 0.3 + 0.4 * q, 0.7 + 0.5 * q,
                           mo.random_B(T, seed + 10 + q)))
    return out


def test_dense_matches_hand_built_matrix():
    terms = _terms(2, 3, n=5)
    A = lo.dense(terms)
    N, T = 5, 3
    for r in range(N * T):
        for c in range(N * T):
            want = 0.0
            for tm in terms:
                k = ok.kernel_matrix(tm["kind"], tm["x1"][r // T:r // T + 1].double(), tm["x1"][c // T:c // T + 1].double(),
                                     tm["ls"], tm["os"], r // T == c // T)[0, 0]
                want += float(k) * float(tm["B"][r % T, c % T])
            assert abs(float(A[r, c]) - want) <= 1e-12 * max(1.0, abs(want))


@pytest.mark.parametrize("cross", [False, True])
def test_products_equal_dense_and_q1_equals_kronecker(cross):
    T, t = 3, 5
    terms = _terms(3, T, cross=cross)
    n2 = terms[0]["x1"].size(0) if not cross else terms[0]["x2"].size(0)
    V = torch.randn(n2 * T, t, generator=torch.Generator().manual_seed(3))
    # kmv_oracle's fp64 evaluation and the dense oracle differ in the last ~1e-7 (it works from the engine's centred inputs)
    ref = lo.dense(terms) @ V.double()
    assert float((lo.exact(terms, V, T, t) - ref).abs().max()) <= 1e-7 * float(ref.abs().max())
    tm = terms[0]
    one = mo.kron_exact(tm["kind"], tm["x1"], tm["x2"], tm["B"], tm["ls"], tm["os"], V, T, t)
    assert torch.equal(lo.exact([tm], V, T, t), one)
    x2 = tm["x1"] if tm["x2"] is None else tm["x2"]
    K1 = kr.kron_matrix(tm["kind"], tm["x1"].double(), x2.double(), tm["ls"], tm["os"], tm["B"].double(), not cross)
    assert torch.allclose(lo.dense([tm]), K1, rtol=1e-12, atol=1e-12)


def test_terms_sharing_one_kernel_sum_their_task_covariances():
    T = 4
    x = ko.points(30, 2, 7)
    Bs = [mo.random_B(T, 20 + q) for q in range(3)]
    terms = [lo.term("matern32", x, None, 0.4, 1.1, B) for B in Bs]
    K = ok.kernel_matrix("matern32", x.double(), x.double(), 0.4, 1.1, True)
    assert torch.allclose(lo.dense(terms), torch.kron(K, sum(B.double() for B in Bs)), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("mutant,arg", [("swap_B", 0), ("swap_B", 1), ("drop_s", 1), ("skip_term", 2)])
def test_bounds_catch_mutants(mutant, arg):
    T, t = 3, 4
    terms = _terms(3, T)
    V = torch.randn(terms[0]["x1"].size(0) * T, t, generator=torch.Generator().manual_seed(5))
    ref = lo.exact(terms, V, T, t)
    bnd = lo.bound(terms, V, T, t)
    assert bool((bnd > 0).all()) and float(bnd.max()) < 1e-3 * float(ref.abs().max())
    bad = lo.exact(terms, V, T, t, mutant=mutant, mutant_arg=arg)
    assert bool(((bad - ref).abs() > bnd).any())
    if mutant in ("skip_term", "swap_B", "drop_s"):
        d, dbad = lo.diag(terms), lo.diag(terms, mutant, arg)
        # the diagonal of a term swap or a dropped scale only moves where B_q[a, a] or s_q changes it
        assert bool(((dbad - d).abs() > (len(terms) + 1) * lo.U32 * d.abs() + lo.ROW_REL * 10).any())


def test_gradients_and_bounds_per_term():
    T, t = 2, 3
    terms = _terms(2, T, n=30)
    n = 30
    L = torch.randn(n * T, t, generator=torch.Generator().manual_seed(8))
    R = torch.randn(n * T, t, generator=torch.Generator().manual_seed(9))
    got = lo.grads(terms, L, R, T, t)
    for tm, (gl, gs, dB) in zip(terms, got):
        ls = torch.tensor(float(tm["ls"]), dtype=torch.float64, requires_grad=True)
        os_ = torch.tensor(float(tm["os"]), dtype=torch.float64, requires_grad=True)
        B = tm["B"].double().clone().requires_grad_(True)
        F = (L.double() * (lo.dense([dict(tm, ls=ls, os=os_, B=B)]) @ R.double())).sum()
        F.backward()
        assert abs(float(torch.as_tensor(gl).reshape(-1)[0]) - float(ls.grad)) <= 1e-6 * max(1.0, abs(float(ls.grad)))
        assert abs(float(gs) - float(os_.grad)) <= 1e-6 * max(1.0, abs(float(os_.grad)))
        assert float((dB - B.grad).abs().max()) <= 1e-6 * float(B.grad.abs().max())
    for (a, s, dB) in lo.grads_bound(terms, L, R, T, t):
        assert float(torch.as_tensor(a).max()) > 0 and float(s) > 0 and bool((dB > 0).all())


def test_lcm_kernel_parameter_tree_matches_reference():
    from gpytorch_b200 import kernels as K

    k = K.LCMKernel([K.RBFKernel(), K.ScaleKernel(K.MaternKernel(nu=2.5))], num_tasks=3, rank=[1, 2])
    names = {n: tuple(p.shape) for n, p in k.named_parameters()}
    assert names == {
        "covar_module_list.0.task_covar_module.covar_factor": (3, 1),
        "covar_module_list.0.task_covar_module.raw_var": (3,),
        "covar_module_list.0.data_covar_module.raw_lengthscale": (1, 1),
        "covar_module_list.1.task_covar_module.covar_factor": (3, 2),
        "covar_module_list.1.task_covar_module.raw_var": (3,),
        "covar_module_list.1.data_covar_module.raw_outputscale": (),
        "covar_module_list.1.data_covar_module.base_kernel.raw_lengthscale": (1, 1),
    }
    assert k.num_outputs_per_input(torch.zeros(4, 1), torch.zeros(4, 1)) == 3
    assert isinstance(k.covar_module_list[0], K.MultitaskKernel)
    assert len(K.LCMKernel([K.RBFKernel()], num_tasks=2, rank=1).covar_module_list) == 1


def test_lcm_kernel_refusals():
    from gpytorch_b200 import kernels as K

    with pytest.raises(ValueError, match="At least one base kernel must be provided."):
        K.LCMKernel([], num_tasks=2)
    with pytest.raises(ValueError, match="base_kernels must only contain Kernel objects"):
        K.LCMKernel([K.RBFKernel(), torch.nn.Linear(1, 1)], num_tasks=2)
    with pytest.raises(NotImplementedError, match="up to 4 base kernels"):
        K.LCMKernel([K.RBFKernel() for _ in range(5)], num_tasks=2)
    with pytest.raises(NotImplementedError, match="priors"):
        K.LCMKernel([K.RBFKernel()], num_tasks=2, task_covar_prior=object())
    with pytest.raises(NotImplementedError, match="ScaleKernel\\(LCMKernel"):
        K.ScaleKernel(K.LCMKernel([K.RBFKernel(), K.RBFKernel()], num_tasks=2))
    x = torch.zeros(4, 1)
    # a base kernel MultitaskKernel refuses is refused with MultitaskKernel's words (before any device work)
    with pytest.raises(NotImplementedError, match="an RQKernel data kernel of a MultitaskKernel"):
        K.LCMKernel([K.RBFKernel(), K.RQKernel()], num_tasks=2)(x)


def test_c_symbols_exported():
    from gpytorch_b200 import build

    lib = build.build()
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    for sym in ("gp_plan_set_kron_terms", "gp_plan_set_kron_term_covars", "gp_kron_terms_grad"):
        assert re.search(rf"\bT {sym}\b", out), sym
    hdr = open(os.path.join(REPO, "include", "gp_bbmm.h")).read()
    for sym in ("gp_plan_set_kron_terms", "gp_plan_set_kron_term_covars", "gp_kron_terms_grad"):
        assert f"int {sym}(" in hdr


@pytest.mark.parametrize("src,kernels", [
    ("kron", ["lcm_scatter_kernel", "lcm_expand_rows_kernel", "lcm_expand_diag_kernel"]),
    ("pivchol", ["pc_persistent1_kernelILi73E", "pc_init_kron_terms_kernel"]),
])
def test_new_kernels_use_no_local_memory(src, kernels):
    from gpytorch_b200 import build

    build.build()
    log = open(os.path.join(build.OBJDIR, f"{src}.o.log")).read()
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    for name in kernels:
        hit = [b for b in blocks if name in b.split("'")[1 if b.startswith("'") else 0]]
        assert hit, name
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in hit[0], (name, hit[0][:400])
