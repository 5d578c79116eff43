"""fp64 results and worst-case entrywise bounds for the Kronecker operator with several terms (the linear model of
coregionalisation, LCMKernel; csrc/kron.cu, gp_plan_set_kron_terms):

    K = sum_q (s_q K_q) (x) B_q   over interleaved rows i T + a,   q = 0 .. Q-1

A term is a dict {kind, x1, x2 (None: square), ls, os, B, geo}: its own inputs (active dimensions), kind, lengthscale,
outputscale, T x T task covariance and its data plan's geometry (ko.geometry).  Test infrastructure for test_lcm_host.py and
test_gpu_lcm.py; it builds on tests/multitask_oracle.py (mo), whose single-term results and bounds it sums.

Bounds (u = 2^-24).
  Product.  Term q runs exactly the single-term pipeline up to its split slots (the B_q mix, ceil(T t / 16) launches of its data
    plan's fused kernel), so mo.kron_bound_q covers the mix, the kernel and the nsplit_q fp32 slot adds, plus one rounding u of
    s_q A_q, A_q = s_q |K_q| Wabs_q, for a multiply by s_q.  The scatter instead takes fmaf(s_q, v_q, acc) over the Q terms in
    order: each of the Q roundings is within u of the running |acc| <= sum_q A_q.  The parent's outputscale is 1 (exact), so
        bound = sum_q mo.kron_bound_q + Q u sum_q A_q   (+ u (|exact| + bound + |noise V|) for the finish's noise fmaf).
  Gradients.  gp_kron_terms_grad runs the single-term passes per term with that term's B_q, so term q's lengthscale,
    outputscale and dB bounds are mo.kron_grad_bound_q and mo.kron_dB_bound_q.
  Rows and diagonal.  Q fmaf roundings of the running sum of s_q k_q B_q[a, b] on top of each term's data-plan rows:
        bound = (Q + 1) u sum_q |s_q k_q B_q[a, b]| + sum_q |B_q[a, b]| rowtol_q
    rowtol_q the data plan's own gp_krows error (3xTF32 packing; ROW_REL of s_q, a documented tolerance, not derived here).
Mutants the bounds must catch: a term's B swapped for another's ("swap_B"), an s_q dropped ("drop_s") and a term skipped
("skip_term")."""
from __future__ import annotations

import torch

import kmv_oracle as ko
import multitask_oracle as mo
from oracle import kernels as ok

U32 = mo.U32
ROW_REL = 2.0 ** -16   # gp_krows of a plain plan: relative to s (the rows are evaluated from the packed, centred inputs)


def term(kind, x1, x2, ls, os_, B, backend="simt", n_sm=132):
    n2 = (x1 if x2 is None else x2).size(0)
    return dict(kind=kind, x1=x1, x2=x2, ls=ls, os=os_, B=B, geo=ko.geometry(x1.size(0), n2, x1.size(1), backend, n_sm))


def _mutated(terms, mutant, mutant_arg):
    """The terms a deliberately wrong engine would use."""
    out = [dict(t) for t in terms]
    if mutant == "swap_B":
        q = mutant_arg
        out[q]["B"] = terms[(q + 1) % len(terms)]["B"]
    elif mutant == "drop_s":
        out[mutant_arg]["os"] = 1.0
    elif mutant == "skip_term":
        out.pop(mutant_arg)
    return out


def dense(terms):
    """sum_q (s_q K_q) (x) B_q as a dense fp64 matrix (autograd-capable in ls / os / B)."""
    out = 0.0
    for t in terms:
        same = t["x2"] is None
        k = ok.kernel_matrix(t["kind"], t["x1"].double(), (t["x1"] if same else t["x2"]).double(), t["ls"], t["os"], same)
        out = out + torch.kron(k, t["B"].double() if torch.is_tensor(t["B"]) else torch.as_tensor(t["B"], dtype=torch.float64))
    return out


def exact(terms, V, T, t, noise=0.0, mutant=None, mutant_arg=None):
    """fp64 (sum_q (s_q K_q) (x) B_q) V (+ noise V on a square operator) [N1 T, t], term by term."""
    out = 0.0
    for tm in _mutated(terms, mutant, mutant_arg):
        out = out + mo.kron_exact(tm["kind"], tm["x1"], tm["x2"], tm["B"], tm["ls"], tm["os"], V, T, t)
    if terms[0]["x2"] is None and noise:
        out = out + float(mo.bo.f32(noise)) * V.double().to(out.device)
    return out


def bound(terms, V, T, t, exact_=None, noise=0.0):
    """Worst-case |engine - exact| [N1 T, t] of gp_kmv (module docstring); `exact_` is needed with noise."""
    Q = len(terms)
    out, tot = 0.0, 0.0
    for tm in terms:
        out = out + mo.kron_bound(tm["kind"], tm["x1"], tm["x2"], tm["B"], tm["ls"], tm["os"], V, T, t, tm["geo"])
        dev = tm["x1"].device
        _, Wabs = mo.kron_mix(tm["B"], V.double().to(dev), T, t)
        same = tm["x2"] is None
        tot = tot + ko.exact(tm["kind"], tm["x1"], tm["x2"], tm["ls"], tm["os"], 0.0, Wabs, same=same).reshape(-1, t)
    out = out + Q * U32 * tot
    if terms[0]["x2"] is None and noise:
        out = out + U32 * (exact_.abs() + out + float(mo.bo.f32(noise)) * V.double().to(out.device).abs())
    return out


def rows_bound(terms, idx):
    """Bound on |engine - dense[idx]| of gp_krows (module docstring) [m, N2 T]."""
    Q = len(terms)
    absum, tol = 0.0, 0.0
    for tm in terms:
        Ba = tm["B"].double().abs()
        absum = absum + dense([dict(tm, os=abs(tm["os"]), B=Ba)])[idx]
        n2 = (tm["x1"] if tm["x2"] is None else tm["x2"]).size(0)
        tol = tol + ROW_REL * abs(tm["os"]) * torch.kron(torch.ones(tm["x1"].size(0), n2, dtype=torch.float64), Ba)[idx]
    return (Q + 1) * U32 * absum + tol


def diag(terms, mutant=None, mutant_arg=None):
    """fp64 sum_q s_q k_q(x1_i, x2_i) B_q[a, a] at row i T + a."""
    out = 0.0
    for tm in _mutated(terms, mutant, mutant_arg):
        x2 = tm["x1"] if tm["x2"] is None else tm["x2"]
        kd = torch.stack([ok.kernel_matrix(tm["kind"], tm["x1"][i:i + 1].double(), x2[i:i + 1].double(), tm["ls"], tm["os"],
                                           tm["x2"] is None)[0, 0] for i in range(tm["x1"].size(0))])
        out = out + torch.kron(kd, torch.diagonal(tm["B"].double()))
    return out


def grads(terms, L, R, T, t):
    """Per term (dF/dl_q, dF/ds_q, dF/dB_q) of F = sum L . (K R) in fp64."""
    out = []
    for tm in terms:
        gl, gs = mo.kron_grad(tm["kind"], tm["x1"], tm["x2"], tm["B"], tm["ls"], tm["os"], L, R, T, t)
        dB = mo.kron_dB(tm["kind"], tm["x1"], tm["x2"], tm["ls"], tm["os"], L, R, T, t)
        out.append((gl, gs, dB))
    return out


def grads_bound(terms, L, R, T, t, n_sm=132):
    """Per term (bound on dl_q, on ds_q, on dB_q) of gp_kron_terms_grad: the single-term bounds with the term's B_q."""
    out = []
    for tm in terms:
        geo = tm["geo"]
        tc = geo["backend"] == "tcgen05"
        path = "tc" if tc and (not torch.is_tensor(tm["ls"]) or torch.as_tensor(tm["ls"]).numel() == 1) else "simt"
        a, s = mo.kron_grad_bound(tm["kind"], tm["x1"], tm["x2"], tm["B"], tm["ls"], tm["os"], L, R, T, t, path, n_sm=n_sm)
        dB = mo.kron_dB_bound(tm["kind"], tm["x1"], tm["x2"], tm["ls"], tm["os"], L, R, T, t, geo)
        out.append((a, s, dB))
    return out
