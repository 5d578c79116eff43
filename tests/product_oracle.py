"""fp64 oracle of kernel products  K = prod_f s_f k_f(x1[:, dims_f], x2[:, dims_f])  (ProductKernel; csrc/product.cu): the dense
product from oracle/kernels.py:kernel_matrix on the active-dimension slices, its K.V with a worst-case bound per output entry, the
MLL through a Cholesky factor, and the hyper-parameter gradients by fp64 autograd.  Test infrastructure for test_product_host.py
and test_gpu_product.py.

A factor is (kind, dims, lengthscale, outputscale): dims the active dimensions (a list), lengthscale a scalar or one value per
active dimension.  Hyper-parameters are taken as the fp32 values the engine holds.

The bound extends the per-pair model of tests/kmv_oracle.py / tests/bilinear_oracle.py to a product.  For factor f with the fp64
value k_f, bo.pair_arg gives the error da_f of the engine's argument on its path, bo._dev the change dk_f of k_f over that interval
and bo.pair_rel the relative evaluation error rel_f, so the engine's factor value lies within kabs_f = k_f (1 + rel_f) + dk_f.  The
engine forms (prod_f poly_f) ex2(sum_f e_f): one sqrt per Matern factor (inside rel_f), 2 n_f fp32 multiplies and adds on top (u
each) and ONE ex2 (rel_f counts one per factor, so the sum over-covers it).  Hence
    kabs  = prod_f kabs_f (1 + 2 n_f u)          bounds the engine's value of the pair
    pair  = kabs - prod_f k_f                    the pair's own error (+ 2^-19 kabs on the tensor cores: GEMM2's hi / lo splits)
and the sums are those of kmv_oracle.bound (eps_sums of the path, nsplit partial adds, the multiply by S); S itself is an fp32
product of n_f scales, n_f u more."""
from __future__ import annotations

import math

import torch

import bilinear_oracle as bo
import kmv_oracle as ko
from oracle import kernels as ok

U32 = bo.U32
# the cases of tests/golden/product_golden.npz: tag -> (n1, n2 (0: square), d, [(kind, dims, lengthscale, outputscale)])
GOLDEN_CASES = {
    "space_time": (9, 0, 3, [("rbf", [0, 1], 0.6, 1.3), ("matern12", [2], 0.9, 0.8)]),
    "rough_pair": (7, 11, 4, [("matern52", [0, 1, 2], 1.1, 1.0), ("matern12", [1, 3], 0.5, 2.0)]),
    "three": (8, 6, 3, [("rbf", [0], 0.4, 1.0), ("matern32", [1], 0.7, 0.5), ("matern52", [0, 2], 1.5, 1.2)]),
}


def _slice(x, dims):
    return x[:, list(dims)].contiguous()


def dense(factors, x1, x2=None):
    """fp64 dense product [n1, n2]; x2 None: the square operator with its exact diagonal.  Hyper-parameters may be fp64 tensors
    that require grad (the autograd reference of the gradients)."""
    K = None
    for kind, dims, ls, os_ in factors:
        a = _slice(x1.double(), dims)
        b = a if x2 is None else _slice(x2.double(), dims)
        Kf = ok.kernel_matrix(kind, a, b, ls, os_, x2 is None)
        K = Kf if K is None else K * Kf
    return K


def f32_factors(factors):
    """The factors with the fp32 values of their hyper-parameters (as fp64 tensors)."""
    return [(k, d, bo.f32(ls) if bo.f32(ls).numel() > 1 else bo.f32(ls)[0], bo.f32(os_)[0]) for k, d, ls, os_ in factors]


def mll_cholesky(K, y, noise):
    """log p(y) / n of N(0, K + noise I) in fp64, and (K + noise I)^-1 y."""
    n = K.size(0)
    L = torch.linalg.cholesky(K + noise * torch.eye(n, dtype=K.dtype))
    sol = torch.cholesky_solve(y.double().unsqueeze(-1), L).squeeze(-1)
    lp = -0.5 * ((y.double() * sol).sum() + 2 * L.diagonal().log().sum() + n * math.log(2 * math.pi)) / n
    return lp, sol


def bilinear_grads(factors, x1, x2, L, R):
    """fp64 autograd of F = sum(L * (K @ R)): [(dF/dl_f [1 or d_f], dF/ds_f)] per factor."""
    leaves = []
    for kind, dims, ls, os_ in factors:
        l = bo.f32(ls).clone().requires_grad_()
        s = bo.f32(os_)[0].clone().requires_grad_()
        leaves.append((kind, dims, l if l.numel() > 1 else l[0], s, l))
    K = dense([(k, d, l, s) for k, d, l, s, _ in leaves], x1, x2)
    F = (L.double() * (K @ R.double())).sum()
    flat = [t for _, _, _, s, l in leaves for t in (l, s)]
    g = torch.autograd.grad(F, flat)
    return [(g[2 * i].detach(), g[2 * i + 1].detach()) for i in range(len(leaves))]


def kv_and_bound(factors, x1, x2, V, path, nsplit, T_per_split, noise=0.0, block=None):
    """(fp64 S prod k V (+ noise V on a square plan) [n1, t], worst-case |engine - fp64| [n1, t]) on V's device.  path "tc"
    (product_tc_kernel) or "simt" (product_simt_kernel); nsplit, T_per_split: the product plan's column splits."""
    same = x2 is None
    dev = V.device
    Vd = V.double()
    Va = Vd.abs()
    nf = len(factors)
    S = 1.0
    packed = []
    for kind, dims, ls, os_ in factors:
        a = _slice(x1, dims).to(dev)
        b = None if same else _slice(x2, dims).to(dev)
        zr, zc, _ = ko._packed(kind, a, b, ls, same, 0, None)
        packed.append((kind, zr, zc, (zc * zc).sum(1), bo.dp_of(len(dims)), bo.kp_of(len(dims))))
        S *= float(bo.f32(os_))
    n1, n2 = packed[0][1].size(0), packed[0][2].size(0)
    if path == "tc":
        eps = ko.TC_CHAIN * (1 + 2.0 ** -11 + 2.0 ** -10) + 2 * U32 + T_per_split * U32
    else:
        eps = min(T_per_split * ko.TILE_J, n2) * U32
    eps += (nsplit + 1 + nf) * U32
    out = torch.empty(n1, Vd.size(1), dtype=torch.float64, device=dev)
    bnd = torch.empty_like(out)
    block = block or ko._block_rows(n2, sum(p[1].size(1) for p in packed), 256)
    for b in bo._blocks(n1, block):
        rows = torch.arange(b.stop - b.start, device=dev)
        g = torch.arange(b.start, b.stop, device=dev)
        k, kabs = 1.0, 1.0
        for kind, zr, zc, nr, DP, KP in packed:
            _, _, _, _, m, da = bo.pair_arg(zr[b], zc, nr, path, DP, KP)
            if same:
                m[rows, g] = 0.0
                da[rows, g] = 0.0
            kf, _ = bo._kg(kind, m)
            dkf, _ = bo._dev(kind, m, da)
            k = k * kf
            kabs = kabs * (kf * (1 + bo.pair_rel(m)) + dkf)
        kabs = kabs * (1 + 2 * nf * U32)
        pair = kabs - k
        if path == "tc":
            pair = pair + 2.0 ** -19 * kabs
        A = kabs @ Va
        out[b] = S * (k @ Vd)
        bnd[b] = S * (pair @ Va + eps * A)
        if same and noise:
            nz = float(bo.f32(noise))
            out[b] += nz * Vd[g]
            bnd[b] += U32 * (S * A + nz * Va[g])
    return out, bnd


def geometry(n1, n2, factor_dims, backends, n_sm=132):
    """product.cu's product_pack: (path, nsplit, tiles per split, total KP, total DP) of a product plan whose factors have
    len(dims) = factor_dims and the given backends ("tcgen05" / "simt" / "auto")."""
    kps = [bo.kp_of(d) for d in factor_dims]
    tc_f = [(b == "tcgen05" or (b == "auto" and kp <= ko.KP_MAX)) for b, kp in zip(backends, kps)]
    tc = len(factor_dims) == 2 and all(tc_f) and sum(kps) <= ko.KP_MAX
    rows_pad = ko.cdiv(n1, 2 * ko.TILE_I) * 2 * ko.TILE_I
    nti = rows_pad // ko.TILE_I if tc else ko.cdiv(n1, ko.SIMT_TI)
    ntj = ko.cdiv(n2, ko.TILE_J)
    slots = n_sm * (2 if tc else 1)
    best, best_eff = 1, -1.0
    for s in range(1, 17):
        if s > ntj:
            break
        per = ko.cdiv(ntj, s)
        if s > 1 and per < 8:
            break
        waves = ko.cdiv(nti * s, slots)
        eff = float(nti * ntj) / float(waves * slots * per)
        if eff > best_eff + 0.02:
            best_eff, best = eff, s
    tps = ko.cdiv(ntj, best)
    return {"path": "tc" if tc else "simt", "nsplit": ko.cdiv(ntj, tps), "T": tps, "KP": sum(kps),
            "DP": sum(bo.dp_of(d) for d in factor_dims)}


def ring_depth(KP):
    """Stages of product_tc_kernel's ring for a total operand width KP = KP_a + KP_b (the formula of kmv_oracle.ring_depth)."""
    return ko.ring_depth(KP)
