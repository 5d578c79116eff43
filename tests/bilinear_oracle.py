"""fp64 closed form of the hyper-parameter gradient and the fp32 error bound of the engine's gp_bilinear_grad (test
infrastructure; imported by test_bilinear_host.py and test_gpu_bilinear.py).

F = sum_ij w_ij s k(x1_i, x2_j), w = L R^T formed in fp64 (lazy_evaluated_kernel_tensor.py:69-105):
    dF/ds   = sum w k
    dF/dl   = (s / l) sum w g,                      g = l dk/dl  (scalar lengthscale)
    dF/dl_c = (s / l_c) sum w g delta_c^2 / r^2     (ARD; delta_c = (x1_ic - x2_jc) / l_c, r^2 = sum_c delta_c^2)
In the engine's packed units (pack.cu: z = (x - mean) sqrt(C) / l, m = -a = |z_i - z_j|^2 / 2):
    RBF         k = 2^-m                 g = 2 ln2 m k
    Matern-1/2  k = e                    g = rho e                  (rho = sqrt(m), e = exp(-rho))
    Matern-3/2  k = (1 + rho) e          g = m e
    Matern-5/2  k = (1 + rho + m/3) e    g = (1 + rho) m e / 3
Evaluated in row blocks on the tensors' own device (float64), so the n = 50 000 case runs on a GPU.
"""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -24
LN2 = math.log(2.0)
_C = {"rbf": 1.0 / LN2, "matern12": 2.0, "matern32": 6.0, "matern52": 10.0}   # pack.cu: z = (x - mean) sqrt(C) / l
KINDS = tuple(_C)


def f32(v):
    """The engine holds hyper-parameters as fp32 (gp_plan_set_hypers): the oracle uses the same values."""
    return torch.as_tensor(v, dtype=torch.float32).double().reshape(-1)


def dp_of(d):
    return next(o for o in (4, 8, 12, 16, 24, 32, 48, 64, 96, 128) if d <= o)


def kp_of(d):
    return (3 * d + 4 + 7) // 8 * 8


def _ls(lengthscale, d):
    ls = f32(lengthscale)
    return ls.expand(d) if ls.numel() == 1 else ls


def _blocks(n, size):
    for i0 in range(0, n, size):
        yield slice(i0, min(n, i0 + size))


def _kg(kind, m):
    """k and g = l dk/dl at m = -a >= 0 (packed units)."""
    if kind == "rbf":
        k = torch.exp2(-m)
        return k, 2 * LN2 * m * k
    rho = m.sqrt()
    e = torch.exp(-rho)
    if kind == "matern12":
        return e, rho * e
    if kind == "matern32":
        return (1 + rho) * e, m * e
    return (1 + rho + m / 3) * e, (1 + rho) * m * e / 3


def _dev(kind, m, da):
    """Largest |k(m') - k(m)|, |g(m') - g(m)| over |m' - m| <= da: |f'| <= Q(hi) decay(lo) on the interval, with Q the
    polynomial of |f| + |f'| (non-negative coefficients, so increasing).  For Matern the interval is taken in rho, where
    sqrt(m + da) - sqrt(m - da) carries the sqrt amplification near m = 0 (Matern-1/2's g = rho e has slope 1 there)."""
    if kind == "rbf":
        lo, hi = m - da, m + da
        dec = torch.exp2(-lo)
        return LN2 * dec * da, 2 * LN2 * (1 + LN2 * hi) * dec * da
    rho = m.sqrt()
    rlo, rhi = (m - da).clamp_min(0).sqrt(), (m + da).sqrt()
    drho = torch.maximum(rhi - rho, rho - rlo) + 2.0 ** -22 * rho          # + sqrt.approx
    r = rhi + drho
    dec = torch.exp(-(rlo - drho).clamp_min(0)) * drho
    qk, qg = {"matern12": (1.0, r + 1), "matern32": (2 + r, r * r + 2 * r),
              "matern52": (2 + 5 * r / 3 + r * r / 3, (r ** 3 + 4 * r * r + 2 * r) / 3)}[kind]
    return qk * dec, qg * dec


def _geometry(x1, x2, L, R, same, row_begin):
    """Local rows of the plan (x1 rows [row_begin, +L rows) of a square plan) and the columns."""
    n_loc = L.size(0)
    xr = x1[row_begin:row_begin + n_loc] if same else x1
    xc = x1 if same else x2
    return xr.double(), xc.double()


def closed_form(kind, x1, x2, lengthscale, outputscale, L, R, same=False, row_begin=0, block=256,
                diag_offset=None, diag_m=None, ard_no_r2=False, ard_shift=0):
    """(dF/dl [1 or d] float64, dF/ds float) for the plan K(x1, x2) (same: K(x1, x1), local rows from row_begin).

    The keyword arguments after `block` make the deliberately wrong variants the bound is tested against: `diag_offset` forces
    m = 0 at the local pairs (i, i + diag_offset); `diag_m` [rows] puts those m on the pairs (i, i + row_begin) instead of
    0; `ard_no_r2` drops the 1 / r^2 of the ARD factor; `ard_shift` rolls the ARD columns."""
    xr, xc = _geometry(x1, x2, L, R, same, row_begin)
    d = xr.size(1)
    ard = f32(lengthscale).numel() > 1
    ls = _ls(lengthscale, d).to(xr.device)
    os_ = float(f32(outputscale))
    sc = math.sqrt(_C[kind]) / ls
    L, R = L.double(), R.double()
    gk = torch.zeros((), dtype=torch.float64, device=xr.device)
    gl = torch.zeros(d if ard else 1, dtype=torch.float64, device=xr.device)
    for b in _blocks(xr.size(0), block):
        w = L[b] @ R.t()
        sq = [((xr[b, c, None] - xc[None, :, c]) * sc[c]) ** 2 for c in range(d)]
        S = sum(sq)
        m = 0.5 * S
        rows = torch.arange(b.start, b.stop, device=xr.device)
        for off, val in ((diag_offset, None), (row_begin if diag_m is not None else None, diag_m)):
            if off is None:
                continue
            cols = rows + off
            ok = (cols >= 0) & (cols < xc.size(0))
            m[(rows - b.start)[ok], cols[ok]] = 0.0 if val is None else val.to(m)[rows[ok]]
        k, g = _kg(kind, m)
        gk += (w * k).sum()
        if not ard:
            gl += (w * g).sum()
            continue
        wg = w * g if ard_no_r2 else torch.where(S > 0, w * g / S, torch.zeros_like(S))
        for c in range(d):
            gl[c] += (wg * sq[(c + ard_shift) % d]).sum()
    return (os_ / ls[: gl.numel()] * gl).cpu(), float(gk)


def simt_cps(rows, n2, n_sm):
    """Columns one thread of bilinear_kernel accumulates in fp32 (gp_bilinear_grad's split of the columns)."""
    cdiv = lambda a, b: -(-a // b)
    ntj = cdiv(n2, 64)
    nsp = min(ntj, max(1, (2 * n_sm) // max(1, cdiv(rows, 128))))
    return min(cdiv(ntj, nsp) * 64, n2)


def pair_arg(zr, zc, nr, path, DP, KP):
    """The per-pair part of the bound below for packed rows zr [r, d] against packed columns zc [c, d] (nr = |zc|^2 per column):
    (dz, Ec, sq, S, m, da) with dz_c = z_ic - z_jc, Ec the packing error of dz_c, sq = dz^2, S = sum sq, m = S / 2 and da the
    bound on the engine's error in a = -m on `path` ("simt": direct differences, "tc": the 3xTF32 GEMM).  Shared with the K.V
    bound of tests/kmv_oracle.py."""
    d = zr.size(1)
    dz = [zr[:, c, None] - zc[None, :, c] for c in range(d)]
    Ec = [2 * U32 * (zr[:, c, None].abs() + zc[None, :, c].abs()) for c in range(d)]
    sq = [v * v for v in dz]
    S = sum(sq)
    E2 = sum(e * e for e in Ec)
    m = 0.5 * S
    da = E2.sqrt() * S.sqrt() + 0.5 * E2
    if path == "simt":
        da = da + (DP + 4) * U32 * m
    else:
        da = da + (1 + KP / 4) * 2.0 ** -21 * ((zr * zr).sum(1)[:, None] + nr[None, :]) + 4 * U32 * m
    return dz, Ec, sq, S, m, da


def pair_rel(m, eps_sum=0.0):
    """eps_sum plus the relative error of one covariance value at m beyond the interval of a (_dev): ex2.approx 2^-21 of the
    value, sqrt.approx, the fp32 product log2(e) rho and the Matern polynomial."""
    return eps_sum + 2.0 ** -21 + 2 * U32 * (1 + m.sqrt()) + 6 * U32


def bound(kind, x1, x2, lengthscale, outputscale, L, R, path, same=False, row_begin=0, n_sm=132, block=256):
    """(bound on |engine - closed_form| for dF/dl [1 or d], same for dF/ds) of gp_bilinear_grad on the same fp32 inputs.
    path: "simt" (bilinear_kernel; every ARD plan) or "tc" (scalar lengthscale on the tensor-core backend).

    With Wabs_ij = sum_c |L_ic| |R_jc| (it dominates |w_ij| and the error of every form of w), u = 2^-24, per pair:
      z      fp32 packing (x - mean) * scale: |dz| <= 2 u |z| per entry, so the difference z_i - z_j is off by
             E = 2 u (|z_i| + |z_j|) and m by  ||E|| ||z_i - z_j|| + ||E||^2 / 2
      a      SIMT: direct differences, (DP + 4) u m  (DP fp32 adds, the fp32 scale, the -0.5)
             tensor cores: the 3xTF32 GEMM drops lo*lo (2^-22 |z_ic||z_jc|), rounds lo to tf32 (2 x 2^-22 |z_ic||z_jc|) and
             n_lo (2^-22 |n|, n = |z|^2 / 2): at most 2^-21 (|z_i|^2 + |z_j|^2); fp32 accumulation over KP products whose
             partial sums stay below |z_i|^2 + |z_j|^2, each add within 2u: KP 2^-23 (|z_i|^2 + |z_j|^2).  Together
             (1 + KP / 4) 2^-21 (|z_i|^2 + |z_j|^2), plus 4 u m.  The diagonal of a square plan is exact (m = 0) on both.
      k, g   |f(m') - f(m)| over |m' - m| <= da (_dev), plus ex2.approx 2^-22 / sqrt.approx 2^-22 / the fp32 product
             log2(e) rho and the polynomial: 2^-21 + 2 u (1 + rho) + 6 u relative
      w      SIMT: a 16-term fp32 dot per column chunk, 16 u of Wabs.  Tensor cores: GEMM2 takes P = P_hi + P_lo with
             P_hi P's top tf32 bits and V = V_hi + V_lo; P_lo V_hi drops P_lo V_lo (2^-21), P_lo is truncated to tf32 by
             the tensor core (2^-20), V_lo rounded (2^-22): 2^-19 of |P| |V|
      sums   SIMT: one thread sums min(cps, n2) terms in fp32 (cps from gp_bilinear_grad's split), then double reductions:
             cps u.  Tensor cores: 8 k-steps per 64-column tile in the tensor core, ntile_j tile folds, <= 16 partials in
             fp32: 2 u (16 + ntile_j + 16); the final dot with L is double.
      ARD    (SIMT) t_c = delta_c^2 / S, S = sum_c delta_c^2: the fp32 delta_c^2 is off by D_c = 2 |delta_c| E_c + E_c^2
             + 3 u delta_c^2 and S by dS = sum D_c + DP u S, so t_c by min(1, (D_c + t_c dS) / (S - dS)).
    It is a worst-case bound (every rounding at its extreme, same sign), not an estimate."""
    xr, xc = _geometry(x1, x2, L, R, same, row_begin)
    n2, d = xc.size(0), xr.size(1)
    ard = f32(lengthscale).numel() > 1
    assert not (ard and path == "tc"), "ARD gradients run on the SIMT kernel"
    DP, KP = dp_of(d), kp_of(d)
    ls = _ls(lengthscale, d).to(xr.device)
    os_ = float(f32(outputscale))
    sc = math.sqrt(_C[kind]) / ls
    mean = x1.double().mean(0)
    zr, zc = (xr - mean) * sc, (xc - mean) * sc
    Labs, Rabs = L.double().abs(), R.double().abs()
    if path == "simt":
        eps_sum = simt_cps(L.size(0), n2, n_sm) * U32 + 16 * U32 + 2 * U32
    else:
        eps_sum = 2 * U32 * (32 + -(-n2 // 64)) + 2.0 ** -19
    bk = torch.zeros((), dtype=torch.float64, device=xr.device)
    bg = torch.zeros(d if ard else 1, dtype=torch.float64, device=xr.device)
    nr = (zc * zc).sum(1)
    for b in _blocks(xr.size(0), block):
        Wabs = Labs[b] @ Rabs.t()
        dz, Ec, sq, S, m, da = pair_arg(zr[b], zc, nr, path, DP, KP)
        if same:   # exact diagonal: a = 0 on both paths
            rows = torch.arange(b.start, b.stop, device=xr.device)
            cols = rows + row_begin
            m[rows - b.start, cols] = 0.0
            da[rows - b.start, cols] = 0.0
        k, g = _kg(kind, m)
        dk, dg = _dev(kind, m, da)
        rel = pair_rel(m, eps_sum)
        bk += (Wabs * (k * rel + dk)).sum()
        eg = g * rel + dg
        if not ard:
            bg += (Wabs * eg).sum()
            continue
        D = [2 * v.abs() * e + e * e + 3 * U32 * s2 for v, e, s2 in zip(dz, Ec, sq)]
        dS = sum(D) + DP * U32 * S
        den = S - dS
        for c in range(d):
            t = torch.where(S > 0, sq[c] / S, torch.zeros_like(S))
            dt = torch.where(den > 0, ((D[c] + t * dS) / den.clamp_min(1e-300)).clamp_max(1.0), torch.ones_like(S))
            bg[c] += (Wabs * ((eg + 3 * U32 * g) * (t + dt).clamp_max(1.0) + g * dt)).sum()
    return (os_ / ls[: bg.numel()] * bg).cpu(), float(bk)
