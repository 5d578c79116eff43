"""fp64 K.V of the fused kernel-matmul (csrc/kmv_tc.cu on the tensor cores, csrc/kmv_simt.cu on CUDA cores, both finished by
kmv_finish_user_kernel), a worst-case bound on |engine - fp64| for every output entry, and a mirror of the launch geometry
(pack.cu: round_dp, KP, choose_geometry; kmv_tc.cu: tc_smem_bytes).  Test infrastructure for test_kmv_host.py and
test_gpu_kmv.py.

    out[i, c] = s sum_j k(x1_i, x2_j) V[j, c]  (+ noise V[row_begin + i, c] on a square plan with the noise added)

The hyper-parameters are held as fp32 values (the engine's gp_plan_set_hypers), the diagonal of a square plan is m = 0 at the
global row, and everything runs in row blocks on the tensors' own device, so the large cases evaluate on a GPU in fp64.

The bound reuses the per-pair model of tests/bilinear_oracle.py (bo.pair_arg, bo._dev, bo.pair_rel): packing 2u|z|; the
argument a by direct differences (SIMT) or through the 3xTF32 GEMM, (1 + KP/4) 2^-21 (|z_i|^2 + |z_j|^2); k over that interval
of a; the MUFU error.  Per entry, with k_ij the fp64 value, rel_ij, dk_ij that model and u = 2^-24:
    kabs_ij  = k_ij (1 + rel_ij) + dk_ij                    bounds the engine's value of the pair
    pair     = sum_j |V_jc| (k_ij rel_ij + dk_ij)           the pairs' own errors
             + 2^-19 sum_j kabs_ij |V_jc|                   tensor cores: GEMM2's P_hi / P_lo and V_hi / V_lo split (as in bo.bound)
    A        = sum_j kabs_ij |V_jc|                         the abs sum every rounding of the sums is measured against
    sums     tensor cores, per 64-column tile: 8 k-steps per wgmma chain, each adding 8 exact tf32 products to the accumulator;
             aligned to the largest addend and truncated, every addend is off by < 2u of that addend, so < 8 (8 + 1) 2u = 144u
             per chain of its abs sum (the V_lo and P_lo chains carry 2^-11 and 2^-10 of it), + 2u for the two adds of the fold
             (o1 + o1' + o2), + T u for the T fp32 tile folds of a split
             SIMT: min(cps, n2) fmaf terms per thread (cps = 64 T columns per split), u each
             then nsplit fp32 partial adds and the fp32 multiply by s (kmv_finish_user_kernel): (nsplit + 1) u
    bound    = s (pair + eps_sums A)  (+ u (s A + noise |V_ic|) for the noise fmaf)
The sums are first order in u; the products u x rel they leave out are below 1e-12 of A and inside kabs >= |engine k|."""
from __future__ import annotations

import math

import torch

import bilinear_oracle as bo

U32 = bo.U32
TILE_I, TILE_J, TP = 128, 64, 16
KP_MAX, MAX_NS = 128, 12
SIMT_TI = 128
V_TF32_BYTES = 2 * TILE_J * TP * 4          # kmv_tc.cu: the tf32 half of a packed V tile
TC_BARS_BYTES = 8 + 2 * MAX_NS * 8          # sizeof(TcBars)
TC_CHAIN = 8 * (8 + 1) * 2 * U32            # one GEMM2 wgmma chain of a 64-column tile (see above)


def cdiv(a, b):
    return -(-a // b)


# ---- launch geometry ----------------------------------------------------------------------------------------------------------
def ring_depth(KP):
    """NS of kmv_tc.cu's tc_smem_bytes: stages of (B tile + tf32 V tile) that fit 226 KB beside the A tile and the barriers."""
    a_bytes = KP * TILE_I * 4
    stage = KP * TILE_J * 4 + V_TF32_BYTES
    return min(MAX_NS, (226 * 1024 - a_bytes - TC_BARS_BYTES) // stage)


def split_rule(nti, ntj, n_sm, tc):
    """(tiles per split, nsplit) of choose_geometry (pack.cu) and segment_split (tasks.cu) for nti row units and ntj column
    tiles: the fewest splits of at least 8 tiles that best fill 2 (tensor cores) or 1 (SIMT) CTAs per SM."""
    slots = n_sm * (2 if tc else 1)
    best, best_eff = 1, -1.0
    for s in range(1, 17):
        if s > ntj:
            break
        per = cdiv(ntj, s)
        if s > 1 and per < 8:
            break
        waves = cdiv(nti * s, slots)
        eff = float(nti * ntj) / float(waves * slots * per)
        if eff > best_eff + 0.02:
            best_eff, best = eff, s
    tps = cdiv(ntj, best)
    return tps, cdiv(ntj, tps)


def geometry(n1, n2, d, backend="auto", n_sm=132, row_count=None):
    """pack.cu's choose_geometry for a plan over row_count (default n1) rows and n2 columns: the backend, DP, KP, the ring depth
    NS (tensor cores), nsplit, the tiles per split T, the tiles of the last split and the columns per SIMT split."""
    rows = row_count or n1
    DP, KP = bo.dp_of(d), bo.kp_of(d)
    if backend == "auto":
        backend = "tcgen05" if KP <= KP_MAX else "simt"
    tc = backend == "tcgen05"
    rows_pad = cdiv(rows, 2 * TILE_I) * 2 * TILE_I
    ntile_i, ntile_j = rows_pad // TILE_I, cdiv(n2, TILE_J)
    nti = ntile_i if tc else cdiv(rows, SIMT_TI)
    ntj = ntile_j                                   # SIMT_TJ == TILE_J
    tps, nsplit = split_rule(nti, ntj, n_sm, tc)
    return {"backend": backend, "DP": DP, "KP": KP, "NS": ring_depth(KP) if tc else None, "rows_pad": rows_pad,
            "ntile_i": ntile_i, "ntile_j": ntile_j, "nsplit": nsplit, "T": tps, "T_last": ntj - (nsplit - 1) * tps,
            "cps": tps * TILE_J}


# ---- fp64 product -------------------------------------------------------------------------------------------------------------
def _packed(kind, x1, x2, lengthscale, same, row_begin, row_count):
    """fp64 packed rows and columns (pack.cu: z = (x - mean(x1)) sqrt(C) / l) and the global row index of each local row."""
    n_loc = row_count or (x1.size(0) - row_begin)
    d = x1.size(1)
    ls = bo._ls(lengthscale, d).to(x1.device)
    sc = math.sqrt(bo._C[kind]) / ls
    mean = x1.double().mean(0)
    zr = (x1.double()[row_begin:row_begin + n_loc] - mean) * sc
    zc = ((x1 if same else x2).double() - mean) * sc
    return zr, zc, torch.arange(row_begin, row_begin + n_loc, device=x1.device)


def _block_rows(n2, d, cap=1024):
    return max(8, min(cap, (1 << 24) // max(1, n2 * d)))


def _tf32_trunc(t):
    """The top 19 bits of fp32(t) (kmv_tc.cu's P_hi)."""
    return (t.float().view(torch.int32) & -8192).view(torch.float32).double()


def _tf32_round(t):
    """gp_common.cuh's tf32_hi: fp32(t) rounded to 10 mantissa bits, ties away; a NaN keeps its bits."""
    f = t.float()
    r = ((f.view(torch.int32) + 0x1000) & -8192).view(torch.float32)
    return torch.where(torch.isnan(f), f, r).double()


def _n_lo(kind, x1, xs, lengthscale):
    """The n_lo operand pack_tc_kernel gives each row of xs: n = -|z|^2 / 2 of the fp32 packed z, minus its tf32 part."""
    d = x1.size(1)
    ls32 = torch.as_tensor(lengthscale, dtype=torch.float32).reshape(-1).expand(d).to(x1.device)
    sc32 = (math.sqrt(bo._C[kind]) / ls32.double()).float()
    mean32 = x1.double().mean(0).float()
    z = ((xs.float() - mean32) * sc32).double()
    nn = -0.5 * (z * z).sum(1)
    return nn - _tf32_round(nn)


def _ordered_cols(n2):
    """Column of K each of the first n2 positions pairs with V in when pack.cu's 0 4 1 5 2 6 3 7 order of an 8-column group is
    not applied: position t + 4e then carries column 2t + e of its group (columns past n2 are padding, k = 1)."""
    q = torch.arange(cdiv(n2, 8) * 8)
    return (q // 8) * 8 + 2 * (q % 4) + (q % 8) // 4


def exact(kind, x1, x2, lengthscale, outputscale, noise, V, same=False, row_begin=0, row_count=None, block=None,
          mutant=None, mutant_arg=None):
    """fp64 s K V (+ noise V on the local rows of a square plan) [row_count, t] on V's device, V [n2, t].

    `mutant` names a deliberately wrong engine the bound is tested against (test_kmv_host.py):
      "p_lo"         GEMM2 without P_lo: k truncated to tf32
      "v_lo"         GEMM2 without V_lo: V rounded to tf32
      "order"        XB's 0 4 1 5 2 6 3 7 column order undone: K's columns permuted within every 8-column group
      "tile"         mutant_arg = (row_tile or None, column tile, factor): that tile's columns counted `factor` times (0: a
                     skipped tile, 2: one counted twice), in one 128-row tile or in all of them
      "diag_shift"   the diagonal mask one column to the right: m = 0 at (i, i + 1)
      "diag_local"   the diagonal mask at local rows on a shard: m = 0 at (i - row_begin, i)
      "diag_da"      mutant_arg = first column: diagonal pairs from that column on left unmasked, with the tensor-core error
                     (1 + KP/4) 2^-21 2|z_i|^2 of a = 0 as their m (bilinear_oracle's unmasked-diagonal variant)
      "noise_cross"  the noise added on a cross plan (rows i < n2)
      "noise_twice"  the noise added twice
      "os_twice"     the outputscale applied to every partial and again to their sum
      "n_lo"         GEMM1 without n_lo: m_ij + n_lo_i + n_lo_j"""
    zr, zc, grow = _packed(kind, x1, x2, lengthscale, same, row_begin, row_count)
    dev = zr.device
    n2, d = zc.size(0), zc.size(1)
    Vd = V.double().to(dev)
    os_ = float(bo.f32(outputscale))
    if mutant == "os_twice":
        os_ = os_ * os_
    if mutant == "v_lo":
        Vd = _tf32_round(Vd)
    xs_rows = x1[row_begin:row_begin + zr.size(0)]
    if mutant == "n_lo":
        nlo_r = _n_lo(kind, x1, xs_rows, lengthscale).to(dev)
        nlo_c = _n_lo(kind, x1, x1 if same else x2, lengthscale).to(dev)
    perm = _ordered_cols(n2).to(dev) if mutant == "order" else None
    out = torch.empty(zr.size(0), Vd.size(1), dtype=torch.float64, device=dev)
    block = block or _block_rows(n2, d)
    for b in bo._blocks(zr.size(0), block):
        m = 0.5 * sum((zr[b, c, None] - zc[None, :, c]) ** 2 for c in range(d))
        rows = torch.arange(b.stop - b.start, device=dev)
        g = grow[b]
        if mutant == "n_lo":
            m = m + nlo_r[b, None] + nlo_c[None, :]
            if kind != "rbf":
                m = m.clamp_min(0)   # the Matern path takes fmaxf(-a, 0); RBF's ex2 takes a as it comes
        if same:
            diag_col = {"diag_shift": g + 1, "diag_local": g - row_begin}.get(mutant, g)
            ok = diag_col < n2
            if mutant == "diag_da" and mutant_arg is not None:
                kp = bo.kp_of(d)
                da = (1 + kp / 4) * 2.0 ** -21 * 2 * (zr[b] * zr[b]).sum(1)
                late = ok & (diag_col >= mutant_arg)
                m[rows[ok & ~late], diag_col[ok & ~late]] = 0.0
                m[rows[late], diag_col[late]] = da[late]
            else:
                m[rows[ok], diag_col[ok]] = 0.0
        k, _ = bo._kg(kind, m)
        if mutant == "p_lo":
            k = _tf32_trunc(k)
        if perm is not None:
            kp_ = torch.ones(k.size(0), perm.numel(), dtype=k.dtype, device=dev)
            kp_[:, :n2] = k
            k = kp_[:, perm[:n2]]
        if mutant == "tile":
            rt, jt, factor = mutant_arg
            sel = slice(None) if rt is None else ((g - row_begin) // TILE_I == rt)
            k[sel, jt * TILE_J:(jt + 1) * TILE_J] *= factor
        out[b] = os_ * (k @ Vd)
    nz = float(bo.f32(noise)) if noise else 0.0
    if mutant == "noise_twice":
        nz *= 2
    if same and nz:
        out += nz * Vd[grow]
    if mutant == "noise_cross" and not same:
        nz = float(bo.f32(mutant_arg))
        r = grow < n2
        out[r] += nz * Vd[grow[r]]
    return out


# ---- the bound ----------------------------------------------------------------------------------------------------------------
def bound(kind, x1, x2, lengthscale, outputscale, noise, V, path, nsplit, T_per_split, same=False, row_begin=0, row_count=None,
          block=None, diag=None):
    """Worst-case |engine - exact| [row_count, t] for every entry of Plan.kmv on the same fp32 inputs (module docstring).
    path "tc" (kmv_tc_kernel) or "simt" (kmv_simt_kernel); nsplit and T_per_split from geometry() (a kernel sum passes the
    number of partial slots of all its terms as nsplit).  diag [rows] (cross form only): the column of x2 that is each row's own
    point, masked to a = 0 by the kernel as on a square plan (-1: none), for columns that are a subset of the rows (one task
    segment of a Hadamard plan, tests/multitask_oracle.py)."""
    zr, zc, grow = _packed(kind, x1, x2, lengthscale, same, row_begin, row_count)
    dev = zr.device
    n2, d = zc.size(0), zc.size(1)
    DP, KP = bo.dp_of(d), bo.kp_of(d)
    Va = V.double().to(dev).abs()
    os_ = float(bo.f32(outputscale))
    if path == "tc":
        eps = TC_CHAIN * (1 + 2.0 ** -11 + 2.0 ** -10) + 2 * U32 + T_per_split * U32
    else:
        eps = min(T_per_split * TILE_J, n2) * U32
    eps += (nsplit + 1) * U32
    nr = (zc * zc).sum(1)
    out = torch.empty(zr.size(0), Va.size(1), dtype=torch.float64, device=dev)
    block = block or _block_rows(n2, d, 256)
    for b in bo._blocks(zr.size(0), block):
        _, _, _, _, m, da = bo.pair_arg(zr[b], zc, nr, path, DP, KP)
        if same or diag is not None:   # exact diagonal: a = 0 on both paths
            rows = torch.arange(b.stop - b.start, device=dev)
            g = grow[b] if diag is None else diag[b].to(dev)
            ok = (g >= 0) & (g < n2)
            m[rows[ok], g[ok]] = 0.0
            da[rows[ok], g[ok]] = 0.0
        k, _ = bo._kg(kind, m)
        dk, _ = bo._dev(kind, m, da)
        rel = bo.pair_rel(m)
        kabs = k * (1 + rel) + dk
        pair = k * rel + dk
        if path == "tc":
            pair = pair + 2.0 ** -19 * kabs
        A = kabs @ Va
        out[b] = os_ * (pair @ Va + eps * A)
        if same and noise:
            out[b] += U32 * (os_ * A + float(bo.f32(noise)) * Va[grow[b]])
    return out


# ---- the cases of test_gpu_kmv.py (fixed inputs; test_kmv_host.py checks that each still reaches its edge on 132 and 114 SMs) --
KP_D = {8: 1, 16: 3, 24: 5, 32: 8, 40: 12, 64: 20, 96: 30, 128: 41}   # operand width KP -> the d that gives it
SIMT_D = [4, 7, 12, 15, 24, 31, 48, 63, 96, 128]                      # one d per SIMT DP instantiation (4 ... 128)
RING_KP = (8, 40, 64, 128)
N1_EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257]
N2_EDGES = [1, 63, 64, 65]
T_EDGES = [1, 15, 16, 17, 33]
SHARD_N = 1500
SHARDS = [(0, SHARD_N), (1, 130), (63, 65), (64, 64), (65, 200), (129, 300), (400, 300)]
SPLIT_SQUARE = (1450, 5)         # square n, d: three splits of 8, 8 and 7 tiles
LARGE_ROWS = 58368               # 456 row tiles: 1 split whether 132 or 114 SMs
CPS_EDGE = (1000, 3585, 4)       # SIMT cross plan n1, n2, d: the last split holds one column (n2 = 7 cps + 1)


def ring_T(NS):
    return [1, 2, NS - 1, NS, NS + 1, 2 * NS, 2 * NS + 1]


def ring_cases():
    """(d, T, n1, n2): tensor-core cross plans with one split of T column tiles, at the ring depth's edges."""
    out = []
    for kp in RING_KP:
        for T in ring_T(ring_depth(kp)):
            out.append((KP_D[kp], T, 200, TILE_J * T - (5 if T % 2 else 0)))
    return out


def large_row_cases():
    """(d, T, n1, n2): cross plans of 456 row tiles (several waves of CTAs) with one long split."""
    return [(KP_D[8], 2 * ring_depth(8) + 1, LARGE_ROWS, TILE_J * 25 - 5), (KP_D[40], 2 * ring_depth(40) + 1, LARGE_ROWS, TILE_J * 23),
            (KP_D[128], 2 * ring_depth(128) + 1, LARGE_ROWS, TILE_J * 9 - 1)]


def points(n, d, seed):
    return torch.rand(n, d, generator=torch.Generator().manual_seed(seed))


def spread_points(n, d, kind, seed, z2):
    """n points in d dimensions whose packed |z|^2 reaches about z2 at lengthscale 1: 1-D uniform over the span, else clusters of
    50 points (spread 0.5) around centres uniform over the span, so every point still has neighbours within a lengthscale."""
    g = torch.Generator().manual_seed(seed)
    half = math.sqrt(z2 / (bo._C[kind] * d))     # |x - mean| per dimension at the edge of the span
    if d == 1:
        return (torch.rand(n, 1, generator=g) * 2 - 1) * half
    centres = (torch.rand(cdiv(n, 50), d, generator=g) * 2 - 1) * half
    return centres.repeat_interleave(50, 0)[:n] + 0.5 * torch.randn(n, d, generator=g)


def identity_cols(n2, picks):
    """V = the identity's columns `picks` (clipped to [0, n2), duplicates dropped, at most 16): each output entry is one kernel
    value."""
    cols = sorted({c for c in picks if 0 <= c < n2})[:16]
    V = torch.zeros(n2, len(cols))
    V[cols, torch.arange(len(cols))] = 1.0
    return V, cols
