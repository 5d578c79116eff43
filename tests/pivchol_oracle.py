"""fp64 checker of a device pivoted-Cholesky factor (gp_pivoted_cholesky, csrc/pivchol.cu).

check_factor(Lt, piv, rank_out, status, diag, col, tol, eps_k, rank) takes the device factor as it comes back (Lt [m, n] fp32, the
pivots, the rank and the status), the fp64 initial diagonal the device pivots on, col(i) -> K[:, i] in fp64 and the fp32 entry
bound eps_k of the operator, and raises AssertionError with the first property that fails.  u = 2^-24, g(k) = k u / (1 - k u).

* structure: distinct pivots; L[m][pi_q] == 0 exactly for q < m; L[m][pi_m] > 0; every entry finite when the status is 0.
* backward identity on the pivot columns: for every row j
      |K[j, pi_m] - sum_{q<=m} L_q[j] L_q[pi_m]| <= eps_K + g(m + 2) sum_{q<=m} |L_q[j]| |L_q[pi_m]|
  (the dot product, the subtraction and the division of step m); for the pivot's own diagonal g(2m + 2) (K_jj + sum L_q[pi_m]^2),
  the running diag -= v v and the square root.
* greedy choice: with the fp64 residuals r_m(j) = K_jj - sum_{q<m} L_q[j]^2 of the device's own L and
  d_m(j) = g(2m + 1) (K_jj + sum_{q<m} L_q[j]^2), r_m(pi_m) >= max_j r_m(j) - d_m(pi_m) - max_j d_m(j).
* ties: rows whose device residual is bit-identical to the pivot's (same initial diagonal, same L columns so far) are decided by
  the earliest position in the running permutation, which the checker replays from the swaps; after swaps that can be a later
  index.  The number of steps where position and index order disagree is returned, so that a test can assert it met one.
* stop rule: rank_out is the first m + 1 at which err = sum |r_{m+1}| / max(diag) <= tol (or the requested rank, or n), checked
  at the steps where |err - tol| lies outside the fp32 uncertainty sum d / max(diag).
"""
from __future__ import annotations

import math

import numpy as np
import torch

U32 = 2.0 ** -24
GP_W_PIVCHOL_NAN = 5


def gamma(k: int) -> float:
    return k * U32 / (1.0 - k * U32)


def generic_entry_bound(kmax: float, dp: int, amax: float) -> float:
    """fp32 bound of a kernel entry s k(a) where no oracle derives one: |K| (DP + 4) u (1 + |a|)."""
    return kmax * (dp + 4) * U32 * (1.0 + amax)


def pivot_gaps(diag, L, piv):
    """Per step of an fp64 factor L [n, m]: the winning residual diagonal minus the best of the other unpivoted candidates."""
    res = diag.clone()
    done = torch.zeros(diag.numel(), dtype=torch.bool)
    gaps = []
    for m, pm in enumerate(piv.tolist()):
        top2 = torch.topk(res.masked_fill(done, -math.inf), 2).values
        gaps.append(float(top2[0] - top2[1]))
        done[pm] = True
        res = res - L[:, m] ** 2
    return gaps


def _eps_col(eps_k, i, n):
    e = eps_k(i) if callable(eps_k) else eps_k
    return np.broadcast_to(np.asarray(e, dtype=np.float64), (n,))


def check_factor(Lt, piv, rank_out, status, diag, col, tol, eps_k, rank=None, chunk=1 << 16):
    """Raise AssertionError unless (Lt, piv, rank_out, status) is a valid fp32 greedy pivoted Cholesky of K (module docstring).

    Lt [m, n] and piv [m] (any device), diag [n] fp64 initial diagonal, col(i) -> K[:, i] fp64 [n], eps_k a scalar or
    eps_k(i) -> [n] bound of the device's fp32 entries of column i, rank the requested rank (None: rank_out).
    Returns {"ties": steps with a tie of bit-identical residuals, "ties_by_position": such steps where the earliest position is
    not the lowest index, "stop_checked": whether the stop rule was decidable at every step}."""
    L32 = Lt.detach().cpu().contiguous().numpy()
    assert L32.dtype == np.float32
    p = piv.detach().cpu().numpy().astype(np.int64)
    m_out, n = L32.shape
    d = diag.detach().cpu().double().numpy()
    assert d.shape == (n,)
    assert m_out == rank_out == p.size, f"Lt has {m_out} rows, {p.size} pivots, rank_out {rank_out}"
    max_rank = min(rank if rank is not None else rank_out, n)
    assert 1 <= rank_out <= max_rank, f"rank_out {rank_out} outside [1, {max_rank}]"
    # ---- structure ----
    assert len(set(p.tolist())) == p.size, "pivots repeat"
    assert ((p >= 0) & (p < n)).all(), "pivot out of range"
    if status == 0:
        assert np.isfinite(L32).all(), "status 0 with a non-finite entry"
    for m in range(m_out):
        assert (L32[m, p[:m]] == 0.0).all(), f"step {m}: an earlier pivot's entry is not zero"
        assert L32[m, p[m]] > 0.0, f"step {m}: pivot entry {L32[m, p[m]]} not positive"
    # ---- backward identity on the pivot columns (row chunks: the factor may be large) ----
    Lp = L32[:, p].astype(np.float64)                     # [m, m]: L_q[pi_m], zero for q > m
    Kp = np.stack([np.asarray(col(int(i)), dtype=np.float64) for i in p])   # [m, n]: K[:, pi_m]
    E = np.stack([_eps_col(eps_k, int(i), n) for i in p]) if callable(eps_k) else None
    gm = np.array([gamma(m + 2) for m in range(m_out)])
    for j0 in range(0, n, chunk):
        Lc = L32[:, j0:j0 + chunk].astype(np.float64)
        R = Lc.T @ Lp                                     # [c, m]: sum_{q<=m} L_q[j] L_q[pi_m]
        A = np.abs(Lc).T @ np.abs(Lp)
        e = E[:, j0:j0 + chunk].T if E is not None else float(eps_k)
        bound = e + A * gm
        js = np.arange(j0, j0 + Lc.shape[1])
        own = (js[:, None] == p[None, :])                 # the pivot's own diagonal
        if own.any():
            r, c = np.nonzero(own)
            dgb = np.array([gamma(2 * int(m) + 2) for m in c]) * (d[js[r]] + A[r, c])
            bound[r, c] = (e[r, c] if E is not None else float(eps_k)) + dgb
        err = np.abs(Kp[:, j0:j0 + chunk].T - R)
        bad = ~(err <= bound)
        if bad.any():
            r, c = np.argwhere(bad)[0]
            raise AssertionError(f"backward identity: row {js[r]}, pivot column {c} (index {p[c]}): |K - LL^T| = {err[r, c]:.3e} "
                                 f"> bound {bound[r, c]:.3e}")
    # ---- greedy choice, ties, stop rule: replay the steps on the device's own L ----
    res = d.copy()
    s2 = np.zeros(n)
    done = np.zeros(n, dtype=bool)
    perm = np.arange(n)
    pos = np.arange(n)
    key = np.zeros(n, dtype=np.uint64)                    # running hash of (diag, L columns so far): bit-identical residuals
    key ^= d.astype(np.float32).view(np.uint32).astype(np.uint64)
    mul = np.uint64(0x9E3779B97F4A7C15)
    orig = float(d.max())
    ties = ties_pos = 0
    stop_checked = True
    for m in range(m_out):
        pm = int(p[m])
        delta = gamma(2 * m + 1) * (d + s2)
        cand = ~done
        rmax = float(res[cand].max())
        dmax = float(delta[cand].max())
        assert res[pm] >= rmax - delta[pm] - dmax, (f"step {m}: pivot {pm} has residual {res[pm]:.9g}, the best candidate "
                                                    f"{rmax:.9g} (margin {delta[pm] + dmax:.3g})")
        # ties: the rows whose residual the device computed bit-identically to the pivot's
        same = np.nonzero(cand & (key == key[pm]))[0]
        if same.size > 1:
            hist = L32[:m, same]
            same = same[(hist == L32[:m, pm:pm + 1]).all(0) & (d[same].astype(np.float32) == np.float32(d[pm]))]
        if same.size > 1:
            ties += 1
            first = int(same[np.argmin(pos[same])])
            assert first == pm, f"step {m}: tie between rows {same.tolist()} goes to position {pos[first]} (row {first}), not row {pm}"
            ties_pos += int(first != int(same.min()))
        # swap of step m in the running permutation
        a, b = m, int(pos[pm])
        ra, rb = int(perm[a]), int(perm[b])
        perm[a], perm[b] = rb, ra
        pos[rb], pos[ra] = a, b
        done[pm] = True
        Lm = L32[m].astype(np.float64)
        res -= Lm * Lm
        s2 += Lm * Lm
        key = (key * mul) ^ L32[m].view(np.uint32).astype(np.uint64)
        # stop rule after step m
        if status != 0:
            continue
        rest = ~done
        err = float(np.abs(res[rest]).sum()) / orig if rest.any() else 0.0
        unc = float((gamma(2 * m + 3) * (d + s2))[rest].sum()) / orig + 4 * U32 * err
        exhausted = rest.any() and float((res - gamma(2 * m + 3) * (d + s2))[rest].max()) <= 0.0   # no residual surely > 0
        if abs(err - tol) <= unc:
            stop_checked = False
            continue
        last = m == m_out - 1
        if not last:
            assert err > tol, f"step {m}: err {err:.6g} <= tol {tol:.6g} but the factor goes on to rank {m_out}"
        elif m_out < max_rank:
            assert err <= tol or exhausted, f"stopped at rank {m_out} < {max_rank} with err {err:.6g} > tol {tol:.6g}"
    return {"ties": ties, "ties_by_position": ties_pos, "stop_checked": stop_checked}
