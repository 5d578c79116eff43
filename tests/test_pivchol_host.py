"""The pivoted-Cholesky checker (tests/pivchol_oracle.py) on the CPU: it accepts the fp64 oracle's factor rounded to fp32 and
rejects each planted fault -- a non-greedy pivot order, one entry off by 8 times its bound, a lost 384-row grid-stride segment,
the later-position duplicate at a tie, and a rank off by one."""
import numpy as np
import pytest
import torch

import pivchol_oracle as po
from oracle import kernels as ok, linalg as ol

N, D, LS = 1000, 3, 0.45
STOP_LS, STOP_TOL = 1.2, 0.1


def _problem(dup=False, ls=LS):
    g = torch.Generator().manual_seed(4)
    if dup:   # every point 3 times (one 4 times) at scattered indices; K indexed from the distinct points: bit-identical duplicate rows
        x = torch.rand(N // 3, D, generator=g, dtype=torch.float64)
        idx = torch.randperm(N, generator=g) % (N // 3)
        K = ok.kernel_matrix("rbf", x, x, ls, 1.0, True)[idx][:, idx].contiguous()
    else:
        x = torch.rand(N, D, generator=g, dtype=torch.float64)
        K = ok.kernel_matrix("rbf", x, x, ls, 1.0, True)
    diag = torch.ones(N, dtype=torch.float64)
    eps = po.generic_entry_bound(1.0, D, float(D) / (2 * ls * ls))
    return K, diag, eps


def _factor(K, rank, order=None):
    """fp64 partial Cholesky L [m, n], greedy with ties to the earliest position of the running permutation (the device's rule;
    torch.max in the oracle sees fp64 sums whose order depends on the column), or in a given pivot order.  Every row is
    updated by the same elementwise operations, so duplicate rows stay bit-identical."""
    n = K.size(0)
    L = torch.zeros(rank, n, dtype=torch.float64)
    res = K.diagonal().clone()
    perm, pos = list(range(n)), list(range(n))
    done = torch.zeros(n, dtype=torch.bool)
    piv = []
    for k in range(rank):
        if order is None:
            r = res.masked_fill(done, -float("inf"))
            top = torch.nonzero(r == r.max()).flatten().tolist()
            pi = min(top, key=lambda j: pos[j])
        else:
            pi = order[k]
        a, b = k, pos[pi]
        perm[a], perm[b] = perm[b], perm[a]
        pos[perm[a]], pos[perm[b]] = a, b
        acc = torch.zeros(n, dtype=torch.float64)
        for q in range(k):
            acc += L[q] * L[q, pi]
        dpiv = res[pi].sqrt()
        v = (K[:, pi] - acc) / dpiv
        v[done] = 0.0
        v[pi] = dpiv
        L[k] = v
        res = res - v * v
        done[pi] = True
        piv.append(pi)
    return L, torch.tensor(piv)


def _check(K, diag, eps, Lt, piv, tol, rank, status=0):
    return po.check_factor(Lt.float(), piv, Lt.size(0), status, diag, lambda i: K[:, i], tol, eps, rank)


def test_accepts_the_fp64_oracle_rounded_to_fp32():
    K, diag, eps = _problem()
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 60, 1e-3)
    assert L.size(1) == 60
    _check(K, diag, eps, L.t(), piv, 1e-3, 60)
    # a tolerance that stops the factor early, far enough from every step's err for the fp32 uncertainty to decide it
    K, diag, eps = _problem(ls=STOP_LS)
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 200, STOP_TOL)
    assert L.size(1) < 200
    assert _check(K, diag, eps, L.t(), piv, STOP_TOL, 200)["stop_checked"]


def test_accepts_ties_and_sees_position_order():
    K, diag, eps = _problem(dup=True)
    L, piv = _factor(K, 60)
    out = _check(K, diag, eps, L, piv, 0.0, 60)
    assert out["ties"] >= 50 and out["ties_by_position"] >= 1


def test_rejects_a_non_greedy_pivot():
    K, diag, eps = _problem()
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 30, 0.0)
    gaps = po.pivot_gaps(diag, L, piv)
    m = next(k for k in range(5, 29) if gaps[k] > 1e-3)   # a step with a clear gap
    order = piv.tolist()
    order[m], order[m + 1] = order[m + 1], order[m]
    _check(K, diag, eps, *_factor(K, 30, piv.tolist()), 0.0, 30)        # the forced replay itself passes
    with pytest.raises(AssertionError, match="pivot"):
        _check(K, diag, eps, *_factor(K, 30, order), 0.0, 30)


def test_rejects_one_entry_off_by_eight_bounds():
    K, diag, eps = _problem()
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 30, 0.0)
    Lt = L.t().float().clone()
    m, pl = 17, piv.tolist()
    j = next(j for j in range(N) if j not in pl)
    Ld = Lt.double()
    bound = eps + po.gamma(m + 2) * float((Ld[: m + 1, j].abs() * Ld[: m + 1, pl[m]].abs()).sum())
    Lt[m, j] += 8 * bound / float(Lt[m, pl[m]])
    with pytest.raises(AssertionError, match="backward identity"):
        _check(K, diag, eps, Lt, piv, 0.0, 30)


def test_rejects_a_lost_grid_stride_segment():
    K, diag, eps = _problem()
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 30, 0.0)
    Lt = L.t().float().clone()
    keep = Lt[20, piv[:21]].clone()
    Lt[20, 384:768] = 0.0          # the second 384-row segment of step 20, its pivot entries left in place
    Lt[20, piv[:21]] = keep
    with pytest.raises(AssertionError, match="backward identity"):
        _check(K, diag, eps, Lt, piv, 0.0, 30)


def test_rejects_the_later_position_duplicate_at_a_tie():
    K, diag, eps = _problem(dup=True)
    L, piv = _factor(K, 40)
    _check(K, diag, eps, L, piv, 0.0, 40)
    order = piv.tolist()
    for m in range(1, 40):
        dups = [j for j in range(N) if j not in order[:m] and torch.equal(L[:m, j], L[:m, order[m]])]
        if len(dups) > 1:
            break
    else:
        pytest.fail("no tie among duplicates")
    order[m] = next(j for j in dups if j != order[m])
    with pytest.raises(AssertionError, match="tie"):
        _check(K, diag, eps, *_factor(K, 40, order), 0.0, 40)


@pytest.mark.parametrize("off", [-1, 1])
def test_rejects_a_rank_off_by_one(off):
    K, diag, eps = _problem(ls=STOP_LS)
    tol = STOP_TOL
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 200, tol)
    r = L.size(1)
    assert r < 200 and _check(K, diag, eps, L.t(), piv, tol, 200)["stop_checked"]
    if off < 0:
        Lt, pv = L.t()[: r - 1], piv[: r - 1]
    else:
        L2, p2 = ol.pivoted_cholesky(diag, lambda i: K[i], r + 1, 0.0)
        Lt, pv = L2.t(), p2
    with pytest.raises(AssertionError, match="err"):
        _check(K, diag, eps, Lt, pv, tol, 200)


def test_pivot_gaps_of_a_constant_diagonal():
    K, diag, _ = _problem()
    L, piv = ol.pivoted_cholesky(diag, lambda i: K[i], 10, 0.0)
    gaps = po.pivot_gaps(diag, L, piv)
    assert gaps[0] == 0.0 and min(gaps[1:]) > 0.0
    assert np.isfinite(gaps).all()
