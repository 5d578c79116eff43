"""fp64 products, gradients and entrywise bounds of the masked Kronecker operator P_r ((s K) (x) B) P_c^T
(gp_plan_set_kron_observed, csrc/kron.cu), built on tests/multitask_oracle.py (mo) with zero-filled operands.

rows / cols are the observed interleaved rows i T + a (int64, strictly increasing; None: all of them).  E_c [N2 T, n_c] puts the
n_c observed columns at their interleaved rows and zeros elsewhere, E_r likewise for the rows, and
    P_r ((s K) (x) B) P_c^T V = E_r^T (((s K) (x) B) (E_c V)),
so the masked product is the unmasked product of the zero-filled V = E_c V, restricted to the observed output rows.

Why the unmasked bounds carry over unchanged.  The masked mix reads V16[colpos[j T + b]] where the column is observed and the
literal 0.f where it is not, so it runs the same T-term fmaf chain over the same values as the unmasked mix over E_c V (an
fmaf(B_ab, 0, s) returns s exactly); the data plan's kernel then sees the same W, and the masked scatter sums the same split
slots of row rowmap[r] that the unmasked scatter sums for that row.  Every rounding the bound of mo.kron_bound charges for row
i T + a is therefore the rounding the engine makes for observed row r with rowmap[r] = i T + a, and
    mask_bound = E_r^T mo.kron_bound(E_c V).
The gradients run the unmasked passes on L = E_r L_obs and R = E_c R_obs (masked_kron_expand_kernel writes exact zeros and copies),
and the missing rows contribute exact zeros to every fp32 and fp64 sum, so
    mask_dB_bound = mo.kron_dB_bound(E_r L, E_c R),   mask_grad_bound = mo.kron_grad_bound(E_r L, E_c R).
Rows and the diagonal are gathers of the unmasked rows and diagonal (no arithmetic), exact as those are.

Mutants (each must leave the bound somewhere on a case with enough structure): "mix_neighbour" (the mix reads the next observed
row), "scatter_shift" (observed row r is written from rowmap[r + 1]), "rowmap_task" (the row map is off by one task) and, for dB,
"drop_expand" (the expand pass loses observed row k)."""
from __future__ import annotations

import torch

import kron_oracle as ko
import multitask_oracle as mo


def expand(V, idx, nfull):
    """E V: [nfull, t] with the rows of V at idx and zeros elsewhere (idx None: V itself)."""
    if idx is None:
        return V.double()
    out = torch.zeros(nfull, V.size(-1), dtype=torch.float64, device=V.device)
    out[idx.to(V.device)] = V.double()
    return out


def _take(out, idx):
    return out if idx is None else out[idx.to(out.device)]


def _sizes(x1, x2, T):
    return x1.size(0) * T, (x1 if x2 is None else x2).size(0) * T


def mask_matrix(kind, x1, x2, ls, os_, B, rows, cols):
    """Dense fp64 P_r ((s K) (x) B) P_c^T (small sizes only)."""
    A = ko.kron_matrix(kind, x1.double(), (x1 if x2 is None else x2).double(), ls, os_, B.double(), x2 is None)
    A = A if rows is None else A[rows]
    return A if cols is None else A[:, cols]


def mask_exact(kind, x1, x2, B, ls, os_, V, T, t, rows, cols, noise=0.0, mutant=None):
    """fp64 P_r ((s K) (x) B) P_c^T V (+ noise V on a square plan) [n_r, t]."""
    n1f, n2f = _sizes(x1, x2, T)
    Vobs = V.double()
    if mutant == "mix_neighbour":            # observed column k reads observed row k + 1 (the last one its own)
        Vobs = torch.cat([Vobs[1:], Vobs[-1:]])
    Vf = expand(Vobs, cols, n2f)
    out = mo.kron_exact(kind, x1, x2, B, ls, os_, Vf, T, t)
    r = rows if rows is not None else torch.arange(n1f)
    if mutant == "scatter_shift":
        r = torch.cat([r[1:], r[-1:]])
    elif mutant == "rowmap_task":
        r = torch.where(r % T == T - 1, r - 1, r + 1) if T > 1 else torch.where(r + T < n1f, r + T, r - T)
    out = out[r.to(out.device)]
    if x2 is None and noise:
        out = out + float(torch.tensor(noise, dtype=torch.float32)) * V.double().to(out.device)
    return out


def mask_bound(kind, x1, x2, B, ls, os_, V, T, t, rows, cols, geo, exact=None, noise=0.0):
    n1f, n2f = _sizes(x1, x2, T)
    Vf = expand(V, cols, n2f)
    out = _take(mo.kron_bound(kind, x1, x2, B, ls, os_, Vf, T, t, geo), rows)
    if x2 is None and noise:
        out = out + mo.U32 * (exact.abs() + out + float(torch.tensor(noise, dtype=torch.float32)) * V.double().abs().to(out.device))
    return out


def mask_dB(kind, x1, x2, ls, os_, L, R, T, t, rows, cols, mutant=None, mutant_arg=0):
    n1f, n2f = _sizes(x1, x2, T)
    Lf = expand(L, rows, n1f)
    if mutant == "drop_expand":
        Lf[(rows[mutant_arg] if rows is not None else mutant_arg)] = 0.0
    return mo.kron_dB(kind, x1, x2, ls, os_, Lf, expand(R, cols, n2f), T, t)


def mask_dB_bound(kind, x1, x2, ls, os_, L, R, T, t, rows, cols, geo):
    n1f, n2f = _sizes(x1, x2, T)
    return mo.kron_dB_bound(kind, x1, x2, ls, os_, expand(L, rows, n1f), expand(R, cols, n2f), T, t, geo)


def mask_grad(kind, x1, x2, B, ls, os_, L, R, T, t, rows, cols):
    n1f, n2f = _sizes(x1, x2, T)
    return mo.kron_grad(kind, x1, x2, B, ls, os_, expand(L, rows, n1f), expand(R, cols, n2f), T, t)


def mask_grad_bound(kind, x1, x2, B, ls, os_, L, R, T, t, rows, cols, path, n_sm=132):
    n1f, n2f = _sizes(x1, x2, T)
    return mo.kron_grad_bound(kind, x1, x2, B, ls, os_, expand(L, rows, n1f), expand(R, cols, n2f), T, t, path, n_sm)


def pattern(name, n, T, seed):
    """Observed interleaved rows (int64, increasing) of an n-point, T-task data set for a named missing pattern."""
    N = n * T
    g = torch.Generator().manual_seed(seed)
    keep = torch.ones(N, dtype=torch.bool)
    if name == "one":
        keep[N // 2] = False
    elif name.startswith("frac"):                  # frac10 / frac50 / frac90: that percentage missing
        keep = torch.rand(N, generator=g) >= int(name[4:]) / 100
    elif name == "point":
        keep[(n // 3) * T:(n // 3 + 1) * T] = False
    elif name == "task":
        keep[torch.arange(N) % T == T - 1] = False
    elif name == "straddle":                       # a run of missing rows either side of the 64-row tile edge, one observed inside
        keep[40:90] = False
        keep[64] = True
    if not bool(keep.any()):
        keep[0] = True
    return keep.nonzero().reshape(-1)
