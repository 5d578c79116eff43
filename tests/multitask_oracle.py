"""Layout mirrors, fp64 products and gradients, and worst-case entrywise bounds for the two multitask operators: the Hadamard
operator s K o B[t, t'] (csrc/tasks.cu) and the Kronecker operator (s K) (x) B (csrc/kron.cu).  Test infrastructure for
test_multitask_host.py and test_gpu_multitask_edges.py; it builds on tests/kmv_oracle.py (ko) and tests/bilinear_oracle.py (bo).

Layout (mirrored from the engine, not read from it).
  Hadamard  gp_plan_set_tasks sorts rows and columns by task (stable counting sort).  The columns of task b form segment b,
            padded to whole 64-column tiles on the tensor-core path (padding columns pack z = 0 with zero V rows) and unpadded
            on SIMT.  segment_split gives each segment tps_b tiles per split and nsplit_b splits (ko.split_rule over the plan's
            row units and the segment's tiles); segment b owns partial slots slot0[b] .. slot0[b + 1] - 1, nslot in all.
            task_dB_kernel reduces sorted rows in chunks of TASK_RED_ROWS, each over the tasks ts1[r0] .. ts1[r1 - 1].
  Kronecker the data plan's geometry (ko.geometry), nchunk = ceil(T t / 16) mixed column chunks of W, each one data-plan
            launch into nsplit slots at chunk offset c nsplit rows_pad 16, and the dB reduction in chunks of KRON_RED_ROWS.

Exact results are fp64 on the inputs' device, built per segment or per chunk from ko.exact / bo.closed_form (nothing (N T)^2
wide):
  Hadamard  out_i = s sum_b B[t_i, b] K[i, cols_b] V[cols_b] (+ noise_i V_i),  dB[a, b] = s sum_{i in a} L_i . (K R)_b[i]
  Kronecker out[i T + a] = s (K W)[i, a t : a t + t],  W[j, a t + c] = sum_b B[a, b] V[j T + b, c],
            dB[a, b] = s sum_i L[i T + a] . (K R_b)[i],  R_b[j] = R[j T + b]

Bounds (u = 2^-24; "ko.bound(..., nsplit, tps)" is the fused kernel's bound of kmv_oracle, which charges (nsplit + 1) u of the
abs sum A for what follows the fused kernel: nsplit fp32 slot adds and the fp32 multiply by s):
  Hadamard product.  The combine takes fmaf(B[a, task(sl)], tpart[sl][i], acc) over all nslot slots: each of the nslot
    roundings is within u of the running |sum| <= sum_b |B_ab| A_b, and the finish's multiply by s adds u more.  Segment b is a
    cross product of the sorted rows against its own columns (the diagonal masked to a = 0 on a square plan: ko.bound's diag),
    so with nsplit = nslot
        bound_i = sum_b |B[t_i, b]| ko.bound_b(s, nsplit = nslot, tps = tps_b)[i]
    (the nslot + 1 roundings, and the kernel's own tps_b tile folds or SIMT fmaf chain of segment b), plus with the noise
    u (|exact_i| + bound_i + |noise_i V_i|) for the finish's noise fmaf.
  Kronecker product.  The mix is a T-term fmaf chain: |W32 - W| <= T u Wabs, Wabs[j, a t + c] = sum_b |B_ab| |V[j T + b, c]|.
    The data plan's kernel runs on W32 into nsplit slots, which the scatter sums in fp32 (nsplit adds) before the finish
    multiplies by s once (nparts = 1), which is ko.bound's (nsplit + 1) u:
        bound = ko.bound(s, W, nsplit, tps) + T u s |K| Wabs   (+ the noise fmaf as above)
    (ko.bound on W rather than W32 and |K| rather than the engine's k leave out u x rel products, as kmv_oracle does.)
  dB (both).  task_dB_kernel / kron_dB_kernel sum a row's split slots in fp32 (nsplit_b - 1 adds; ko.bound with nsplit_b
    charges nsplit_b + 1, 2u more than needed) and take the dot with L in fp64 (products exact), so
        bound[a, b] = sum_{i in a} sum_c |L_ic| ko.bound_b(s, nsplit_b, tps_b)[i, c] + 64 2^-53 s sum |L| |K| |R|
    the last term the fp64 sums (16 products per row, <= 8 rows per thread, an 8-level tree, chunk, column-block and host sums
    and the multiply by s: fewer than 64 roundings of 2^-53).
  Hyper-parameter gradients (Hadamard).  F = sum_b sum_{i, j in b} (B[t_i, b] L_i . R_j) s k_ij, i.e. bo.closed_form per segment
    with B folded into L.
    - scalar lengthscale on tensor cores: tasks_kmv_partials with the value kind, then the derivative kind, each combined into
      one slot and dotted with L in fp64 (bilin_dot_kernel).  Per segment this is bo.bound's tensor-core path (its tile folds
      and <= 16 fp32 partials cover the segment's nsplit_b <= 16 slots), and the combine adds nslot fmaf roundings of the
      running sum:  bound = sum_b bo.bound_b(B[t, b] L, "tc") + nslot u bo.closed_form_b(|B[t, b] L|, |R|).
    - ARD, or a SIMT plan: tasks_bilinear launches bilinear_kernel per segment on Lb = fp32(B[t_i, b] L_i), one rounding of u
      more: bound = sum_b bo.bound_b(B[t, b] L, "simt") + u bo.closed_form_b(|B[t, b] L|, |R|).
    bo.bound's pairs are taken unmasked on a square plan (the engine masks the diagonal, a = 0, which bo.bound's interval
    around m = 0 contains), so on the diagonal the bound is looser than it needs to be, never tighter.
  Hyper-parameter gradients (Kronecker).  The data plan's bilinear derivative over the unmixed L chunks and the mixed R chunks:
        bound = bo.bound(Lw, W, path) + T u bo.closed_form(|Lw|, Wabs)   (Lw[i, a t + c] = L[i T + a, c])
Every bound is a worst case (every rounding at its extreme, same sign), not an estimate; none is tuned to the observed error."""
from __future__ import annotations

import torch

import bilinear_oracle as bo
import kmv_oracle as ko

U32 = bo.U32
TILE_J, TP, SIMT_TI = ko.TILE_J, ko.TP, ko.SIMT_TI
TASK_RED_ROWS = 2048        # tasks.cu: sorted rows per block of the dB reduction
KRON_RED_ROWS = 2048        # kron.cu: points per block of the dB reduction
EPS64 = 64 * 2.0 ** -53     # the fp64 sums of a dB entry (module docstring)
cdiv = ko.cdiv


# ---- layout mirrors -----------------------------------------------------------------------------------------------------------
def sort_by_task(t, T):
    """gp_plan_set_tasks' stable counting sort: (off [T + 1], perm [n]) with perm[off[b] + k] the k-th index of task b."""
    t = torch.as_tensor(t).reshape(-1).long().cpu()
    off = [0] * (T + 1)
    for v in t.tolist():
        off[v + 1] += 1
    for b in range(T):
        off[b + 1] += off[b]
    perm = torch.sort(t, stable=True).indices
    return off, perm


def segment_split(n1, cnt, tc, n_sm):
    """tasks.cu's segment_split for a segment of cnt columns on a plan of n1 rows: (tiles per split, nsplit)."""
    nti = cdiv(n1, 2 * ko.TILE_I) * 2 if tc else cdiv(n1, SIMT_TI)     # ntile_i of rows_pad, or the SIMT row blocks
    return ko.split_rule(nti, cdiv(cnt, TILE_J), n_sm, tc)


def task_layout(t1, t2, T, backend, n_sm=132):
    """Mirror of tasks_layout for task ids t1 [n1] and t2 [n2] (None: square plan).  Per task b: cnt, seg[b], tps, nsplit,
    slot0[b], the user columns `cols[b]` in segment order and the user columns of each of its slots; the layout map `map2`
    (layout column -> user column, -1 for padding), slot_task, nslot, and the sorted rows (perm1, ts1)."""
    tc = backend == "tcgen05"
    t1 = torch.as_tensor(t1).reshape(-1).long().cpu()
    t2 = t1 if t2 is None else torch.as_tensor(t2).reshape(-1).long().cpu()
    off1, perm1 = sort_by_task(t1, T)
    off2, perm2 = sort_by_task(t2, T)
    n1 = t1.numel()
    seg, tps, nsplit, slot0 = [0], [], [], [0]
    cols, slots, slot_task, map2 = [], [], [], []
    for b in range(T):
        cnt = off2[b + 1] - off2[b]
        cb = perm2[off2[b]:off2[b + 1]]
        width = cdiv(cnt, TILE_J) * TILE_J if tc else cnt
        seg.append(seg[-1] + width)
        tp, ns = segment_split(n1, cnt, tc, n_sm) if cnt > 0 else (0, 0)
        tps.append(tp)
        nsplit.append(ns)
        slot0.append(slot0[-1] + ns)
        cols.append(cb)
        for s in range(ns):
            slots.append(cb[s * tp * TILE_J:(s + 1) * tp * TILE_J])
            slot_task.append(b)
        map2 += cb.tolist() + [-1] * (width - cnt)
    return {"T": T, "tc": tc, "n1": n1, "n2": t2.numel(), "off1": off1, "perm1": perm1, "ts1": t1[perm1], "off2": off2,
            "perm2": perm2, "seg": seg, "tps": tps, "nsplit": nsplit, "slot0": slot0, "nslot": slot0[-1], "cols": cols,
            "slots": slots, "slot_task": slot_task, "map2": torch.tensor(map2, dtype=torch.long), "ncol": seg[-1]}


def dB_chunks(lay):
    """task_dB_kernel's row chunks: (z, r0, r1, a_lo, a_hi) over the sorted rows."""
    n1, ts1 = lay["n1"], lay["ts1"]
    out = []
    for z in range(cdiv(n1, TASK_RED_ROWS)):
        r0, r1 = z * TASK_RED_ROWS, min(n1, (z + 1) * TASK_RED_ROWS)
        out.append((z, r0, r1, int(ts1[r0]), int(ts1[r1 - 1])))
    return out


def kron_layout(N1, N2, d, T, t, backend, n_sm=132):
    """kron_chunks' geometry: the data plan's (ko.geometry), nchunk mixed chunks, the W chunk pitch npad, the dB chunks."""
    geo = ko.geometry(N1, N2, d, backend, n_sm)
    tc = geo["backend"] == "tcgen05"
    return dict(geo, T_tasks=T, t=t, nchunk=cdiv(T * t, TP), npad=geo["ntile_j"] * TILE_J if tc else N2,
                nred=cdiv(N1, KRON_RED_ROWS), slot_floats=geo["rows_pad"] * TP)


# ---- Hadamard: fp64 exact -----------------------------------------------------------------------------------------------------
def _cols_exact(kind, x1, xc, cols, ls, os_, V):
    """s K(x1, xc[cols]) V[cols] in fp64 [n1, t] (the rows' own points give a = 0 exactly, as the engine's mask does)."""
    dev = x1.device
    cols = cols.to(dev)
    if cols.numel() == 0:
        return torch.zeros(x1.size(0), V.size(1), dtype=torch.float64, device=dev)
    return ko.exact(kind, x1, xc[cols], ls, os_, 0.0, V.to(dev)[cols])


def hadamard_exact(kind, x1, x2, B, ls, os_, V, lay, noise_diag=None, mutant=None, mutant_arg=None):
    """fp64 (s K o B[t1, t2]) V (+ noise_diag V on a square plan) [n1, t] in user row order, slot by slot.

    `mutant` names a deliberately wrong engine (test_multitask_host.py):
      "drop_slot"   mutant_arg = slot: that partial slot left out of the combine
      "slot_task"   mutant_arg = slot: the slot weighted by B[:, task + 1] (slot_task off by one)
      "tile_late"   mutant_arg = task b: segment b read one 64-column tile late (its layout columns shifted by 64)
      "pad_v"       mutant_arg = task b: segment b's first padding column (z = 0) carrying the V row of its last column"""
    dev = x1.device
    xc = x1 if x2 is None else x2
    Bd = B.double().to(dev)
    t1 = lay["ts1"].new_empty(lay["n1"])
    t1[lay["perm1"]] = lay["ts1"]
    t1 = t1.to(dev)
    out = torch.zeros(x1.size(0), V.size(1), dtype=torch.float64, device=dev)
    for sl, (b, cols) in enumerate(zip(lay["slot_task"], lay["slots"])):
        if mutant == "drop_slot" and sl == mutant_arg:
            continue
        if mutant == "tile_late" and b == mutant_arg:
            s = sl - lay["slot0"][b]
            lo = lay["seg"][b] + TILE_J + s * lay["tps"][b] * TILE_J
            hi = min(lay["seg"][b + 1] + TILE_J, lo + lay["tps"][b] * TILE_J, lay["ncol"])
            cols = lay["map2"][lo:hi]
            cols = cols[cols >= 0]
        w = b + 1 if (mutant == "slot_task" and sl == mutant_arg) else b
        out += Bd[t1, w % lay["T"]][:, None] * _cols_exact(kind, x1, xc, cols, ls, os_, V)
    if mutant == "pad_v":
        b = mutant_arg
        mean = x1.double().mean(0, keepdim=True)
        vrow = V.to(dev)[lay["cols"][b][-1:].to(dev)]
        out += Bd[t1, b][:, None] * ko.exact(kind, x1, mean, ls, os_, 0.0, vrow)
    if noise_diag is not None:
        out += noise_diag.double().to(dev)[:, None] * V.double().to(dev)
    return out


def _diag_pos(lay, b, same, dev):
    """Per user row: its own column's position in segment b on a square plan (-1 where it is not there), else None."""
    if not same:
        return None
    pos = torch.full((lay["n1"],), -1, dtype=torch.long)
    pos[lay["cols"][b]] = torch.arange(lay["cols"][b].numel())
    return pos.to(dev)


def _task_rows(lay, dev):
    t1 = lay["ts1"].new_empty(lay["n1"])
    t1[lay["perm1"]] = lay["ts1"]
    return t1.to(dev)


def hadamard_bound(kind, x1, x2, B, ls, os_, V, lay, exact=None, noise_diag=None):
    """Worst-case |engine - hadamard_exact| [n1, t] of Plan.kmv (module docstring); `exact` is needed with noise_diag."""
    dev = x1.device
    same = x2 is None
    xc = x1 if same else x2
    path = "tc" if lay["tc"] else "simt"
    Ba = B.double().abs().to(dev)
    t1 = _task_rows(lay, dev)
    Vd = V.double().to(dev)
    out = torch.zeros(x1.size(0), V.size(1), dtype=torch.float64, device=dev)
    for b in range(lay["T"]):
        cols = lay["cols"][b].to(dev)
        if cols.numel() == 0:
            continue
        kb = ko.bound(kind, x1, xc[cols], ls, os_, 0.0, Vd[cols], path, lay["nslot"], lay["tps"][b],
                      diag=_diag_pos(lay, b, same, dev))
        out += Ba[t1, b][:, None] * kb
    if noise_diag is not None:
        nv = (noise_diag.double().to(dev)[:, None] * Vd).abs()
        out += U32 * (exact.abs() + out + nv)
    return out


def hadamard_dB(kind, x1, x2, ls, os_, L, R, lay, drop_rows=None):
    """fp64 dB [T, T] of sum L . ((s K o B) R); drop_rows (user rows) leaves those rows out (a lost reduction chunk)."""
    dev = x1.device
    xc = x1 if x2 is None else x2
    T = lay["T"]
    t1 = _task_rows(lay, dev)
    Ld = L.double().to(dev)
    if drop_rows is not None:
        Ld = Ld.clone()
        Ld[drop_rows.to(dev)] = 0.0
    out = torch.zeros(T, T, dtype=torch.float64)
    for b in range(T):
        P = _cols_exact(kind, x1, xc, lay["cols"][b], ls, os_, R)
        rowdot = (Ld * P).sum(1)
        out[:, b] = torch.zeros(T, dtype=torch.float64, device=dev).index_add_(0, t1, rowdot).cpu()
    return out


def hadamard_dB_bound(kind, x1, x2, ls, os_, L, R, lay):
    dev = x1.device
    same = x2 is None
    xc = x1 if same else x2
    path = "tc" if lay["tc"] else "simt"
    T = lay["T"]
    t1 = _task_rows(lay, dev)
    La, Ra = L.double().abs().to(dev), R.double().abs().to(dev)
    out = torch.zeros(T, T, dtype=torch.float64)
    for b in range(T):
        cols = lay["cols"][b].to(dev)
        if cols.numel() == 0:
            continue
        kb = ko.bound(kind, x1, xc[cols], ls, os_, 0.0, Ra[cols], path, lay["nsplit"][b], lay["tps"][b],
                      diag=_diag_pos(lay, b, same, dev))
        kb = kb + EPS64 * ko.exact(kind, x1, xc[cols], ls, os_, 0.0, Ra[cols])
        out[:, b] = torch.zeros(T, dtype=torch.float64, device=dev).index_add_(0, t1, (La * kb).sum(1)).cpu()
    return out


def hadamard_grad(kind, x1, x2, B, ls, os_, L, R, lay):
    """fp64 (dF/dl [1 or d], dF/ds) of F = sum L . ((s K o B) R), segment by segment with B folded into L."""
    dev = x1.device
    xc = x1 if x2 is None else x2
    Bd = B.double().to(dev)
    t1 = _task_rows(lay, dev)
    Ld, Rd = L.double().to(dev), R.double().to(dev)
    gl, gs = 0.0, 0.0
    for b in range(lay["T"]):
        cols = lay["cols"][b].to(dev)
        if cols.numel() == 0:
            continue
        a, s = bo.closed_form(kind, x1, xc[cols], ls, os_, Ld * Bd[t1, b][:, None], Rd[cols])
        gl, gs = gl + a, gs + s
    return gl, gs


def hadamard_grad_bound(kind, x1, x2, B, ls, os_, L, R, lay, path, n_sm=132):
    """Bound on |engine - hadamard_grad| for path "tc" (scalar lengthscale, tensor-core plan) or "simt" (ARD or a SIMT plan)."""
    dev = x1.device
    xc = x1 if x2 is None else x2
    Bd = B.double().to(dev)
    t1 = _task_rows(lay, dev)
    Ld, Rd = L.double().to(dev), R.double().to(dev)
    extra = lay["nslot"] * U32 if path == "tc" else U32
    gl, gs = 0.0, 0.0
    for b in range(lay["T"]):
        cols = lay["cols"][b].to(dev)
        if cols.numel() == 0:
            continue
        Lb = Ld * Bd[t1, b][:, None]
        a, s = bo.bound(kind, x1, xc[cols], ls, os_, Lb, Rd[cols], path, n_sm=n_sm)
        aa, sa = bo.closed_form(kind, x1, xc[cols], ls, os_, Lb.abs(), Rd[cols].abs())
        gl, gs = gl + a + extra * aa, gs + s + extra * sa
    return gl, gs


# ---- Kronecker ----------------------------------------------------------------------------------------------------------------
def kron_mix(B, V, T, t):
    """W [N2, T t] (fp64) and Wabs of V [N2 T, t]: W[j, a t + c] = sum_b B[a, b] V[j T + b, c]."""
    Vr = V.double().reshape(-1, T, t)
    Bd = B.double().to(Vr.device)
    W = torch.einsum("ab,jbc->jac", Bd, Vr).reshape(Vr.size(0), T * t)
    Wabs = torch.einsum("ab,jbc->jac", Bd.abs(), Vr.abs()).reshape(Vr.size(0), T * t)
    return W, Wabs


def _unmix(V, T, t):
    """[N T, t] -> [N, T t]: row j, column a t + c = V[j T + a, c] (kron_mix_kernel with B = nullptr)."""
    return V.double().reshape(-1, T * t)


def _split_cols(geo, n2, sp):
    lo = sp * geo["T"] * TILE_J
    return torch.arange(lo, min(n2, lo + geo["T"] * TILE_J))


def kron_exact(kind, x1, x2, B, ls, os_, V, T, t, noise=0.0, geo=None, mutant=None, mutant_arg=None):
    """fp64 ((s K) (x) B) V (+ noise V on a square plan) [N1 T, t].

      "scatter_chunk"  mutant_arg = (q, sp): kron_scatter_kernel reads split slot sp of chunk q from the neighbouring chunk
                       (q + 1, or q - 1 for the last chunk) (needs geo)
      "mix_drop"       mutant_arg = (a, b): kron_mix_kernel leaves out the term B[a, b] V[j T + b] of row a"""
    dev = x1.device
    same = x2 is None
    xc = x1 if same else x2
    Vd = V.double().to(dev)
    W, _ = kron_mix(B, Vd, T, t)
    if mutant == "mix_drop":
        a, b = mutant_arg
        W = W.clone()
        W[:, a * t:(a + 1) * t] -= float(B[a, b]) * Vd.reshape(-1, T, t)[:, b, :]
    out = ko.exact(kind, x1, x2, ls, os_, 0.0, W, same=same)
    if mutant == "scatter_chunk":
        q, sp = mutant_arg
        nchunk = cdiv(T * t, TP)
        q2 = q + 1 if q + 1 < nchunk else q - 1
        Wp = torch.zeros(W.size(0), nchunk * TP, dtype=torch.float64, device=dev)
        Wp[:, :T * t] = W
        cols = _split_cols(geo, xc.size(0), sp).to(dev)
        Kc = lambda c: ko.exact(kind, x1, xc[cols], ls, os_, 0.0, Wp[cols, c * TP:(c + 1) * TP])
        fix = Kc(q2) - Kc(q)
        hi = min(T * t, (q + 1) * TP)
        out[:, q * TP:hi] += fix[:, :hi - q * TP]
    out = out.reshape(-1, t)
    if same and noise:
        out += float(bo.f32(noise)) * Vd
    return out


def kron_bound(kind, x1, x2, B, ls, os_, V, T, t, geo, exact=None, noise=0.0):
    dev = x1.device
    same = x2 is None
    Vd = V.double().to(dev)
    W, Wabs = kron_mix(B, Vd, T, t)
    path = "tc" if geo["backend"] == "tcgen05" else "simt"
    out = ko.bound(kind, x1, x2, ls, os_, 0.0, W, path, geo["nsplit"], geo["T"], same=same)
    out = out + T * U32 * ko.exact(kind, x1, x2, ls, os_, 0.0, Wabs, same=same)
    out = out.reshape(-1, t)
    if same and noise:
        out += U32 * (exact.abs() + out + float(bo.f32(noise)) * Vd.abs())
    return out


def kron_dB(kind, x1, x2, ls, os_, L, R, T, t):
    """fp64 dB [T, T] of sum L . (((s K) (x) B) R), L [N1 T, t], R [N2 T, t]."""
    dev = x1.device
    P = ko.exact(kind, x1, x2, ls, os_, 0.0, _unmix(R.to(dev), T, t), same=x2 is None).reshape(-1, T, t)
    Lr = L.double().to(dev).reshape(-1, T, t)
    return torch.einsum("iac,ibc->ab", Lr, P).cpu()


def kron_dB_bound(kind, x1, x2, ls, os_, L, R, T, t, geo):
    dev = x1.device
    same = x2 is None
    path = "tc" if geo["backend"] == "tcgen05" else "simt"
    Ra = _unmix(R.to(dev), T, t).abs()
    kb = ko.bound(kind, x1, x2, ls, os_, 0.0, Ra, path, geo["nsplit"], geo["T"], same=same)
    kb = kb + EPS64 * ko.exact(kind, x1, x2, ls, os_, 0.0, Ra, same=same)
    La = L.double().to(dev).abs().reshape(-1, T, t)
    return torch.einsum("iac,ibc->ab", La, kb.reshape(-1, T, t)).cpu()


def kron_grad(kind, x1, x2, B, ls, os_, L, R, T, t):
    """fp64 (dF/dl, dF/ds) of F = sum L . (((s K) (x) B) R)."""
    dev = x1.device
    W, _ = kron_mix(B, R.to(dev), T, t)
    return bo.closed_form(kind, x1, x1 if x2 is None else x2, ls, os_, _unmix(L.to(dev), T, t), W, same=x2 is None)


def kron_grad_bound(kind, x1, x2, B, ls, os_, L, R, T, t, path, n_sm=132):
    dev = x1.device
    W, Wabs = kron_mix(B, R.to(dev), T, t)
    Lw = _unmix(L.to(dev), T, t)
    xc = x1 if x2 is None else x2
    a, s = bo.bound(kind, x1, xc, ls, os_, Lw, W, path, same=x2 is None, n_sm=n_sm)
    aa, sa = bo.closed_form(kind, x1, xc, ls, os_, Lw.abs(), Wabs, same=x2 is None)
    return a + T * U32 * aa, s + T * U32 * sa


# ---- the cases of test_gpu_multitask_edges.py (test_multitask_host.py checks each still reaches its edge on 132 and 114 SMs) --
# Hadamard products: T = 7 tasks, square n = 3000 (user order shuffled) with segments of 1 (one padded tile), 63, 64, 897 and
# 1025 columns (2 splits: 8 + 7 and 9 + 8 tiles) and an empty task; the cross plan's rows over the same tasks, where task 2 has
# rows and no columns and task 3 columns and no rows
PROD_COLS = [897, 1, 0, 63, 1025, 64, 950]
PROD_ROWS = [300, 200, 400, 0, 500, 1, 599]
# dB reductions (sorted task sizes, chunks of 2048 rows)
RED_CASES = {
    "n2048": [700, 1000, 0, 348, 0],                 # one chunk, ending on the edge; empty tasks
    "n2049": [1024, 1025, 0],                        # task 1 straddles 2048 with one row in chunk 1
    "n4200_starts": [1000, 1048, 1100, 948, 0, 104], # tasks starting exactly at 2048 and at 4096
    "n4200_straddle": [1500, 1000, 0, 1200, 400, 100],   # tasks straddling 2048 and 4096
    "T32": {3: 1000, 9: 1048, 17: 2048, 30: 104},    # 32 tasks: chunk 1 holds task 17 alone, task 30 starts at 4096
}
KRON_SPLIT = ko.SPLIT_SQUARE                          # N = 1450, d = 5: 3 splits of 8, 8, 7 tiles
KRON_TT = [(4, 4), (3, 6), (7, 7), (32, 1), (1, 16)]  # 1, 2, 4, 2, 1 chunks
KRON_RED = [(2048, 1000), (2049, 1000), (4100, 1000)]  # cross N1, N2 (2 splits of 8 tiles): 1, 2, 3 dB chunks


def sizes_list(sizes):
    """Task sizes as a list of T counts (RED_CASES' T = 32 case is given as {task: count})."""
    if isinstance(sizes, dict):
        return [sizes.get(b, 0) for b in range(32)]
    return list(sizes)


def task_ids(sizes, seed=None):
    """Task ids with the given per-task counts, shuffled by seed (None: sorted)."""
    t = torch.cat([torch.full((c,), b, dtype=torch.long) for b, c in enumerate(sizes_list(sizes))])
    if seed is None:
        return t
    return t[torch.randperm(t.numel(), generator=torch.Generator().manual_seed(seed))]


def hadamard_case(name, seed, d=4, t=16):
    """Inputs of a GPU case: (x1, x2 or None, t1, t2 or None, T, V [n2, t]), task ids shuffled by seed.  name: "square" or
    "cross" (PROD_*), or a key of RED_CASES (square)."""
    if name in ("square", "cross"):
        T = len(PROD_COLS)
        t2 = task_ids(PROD_COLS, seed)
        t1 = task_ids(PROD_ROWS, seed + 1) if name == "cross" else t2
    else:
        sizes = sizes_list(RED_CASES[name])
        T = len(sizes)
        t1 = t2 = task_ids(sizes, seed)
    x1 = ko.points(t1.numel(), d, seed)
    x2 = ko.points(t2.numel(), d, seed + 2) if name == "cross" else None
    V = torch.randn(t2.numel(), t, generator=torch.Generator().manual_seed(seed + 3))
    return x1, x2, t1, (t2 if name == "cross" else None), T, V


def random_B(T, seed, rank=2):
    """fp32-representable IndexKernel covariance F F^T + diag(v)."""
    g = torch.Generator().manual_seed(seed)
    F = torch.randn(T, rank, generator=g, dtype=torch.float64)
    return (F @ F.t() + torch.diag(0.1 + torch.rand(T, generator=g, dtype=torch.float64))).float()
