"""The Hadamard (tasks.cu) and Kronecker (kron.cu) multitask operators entry by entry against the fp64 results of
tests/multitask_oracle.py, within its derived worst-case bounds, at the sizes where their layout code changes shape: task
segments of several column splits with a shorter last split, one-column, empty and row-only / column-only tasks, dB reductions
over several 2048-row chunks with tasks straddling or starting on a chunk edge, Kronecker data plans of three splits with
1 to 4 mixed column chunks, single kernel values through identity columns (the diagonal bit for bit), determinism and NaN
propagation.  Every case asserts its backend (and the Kronecker data plan's nsplit) against the mirrors, which
test_multitask_host.py checks still reach their edges."""
import math
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu

import bilinear_oracle as bo  # noqa: E402
import kmv_oracle as ko  # noqa: E402
import multitask_oracle as mo  # noqa: E402

KINDS = list(bo.KINDS)
BACKENDS = ["tcgen05", "simt"]
PATH = {"tcgen05": "tc", "simt": "simt"}
LS, OS = 0.5, 1.3
RATIOS = {}   # (operator, path, kind) -> largest |engine - fp64| / bound seen
CANONICAL_NAN = torch.tensor([0x7FFFFFFF], dtype=torch.int32).view(torch.float32)[0]


def _within(key, tag, got, ref, bnd):
    got, ref, bnd = (torch.as_tensor(v, dtype=torch.float64).to(ref.device if torch.is_tensor(ref) else "cpu")
                     for v in (got, ref, bnd))
    err = (got - ref).abs()
    frac = torch.where(bnd > 0, err / bnd, torch.where(err > 0, torch.inf, 0.0))
    worst = int(frac.argmax())
    assert bool(torch.isfinite(got).all()) and float(frac.max()) <= 1.0, \
        (tag, key, worst, float(err.reshape(-1)[worst]), float(bnd.reshape(-1)[worst]), float(got.reshape(-1)[worst]),
         float(ref.reshape(-1)[worst]))
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(frac.max()))


def _hadamard(dev, kind, x1, x2, t1, t2, T, B, backend, ls=LS):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend).set_hypers(kind, ls, OS, 0.0)
    p.set_tasks(t1.to(dev), None if t2 is None else t2.to(dev), T)
    p.set_task_covar(B)
    assert p.info()["backend"] == backend
    return p, mo.task_layout(t1, t2, T, backend, p.info()["n_sm"])


def _kron(dev, kind, x1, x2, T, B, backend, noise=0.0, ls=LS):
    from gpytorch_b200.engine import KronPlan, Plan

    data = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend).set_hypers(kind, ls, OS, 0.0)
    n2 = (x1 if x2 is None else x2).size(0)
    geo = ko.geometry(x1.size(0), n2, x1.size(1), backend, data.info()["n_sm"])
    assert (data.info()["backend"], data.info()["nsplit"]) == (geo["backend"], geo["nsplit"]), (data.info(), geo)
    p = KronPlan(data, T)
    p.set_noise(noise)
    p.set_task_covar(B)
    assert p.info()["backend"] == "kron"
    return p, geo


# ---- Hadamard products --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name", ["square", "cross"])
def test_hadamard_products_within_bound(cuda_dev, backend, name):
    """T = 7 over 3000 columns: segments of 897 and 1025 columns in two splits, of 1, 63 and 64 columns, an empty task; the
    cross plan has a task with rows and no columns and one with columns and no rows.  The square plan adds a per-task noise
    diagonal.  Repeated products are bit-identical."""
    x1, x2, t1, t2, T, V = mo.hadamard_case(name, 11)
    B = mo.random_B(T, 12)
    nd = None if x2 is not None else (0.05 + 0.05 * torch.arange(T, dtype=torch.float32))[t1]
    x1d, x2d, Vd = x1.to(cuda_dev), None if x2 is None else x2.to(cuda_dev), V.to(cuda_dev)
    for k, kind in enumerate(KINDS):
        p, lay = _hadamard(cuda_dev, kind, x1, x2, t1, t2, T, B, backend)
        if nd is not None:
            p.set_noise_diag(nd.to(cuda_dev))
        out = p.kmv(Vd, add_noise=nd is not None)
        ref = mo.hadamard_exact(kind, x1d, x2d, B, LS, OS, Vd, lay, noise_diag=nd)
        bnd = mo.hadamard_bound(kind, x1d, x2d, B, LS, OS, Vd, lay, exact=ref, noise_diag=nd)
        _within(("hadamard", PATH[backend], kind), name, out, ref, bnd)
        assert torch.equal(out, p.kmv(Vd, add_noise=nd is not None))


@pytest.mark.parametrize("backend", BACKENDS)
def test_hadamard_identity_columns_and_exact_diagonal(cuda_dev, backend):
    """V = identity columns at segment starts and ends and at split starts and ends: each output entry is one s k B value.  On
    the diagonal it is fp32(fp32(s) B[t, t]) bit for bit: the masked a = 0 gives k = 1 exactly, every other slot holds an exact
    0, so the combine's fmaf chain yields B[t, t] and the finish rounds its product with s once."""
    x1, _, t1, _, T, _ = mo.hadamard_case("square", 11)
    B = mo.random_B(T, 12)
    lay = mo.task_layout(t1, None, T, backend)
    picks = []
    for b in range(T):
        c = lay["cols"][b].tolist()
        picks += c[:1] + c[-1:]
        if b in (0, 4):   # the two-split segments of 897 and 1025 columns
            edge = lay["tps"][b] * ko.TILE_J
            picks += [c[edge - 1], c[edge]]
    Vi, cols = ko.identity_cols(x1.size(0), picks)
    assert len(cols) == 15 and all(lay["nsplit"][b] == 2 for b in (0, 4))
    os32 = torch.tensor(float(bo.f32(OS)), dtype=torch.float32)
    x1d, Vd = x1.to(cuda_dev), Vi.to(cuda_dev)
    for kind in KINDS:
        p, lay = _hadamard(cuda_dev, kind, x1, None, t1, None, T, B, backend)
        out = p.kmv(Vd)
        ref = mo.hadamard_exact(kind, x1d, None, B, LS, OS, Vd, lay)
        _within(("hadamard", PATH[backend], kind), "identity", out, ref, mo.hadamard_bound(kind, x1d, None, B, LS, OS, Vd, lay))
        for c, j in enumerate(cols):
            a = int(t1[j])
            assert out[j, c].item() == (os32 * B[a, a]).item(), (kind, j, a, out[j, c].item())


# ---- Hadamard reductions ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name", list(mo.RED_CASES))
def test_hadamard_dB_at_chunk_edges_within_bound(cuda_dev, backend, name):
    """n1 in {2048, 2049, 4200}: tasks straddling rows 2048 and 4096, starting exactly on them, a chunk of one task (T = 32),
    segments of two splits.  Repeated calls are bit-identical."""
    kind = KINDS[list(mo.RED_CASES).index(name) % 4]
    x1, _, t1, _, T, _ = mo.hadamard_case(name, 21, t=5)
    B = mo.random_B(T, 22)
    g = torch.Generator().manual_seed(23)
    L, R = torch.randn(x1.size(0), 5, generator=g), torch.randn(x1.size(0), 5, generator=g)
    p, lay = _hadamard(cuda_dev, kind, x1, None, t1, None, T, B, backend)
    assert max(lay["nsplit"]) >= 2
    x1d, Ld, Rd = x1.to(cuda_dev), L.to(cuda_dev), R.to(cuda_dev)
    dB = p.task_covar_grad(Ld, Rd)
    ref = mo.hadamard_dB(kind, x1d, None, LS, OS, Ld, Rd, lay)
    _within(("hadamard dB", PATH[backend], kind), name, dB, ref, mo.hadamard_dB_bound(kind, x1d, None, LS, OS, Ld, Rd, lay))
    assert torch.equal(dB, p.task_covar_grad(Ld, Rd))


@pytest.mark.parametrize("config", ["tc-scalar", "tc-ard", "simt-scalar"])
@pytest.mark.parametrize("name", ["n4200_straddle", "T32"])
def test_hadamard_hyper_gradients_within_bound(cuda_dev, config, name):
    """Lengthscale and outputscale gradients on 4200 rows with two-split segments: the scalar lengthscale on a tensor-core plan
    (fused kernel + combine + fp64 dot), ARD on a tensor-core plan and a scalar lengthscale on a SIMT plan (the per-segment
    bilinear kernel with B folded into the left factor)."""
    backend = "simt" if config.startswith("simt") else "tcgen05"
    ard = config.endswith("ard")
    path = "tc" if config == "tc-scalar" else "simt"
    kind = KINDS[(["tc-scalar", "tc-ard", "simt-scalar"].index(config) + 2 * (name == "T32")) % 4]
    x1, _, t1, _, T, _ = mo.hadamard_case(name, 31, t=4)
    ls = [0.4, 0.5, 0.6, 0.7] if ard else LS
    B = mo.random_B(T, 32)
    g = torch.Generator().manual_seed(33)
    L, R = torch.randn(x1.size(0), 4, generator=g), torch.randn(x1.size(0), 4, generator=g)
    p, lay = _hadamard(cuda_dev, kind, x1, None, t1, None, T, B, backend, ls=ls)
    x1d, Ld, Rd = x1.to(cuda_dev), L.to(cuda_dev), R.to(cuda_dev)
    gl, gs = p.bilinear_grad(Ld, Rd)
    rl, rs = mo.hadamard_grad(kind, x1d, None, B, ls, OS, Ld, Rd, lay)
    bl, bs = mo.hadamard_grad_bound(kind, x1d, None, B, ls, OS, Ld, Rd, lay, path, p.info()["n_sm"])
    _within(("hadamard grad", path, kind), name, torch.tensor(list(gl) + [gs]), torch.cat([rl, torch.tensor([rs])]),
            torch.cat([bl, torch.tensor([bs])]))
    gl2, gs2 = p.bilinear_grad(Ld, Rd)
    assert list(gl2) == list(gl) and gs2 == gs


# ---- Kronecker ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("Tt", mo.KRON_TT, ids=lambda v: f"T{v[0]}t{v[1]}")
def test_kron_products_within_bound(cuda_dev, backend, Tt):
    """N = 1450 (three splits of 8, 8 and 7 tiles), 1, 2, 4, 2 and 1 mixed chunks, T t not a multiple of 16 for (3, 6) and
    (7, 7); the noise added.  Repeated products are bit-identical."""
    T, t = Tt
    kind = KINDS[mo.KRON_TT.index(Tt) % 4]
    n, d = mo.KRON_SPLIT
    x = ko.points(n, d, 41)
    B = mo.random_B(T, 42)
    V = torch.randn(n * T, t, generator=torch.Generator().manual_seed(43))
    p, geo = _kron(cuda_dev, kind, x, None, T, B, backend, noise=0.1)
    assert geo["nsplit"] == 3
    xd, Vd = x.to(cuda_dev), V.to(cuda_dev)
    out = p.kmv(Vd, add_noise=True)
    ref = mo.kron_exact(kind, xd, None, B, LS, OS, Vd, T, t, noise=0.1)
    _within(("kron", PATH[backend], kind), f"T={T} t={t}", out, ref, mo.kron_bound(kind, xd, None, B, LS, OS, Vd, T, t, geo, exact=ref,
                                                                                   noise=0.1))
    assert torch.equal(out, p.kmv(Vd, add_noise=True))


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("N", mo.KRON_RED, ids=lambda v: f"N1={v[0]}")
def test_kron_dB_and_gradients_within_bound(cuda_dev, backend, N):
    """Cross plans of N1 in {2048, 2049, 4100} points against 1000 (two splits): dB over 1, 2 and 3 reduction chunks; the
    lengthscale and outputscale gradients over 2 mixed chunks (T = 3, t = 6), scalar and ARD.  Repeated calls are bit-identical."""
    N1, N2 = N
    T, t, d = 3, 6, 3
    kind = KINDS[(mo.KRON_RED.index(N) + 2 * (backend == "simt")) % 4]
    x1, x2 = ko.points(N1, d, 51), ko.points(N2, d, 52)
    B = mo.random_B(T, 53)
    g = torch.Generator().manual_seed(54)
    L, R = torch.randn(N1 * T, t, generator=g), torch.randn(N2 * T, t, generator=g)
    x1d, x2d, Ld, Rd = x1.to(cuda_dev), x2.to(cuda_dev), L.to(cuda_dev), R.to(cuda_dev)
    p, geo = _kron(cuda_dev, kind, x1, x2, T, B, backend)
    assert geo["nsplit"] == 2
    dB = p.task_covar_grad(Ld, Rd)
    _within(("kron dB", PATH[backend], kind), f"N1={N1}", dB, mo.kron_dB(kind, x1d, x2d, LS, OS, Ld, Rd, T, t),
            mo.kron_dB_bound(kind, x1d, x2d, LS, OS, Ld, Rd, T, t, geo))
    assert torch.equal(dB, p.task_covar_grad(Ld, Rd))
    for ls in (LS, [0.4, 0.5, 0.6]):
        path = "simt" if isinstance(ls, list) or backend == "simt" else "tc"
        p, _ = _kron(cuda_dev, kind, x1, x2, T, B, backend, ls=ls)
        gl, gs = p.bilinear_grad(Ld, Rd)
        rl, rs = mo.kron_grad(kind, x1d, x2d, B, ls, OS, Ld, Rd, T, t)
        bl, bs = mo.kron_grad_bound(kind, x1d, x2d, B, ls, OS, Ld, Rd, T, t, path, p.data.info()["n_sm"])
        _within(("kron grad", path, kind), f"N1={N1} ls={ls}", torch.tensor(list(gl) + [gs]), torch.cat([rl, torch.tensor([rs])]),
                torch.cat([bl, torch.tensor([bs])]))


# ---- NaN ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
def test_nan_in_a_second_split_poisons_exactly_its_column(cuda_dev, backend):
    """A NaN in one V entry whose column lies in a task's (Hadamard) or the data plan's (Kronecker) second split: every row of
    its output column is NaN, the other columns keep their bits.  The NaN is CUDA's canonical 0x7fffffff, which the Kronecker
    mix's fmaf returns for any NaN operand: the tensor-core V split once rounded it to -0 and the NaN vanished."""
    x1, _, t1, _, T, V = mo.hadamard_case("square", 61, t=7)
    p, lay = _hadamard(cuda_dev, "rbf", x1, None, t1, None, T, mo.random_B(T, 62), backend)
    j = int(lay["cols"][0][lay["tps"][0] * ko.TILE_J + 3])
    n, d = mo.KRON_SPLIT
    pk, geo = _kron(cuda_dev, "matern32", ko.points(n, d, 63), None, 3, mo.random_B(3, 64), backend)
    jk = (geo["T"] * ko.TILE_J + 3) * 3 + 1
    Vk = torch.randn(n * 3, 7, generator=torch.Generator().manual_seed(65))
    for op, row, VV in ((p, j, V), (pk, jk, Vk)):
        VV = VV.to(cuda_dev)
        clean = op.kmv(VV)
        Vn = VV.clone()
        Vn[row, 4] = CANONICAL_NAN
        out = op.kmv(Vn)
        assert torch.isnan(out[:, 4]).all(), row
        keep = [c for c in range(7) if c != 4]
        assert torch.equal(out[:, keep], clean[:, keep]), row


def test_zz_report_fraction_of_bound(cuda_dev):
    """Largest observed |engine - fp64| / bound per operator, path and kind over this module's cases (printed with -s)."""
    name = torch.cuda.get_device_name(0)
    smi = shutil.which("nvidia-smi")
    q = subprocess.run([smi, "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True) if smi else None
    name += f", power limit {(q.stdout.strip() if q else '') or 'unknown'}"
    for (op, path, kind), r in sorted(RATIOS.items()):
        print(f"[{name}] {op:13s} {path:4s} {kind:9s} max err / bound = {r:.3e}")
    assert RATIOS and all(r <= 1.0 and not math.isnan(r) for r in RATIOS.values())
