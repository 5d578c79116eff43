"""The fused K.V kernels (kmv_tc_kernel on the tensor cores, kmv_simt_kernel on CUDA cores, finished by kmv_finish_user_kernel)
entry by entry against the fp64 product of tests/kmv_oracle.py, within its derived worst-case bound, at their edges: every
operand width and ring depth with T tiles per split at the ring's phase flips, every SIMT DP, row / column / column-count edges,
diagonal tiles on shards, single kernel values through identity columns (the diagonal bit for bit), cancelling right-hand sides,
spread inputs, column independence, NaN propagation and kernel sums.  Every case asserts its backend and nsplit against the
geometry mirror, so it cannot silently stop reaching its edge (test_kmv_host.py checks the edges on 132 and 114 SMs)."""
import math
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu

import bilinear_oracle as bo  # noqa: E402
import kmv_oracle as ko  # noqa: E402

KINDS = list(bo.KINDS)
PATH = {"tcgen05": "tc", "simt": "simt"}
RATIOS = {}   # (path, kind) -> largest |engine - fp64| / bound seen
SPREAD = {}   # (kind, d) -> {path: largest |engine - fp64| / s}


def _plan(dev, kind, x1, x2, ls, os_, noise, backend, rb=0, rc=0):
    from gpytorch_b200.engine import Plan

    p = Plan(x1.to(dev), None if x2 is None else x2.to(dev), backend=backend, row_begin=rb, row_count=rc)
    p.set_hypers(kind, ls, os_, noise)
    n2 = x1.size(0) if x2 is None else x2.size(0)
    geo = ko.geometry(x1.size(0), n2, x1.size(1), backend, p.info()["n_sm"], rc or None)
    info = p.info()
    assert (info["backend"], info["nsplit"]) == (geo["backend"], geo["nsplit"]), (info, geo)
    return p, geo


def _check(tag, kind, x1, x2, ls, os_, noise, V, backend, rb=0, rc=0, add_noise=False, dev=None, nsplit=None, p=None):
    """Plan.kmv within the bound for every entry; returns (engine output [rows, t] on the device, fp64 exact, geometry)."""
    dev = dev or torch.device("cuda:0")
    if p is None:
        p, geo = _plan(dev, kind, x1, x2, ls, os_, noise, backend, rb, rc)
    else:
        geo = ko.geometry(x1.size(0), (x1 if x2 is None else x2).size(0), x1.size(1), backend, p.info()["n_sm"], rc or None)
    same = x2 is None
    out = p.kmv(V.to(dev), add_noise=add_noise)
    xd1, xd2 = x1.to(dev), None if same else x2.to(dev)
    nz = noise if add_noise else 0.0
    ref = ko.exact(kind, xd1, xd2, ls, os_, nz, V.to(dev), same=same, row_begin=rb, row_count=rc or None)
    path = PATH[backend]
    bnd = ko.bound(kind, xd1, xd2, ls, os_, nz, V.to(dev), path, nsplit or geo["nsplit"], geo["T"], same=same, row_begin=rb,
                   row_count=rc or None)
    err = (out.double() - ref).abs()
    frac = torch.where(bnd > 0, err / bnd, torch.where(err > 0, torch.inf, 0.0))
    worst = int(frac.argmax())
    r, c = divmod(worst, frac.size(1))
    assert bool(torch.isfinite(out).all()) and float(frac.max()) <= 1.0, \
        (tag, backend, kind, f"local row {r} (row tile {r // ko.TILE_I}, consumer {r % ko.TILE_I // 64}) column {c}",
         float(err.view(-1)[worst]), float(bnd.view(-1)[worst]), float(out.view(-1)[worst]), float(ref.view(-1)[worst]), geo)
    key = (path, kind)
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(frac.max()))
    return out, ref, geo


# ---- operand widths and ring depths -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kp", sorted(ko.KP_D))
def test_operand_widths_within_bound(cuda_dev, kp):
    d = ko.KP_D[kp]
    kind = KINDS[kp // 8 % 4]
    x1, x2 = ko.points(300, d, kp), ko.points(700, d, kp + 1)
    V = torch.randn(700, 17, generator=torch.Generator().manual_seed(kp))
    for backend in ("tcgen05", "simt"):
        _, _, geo = _check(f"KP={kp}", kind, x1, x2, 0.5 * math.sqrt(d), 1.3, 0.1, V, backend, add_noise=True)
        assert backend == "simt" or geo["KP"] == kp


@pytest.mark.parametrize("kp", ko.RING_KP)
def test_ring_edges_within_bound(cuda_dev, kp):
    """T tiles in one split, T in {1, 2, NS - 1, NS, NS + 1, 2 NS, 2 NS + 1}: the first ring pass, the producer's first wait on
    b_empty, the consumers' parity flips.  Cross plans, the noise asked for and ignored (test_kmv_host's noise_cross mutant)."""
    for d, T, n1, n2 in ko.ring_cases():
        if d != ko.KP_D[kp]:
            continue
        x1, x2 = ko.points(n1, d, 10 + T), ko.points(n2, d, 20 + T)
        V = torch.randn(n2, 17, generator=torch.Generator().manual_seed(T))
        kind = KINDS[T % 4]
        _, _, geo = _check(f"KP={kp} T={T}", kind, x1, x2, 0.5 * d ** 0.5, 1.3, 0.1, V, "tcgen05", add_noise=True)
        assert geo["T"] == T


@pytest.mark.parametrize("case", range(3))
def test_large_row_plans_within_bound(cuda_dev, case):
    """456 row tiles (several waves of one CTA per SM) and one long split: nsplit = 1 is what the heuristic picks."""
    d, T, n1, n2 = ko.large_row_cases()[case]
    x1, x2 = ko.points(n1, d, 40 + case), ko.points(n2, d, 50 + case)
    V = torch.randn(n2, 16, generator=torch.Generator().manual_seed(case))
    _check(f"large {case}", KINDS[case], x1, x2, 0.5 * d ** 0.5, 0.7, 0.0, V, "tcgen05")


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_several_splits_with_a_shorter_last_split(cuda_dev, backend):
    n, d = ko.SPLIT_SQUARE
    x = ko.points(n, d, 61)
    V = torch.randn(n, 33, generator=torch.Generator().manual_seed(62))
    for kind in KINDS:
        _check("splits", kind, x, None, 0.6, 1.1, 0.2, V, backend, add_noise=True)


# ---- SIMT ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", ko.SIMT_D)
def test_simt_every_dp_within_bound(cuda_dev, d):
    x1, x2 = ko.points(300, d, d), ko.points(500, d, d + 1)
    V = torch.randn(500, 16, generator=torch.Generator().manual_seed(d))
    _check(f"simt d={d}", KINDS[d % 4], x1, x2, 0.4 * math.sqrt(d), 1.2, 0.0, V, "simt")


def test_simt_last_split_of_one_column_within_bound(cuda_dev):
    n1, n2, d = ko.CPS_EDGE
    x1, x2 = ko.points(n1, d, 71), ko.points(n2, d, 72)
    V = torch.randn(n2, 5, generator=torch.Generator().manual_seed(73))
    _, _, geo = _check("cps edge", "matern32", x1, x2, 0.5, 1.0, 0.0, V, "simt")
    assert geo["nsplit"] > 1 and n2 % geo["cps"] == 1


# ---- row and column edges -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_row_column_and_width_edges_within_bound(cuda_dev, backend):
    for a, n1 in enumerate(ko.N1_EDGES):
        for b, n2 in enumerate(ko.N2_EDGES):
            t = ko.T_EDGES[(a + b) % len(ko.T_EDGES)]
            kind = KINDS[(a + 2 * b) % 4]
            x1, x2 = ko.points(n1, 3, 100 + a), ko.points(n2, 3, 200 + b)
            V = torch.randn(n2, t, generator=torch.Generator().manual_seed(a * 7 + b))
            _check(f"{n1}x{n2} t={t}", kind, x1, x2, 0.5, 1.3, 0.1, V, backend, add_noise=True)
        t = ko.T_EDGES[a % len(ko.T_EDGES)]
        x = ko.points(n1, 3, 300 + a)
        V = torch.randn(n1, t, generator=torch.Generator().manual_seed(a))
        _check(f"square {n1} t={t}", KINDS[a % 4], x, None, 0.5, 1.3, 0.1, V, backend, add_noise=True)


# ---- diagonal tiles, shards and single entries --------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
@pytest.mark.parametrize("kind", KINDS)
def test_shards_within_bound_and_exact_diagonal(cuda_dev, backend, kind):
    """Square plans and shards whose diagonal crosses 64-column tiles and split starts, with random V and with identity columns
    at tile edges, split starts and the diagonal.  With V = e_j every output entry is one kernel value, and on the diagonal it
    is fp32(outputscale) bit for bit: a = 0 gives k = 1 exactly, P_lo = V_lo = 0, every other product is an exact 0."""
    x = ko.points(ko.SHARD_N, 3, 5)
    os32 = float(bo.f32(1.3))
    for rb, rc in ko.SHARDS:
        V = torch.randn(ko.SHARD_N, 17, generator=torch.Generator().manual_seed(rb))
        p, geo = _plan(cuda_dev, kind, x, None, 0.5, 1.3, 0.1, backend, rb, rc)
        _check(f"shard {rb}+{rc}", kind, x, None, 0.5, 1.3, 0.1, V, backend, rb, rc, add_noise=True, p=p)
        first = geo["T"] * ko.TILE_J
        picks = [0, 63, 64, 127, 128, first - 1, first, first + 1, rb, rb + 1, rb + 63, rb + 64, rb + rc - 1, first + 64]
        Vi, cols = ko.identity_cols(ko.SHARD_N, picks)
        out, _, _ = _check(f"shard {rb}+{rc} identity", kind, x, None, 0.5, 1.3, 0.0, Vi, backend, rb, rc, p=p)
        ndiag = 0
        for c, j in enumerate(cols):
            if rb <= j < rb + rc:
                assert out[j - rb, c].item() == os32, (rb, rc, j, out[j - rb, c].item())
                ndiag += 1
        assert ndiag >= 3


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_cross_plan_of_coinciding_points_within_bound(cuda_dev, backend):
    """x2 a copy of x1: no mask, every diagonal pair at distance 0 through the GEMM (RBF may exceed 1 by rounding)."""
    x = ko.points(700, 4, 81)
    V = torch.randn(700, 16, generator=torch.Generator().manual_seed(82))
    for kind in KINDS:
        _check("coinciding", kind, x, x.clone(), 0.7, 1.0, 0.0, V, backend)


# ---- cancelling right-hand sides ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
@pytest.mark.parametrize("kind", KINDS)
def test_cancelling_rhs_is_pure_error_within_bound(cuda_dev, backend, kind):
    """x repeated twice and V[j + n] = -V[j]: columns j and j + n of K are equal, so the exact product is 0 and the output is
    the engine's error alone, against the bound's absolute allowance."""
    n = 700
    x = ko.points(n, 3, 91).repeat(2, 1)
    v = torch.randn(n, 16, generator=torch.Generator().manual_seed(92))
    V = torch.cat([v, -v])
    out, ref, _ = _check("cancel square", kind, x, None, 0.5, 1.3, 0.0, V, backend)
    assert ref.abs().max().item() < 1e-12
    xr = ko.points(300, 3, 93)
    _check("cancel cross", kind, xr, x, 0.5, 1.3, 0.0, V, backend)


# ---- spread inputs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,z2", [(1, 4e3), (3, 4e3), (41, 1e3)])
@pytest.mark.parametrize("kind", KINDS)
def test_spread_inputs_within_bound(cuda_dev, d, z2, kind):
    """Packed |z|^2 up to z2 (span 40-130 lengthscales in 1-D): the 3xTF32 term of GEMM1 grows with |z|^2, the SIMT path's
    direct differences do not.  Prints both paths' largest error relative to s (-s)."""
    x = ko.spread_points(2000, d, kind, 3 + d, z2)
    V = torch.randn(2000, 4, generator=torch.Generator().manual_seed(5 + d))
    res = {}
    for backend in ("tcgen05", "simt"):
        out, ref, _ = _check(f"spread d={d}", kind, x, None, 1.0, 1.0, 0.0, V, backend)
        res[PATH[backend]] = (out.double() - ref).abs().max().item()
    SPREAD[(kind, d)] = res
    print(f"spread {kind:9s} d={d:2d} |z|^2<={z2:.0e}: max err tc {res['tc']:.3e}  simt {res['simt']:.3e}")


# ---- column independence, determinism, NaN ------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_columns_are_independent_and_calls_deterministic(cuda_dev, backend):
    from gpytorch_b200.engine import Plan

    x = ko.points(900, 5, 11).to(cuda_dev)
    p = Plan(x, backend=backend).set_hypers("matern52", 0.6, 1.2, 0.1)
    V = torch.randn(900, 33, generator=torch.Generator().manual_seed(12)).to(cuda_dev)
    o16 = p.kmv(V[:, :16].contiguous(), add_noise=True)
    for c in range(16):
        assert torch.equal(o16[:, c], p.kmv(V[:, c:c + 1].contiguous(), add_noise=True)[:, 0]), c
    o33 = p.kmv(V, add_noise=True)
    parts = [p.kmv(V[:, a:b].contiguous(), add_noise=True) for a, b in ((0, 16), (16, 32), (32, 33))]
    assert torch.equal(o33, torch.cat(parts, 1))
    for _ in range(3):
        assert torch.equal(p.kmv(V, add_noise=True), o33)


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_nan_in_one_entry_of_v_poisons_exactly_its_column(cuda_dev, backend):
    """As fp32 K @ V in the reference: the NaN reaches every row of its column, also through pairs where k underflows to 0,
    and the other columns keep their bits."""
    from gpytorch_b200.engine import Plan

    x1 = ko.points(300, 2, 13)
    x2 = torch.cat([ko.points(200, 2, 14), ko.points(1, 2, 15) + 50.0])   # the last column is far from every row: k = 0
    p = Plan(x1.to(cuda_dev), x2.to(cuda_dev), backend=backend).set_hypers("rbf", 0.3, 1.0, 0.0)
    V = torch.randn(201, 7, generator=torch.Generator().manual_seed(16)).to(cuda_dev)
    clean = p.kmv(V)
    for j, c in ((5, 2), (200, 6)):
        Vn = V.clone()
        Vn[j, c] = float("nan")
        out = p.kmv(Vn)
        assert torch.isnan(out[:, c]).all(), (j, c)
        keep = [q for q in range(7) if q != c]
        assert torch.equal(out[:, keep], clean[:, keep]), (j, c)


# ---- kernel sums --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backends", [("tcgen05", "tcgen05"), ("tcgen05", "simt")])
def test_kernel_sum_within_the_sum_of_term_bounds(cuda_dev, backends):
    """The finish kernel's per-slot fmaf: each term's bound with the partial slots of both terms as its nsplit (every slot
    is one fmaf of the running sum of both terms), and the sum plan's noise once."""
    from gpytorch_b200.engine import Plan

    n = 1450
    x = ko.points(n, 4, 17)
    V = torch.randn(n, 17, generator=torch.Generator().manual_seed(18))
    pa, ga = _plan(cuda_dev, "rbf", x, None, 0.6, 1.2, 0.0, backends[0])
    pb, gb = _plan(cuda_dev, "matern32", x, None, 0.9, 0.7, 0.0, backends[1])
    ps = Plan(x.to(cuda_dev)).set_sum([pa, pb]).set_hypers("rbf", [1.0], 1.0, 0.1)
    slots = ga["nsplit"] + gb["nsplit"]
    assert ps.info()["nsplit"] == slots and slots > 2
    out = ps.kmv(V.to(cuda_dev), add_noise=True).double()
    xd, Vd = x.to(cuda_dev), V.to(cuda_dev)
    ref = ko.exact("rbf", xd, None, 0.6, 1.2, 0.1, Vd, same=True) + ko.exact("matern32", xd, None, 0.9, 0.7, 0.0, Vd, same=True)
    bnd = ko.bound("rbf", xd, None, 0.6, 1.2, 0.1, Vd, PATH[backends[0]], slots, ga["T"], same=True) \
        + ko.bound("matern32", xd, None, 0.9, 0.7, 0.0, Vd, PATH[backends[1]], slots, gb["T"], same=True)
    err = (out - ref).abs()
    assert (err <= bnd).all(), float((err / bnd).max())
    RATIOS[("sum", "+".join(PATH[b] for b in backends))] = float((err / bnd).max())


def test_zz_report_fraction_of_bound(cuda_dev):
    """Largest observed |engine - fp64| / bound per path and kind over this module's cases (printed with -s)."""
    name = torch.cuda.get_device_name(0)
    smi = shutil.which("nvidia-smi")
    q = subprocess.run([smi, "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True) if smi else None
    name += f", power limit {(q.stdout.strip() if q else '') or 'unknown'}"
    for (path, kind), r in sorted(RATIOS.items()):
        print(f"[{name}] kmv {path:4s} {kind:9s} max err / bound = {r:.3e}")
    for (kind, d), res in sorted(SPREAD.items()):
        print(f"[{name}] kmv spread {kind:9s} d={d:2d} max err tc {res['tc']:.3e} simt {res['simt']:.3e}")
    assert all(r <= 1.0 for r in RATIOS.values())
