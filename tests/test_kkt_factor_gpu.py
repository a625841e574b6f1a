"""The KKT factorisation and solve (csrc/chd_kkt.cu) against a dense-order fp64 / extended-precision reference, kernel by
kernel, through the test harness tests/kkt/kkt_harness.cu (the product's phase functions in chd_kkt_body's order:
context, right-hand side, band LDL^T, border Schur complement, back-substitution).

Each case packs seeded quasi-definite matrices (tests/kkt_reference.py) into the tile format, runs one launch and checks
every sequence:
* no pivot failure;
* factors: per block column (diagonal tile, panel tiles, border tiles incl. the right-hand-side row), the largest
  distance of the kernel's L and d to the extended-precision (np.longdouble) elimination in the same order, in units of
  each entry's first-order rounding bound  eps (|L||D||L^T|_ij + |L_ij| |L||D||L^T|_jj) / |d_j|  (eps |L||D||L^T|_jj
  for d), is at most FACTOR_SLACK times the largest such distance of the fp64 CPU elimination over all block columns
  (floored at 1).  The fp64 CPU run measures how far this elimination's rounding propagates -- its growth: the
  matrices have kappa up to 1e16, so the propagated part dwarfs the local bound, and where in the elimination it
  surfaces depends on the rounding of each run, so the bound is elimination-wide rather than per column; the GPU's fp64
  arithmetic differs only in the order of the 8-term sums and FMA contraction;
* backward error  ||r - K x||_inf / (||K||_inf ||x||_inf + ||r||_inf)  at most BERR_SLACK times the fp64 CPU
  elimination's, floored at BERR_FLOOR;
* forward error against splu + two refinement steps (residual in long double) within FWD_SLACK * kappa * berr + FWD_FLOOR.
Beside that: bitwise equalities the storage contract promises (ragged batches, storage a stage does not use,
determinism) and the failure flags.  Both kernels run every shape the plan allows: chd_k_kkt naturally, chd_k_kkt_gwin
forced through a small shared-memory opt-in limit (GWIN_OPTIN)."""
import numpy as np
import pytest

import tests.kkt_reference as R
from tests.test_kkt_plan_cpu import parent_plan

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
GWIN_OPTIN = 101376   # per-block opt-in limit under which every window of these shapes goes to chd_k_kkt_gwin
# the GPU's rounding differs from the fp64 CPU elimination's only in the order of sums (8 terms per tile product, then
# one product per block column) and FMA contraction: same size, not the same values.  16x covers the spread of the
# largest such error; a skipped tile, a wrong scale or a dropped term is off by orders of magnitude (~1/eps)
FACTOR_SLACK = 16.0
BERR_SLACK, BERR_FLOOR = 8.0, 4 * EPS
# first-order perturbation bound ||dx|| / ||x|| <= 2 kappa berr; onenormest may underestimate kappa by a small factor
FWD_SLACK, FWD_FLOOR = 20.0, 16 * EPS
FACTOR_COLS = 160


def _kernel_for(dims, optin):
    p = parent_plan(*dims, optin=optin)
    if p["status"] != 0:
        return None
    return "chd_k_kkt" if p["win_smem"] else "chd_k_kkt_gwin"


def _modes(dims):
    """(optin, kernel) pairs this shape runs on: the device limit, and the forced global window if that differs."""
    out = [(0, _kernel_for(dims, R_OPTIN))]
    g = _kernel_for(dims, GWIN_OPTIN)
    if out[0][1] == "chd_k_kkt" and g == "chd_k_kkt_gwin":
        out.append((GWIN_OPTIN, g))
    return out


R_OPTIN = 232448      # H100 per-block opt-in limit (cudaDevAttrMaxSharedMemoryPerBlockOptin)


@pytest.fixture(scope="module")
def H():
    return R.Harness()


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
class Seq:
    """One sequence of a launch: Na band unknowns, nb / nb_fix border unknowns, half bandwidths w / w_fix, stage."""

    def __init__(self, Na, nb, w, opt_dur=1, nb_fix=None, w_fix=None, zero_tiles=False, seed=0):
        self.Na, self.nb, self.w, self.opt_dur = Na, nb, w, opt_dur
        self.nb_fix = nb if nb_fix is None else nb_fix
        self.w_fix = w if w_fix is None else w_fix
        self.zero_tiles, self.seed = zero_tiles, seed

    @property
    def nbl(self):
        return self.nb if self.opt_dur else self.nb_fix


def build(dims, seqs):
    """Packed buffers, right-hand sides and the systems of a launch with strides dims = (Na_max, nb_max, w_max,
    w_fix_max, n_max)."""
    Na_max, nb_max = dims[0], dims[1]
    st = R.strides(*dims[:4])
    B, nv = len(seqs), Na_max + nb_max
    Kbuf = np.zeros((B, st["kstride"]))
    rhs0, rhs1, mu = np.zeros((B, nv)), np.zeros((B, nv)), np.zeros(B)
    systems = []
    for b, s in enumerate(seqs):
        rng = np.random.default_rng(1000 + s.seed)
        nbl, Qst = s.nbl, (st["Q"] if s.opt_dur else st["Qfix"])
        K, _ = R.make_kkt(rng, s.Na, nbl, s.w if s.opt_dur else s.w_fix, zero_tiles=s.zero_tiles)
        idx = np.concatenate([np.arange(s.Na), Na_max + np.arange(nbl)])
        rhs0[b, idx] = rng.standard_normal(len(idx)) * 10.0 ** rng.uniform(-2, 2, len(idx))
        rhs1[b, idx] = rng.standard_normal(len(idx))
        mu[b] = 10.0 ** rng.uniform(-9, -1)
        r = rhs0[b, idx] + mu[b] * rhs1[b, idx]      # what chd_kkt_assemble writes: rhs0 + mu * rhs1 in fp64
        R.pack(K, r, s.Na, nbl, st, Qst, out=Kbuf[b])
        systems.append((K, r, nbl, Qst))
    return st, Kbuf, rhs0, rhs1, mu, systems


def run(H, dims, seqs, optin=0, built=None):
    st, Kbuf, rhs0, rhs1, mu, systems = built or build(dims, seqs)
    Kf, sol, fail, kernel = H.run(dims, [(s.Na, s.nb, s.nb_fix, s.opt_dur) for s in seqs], Kbuf, rhs0, rhs1, mu, optin)
    return dict(st=st, K=Kbuf, Kf=Kf, sol=sol, fail=fail, kernel=kernel, systems=systems)


def _col_ratio(got, ld, bound):
    """Per-entry |got - ld| / bound; exact agreement required where the bound is zero."""
    diff = np.abs(got - ld).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, diff / np.where(bound > 0, bound, 1.0), np.where(diff > 0, np.inf, 0.0))
    return r


def check_factors(st, Kin, Kf, s, nbl, Qst, where):
    """Factors left in Kwork against the same-order references (see the module docstring)."""
    f64 = R.ldl_solve(Kin, s.Na, nbl, st, Qst)
    # the factors of the leading block columns depend on the leading part of the matrix only: the extended-precision
    # elimination (numpy's long double has no BLAS) stops after FACTOR_COLS block columns on long horizons
    nbc = min((s.Na + 7) // 8, FACTOR_COLS)
    Na_f = s.Na if nbc == (s.Na + 7) // 8 else 8 * nbc
    fld = R.ldl_solve(Kin, Na_f, nbl, st, Qst, dtype=np.longdouble)
    if Na_f < s.Na:
        f64c = R.ldl_solve(Kin, Na_f, nbl, st, Qst)
    else:
        f64c = f64
    q, nbt_s = Qst - 1, (nbl + 1 + 7) // 8
    g_band, g_bord, _ = R.views(Kf, st)
    c_band, c_bord, _ = R.views(f64c["fac"], st)
    l_band, l_bord, _ = R.views(fld["fac"], st)
    e_band, e_bord, _ = R.views(fld["E"], st)
    d = np.abs(np.diagonal(l_band[:nbc, 0], axis1=1, axis2=2)).astype(np.float64)          # (nbc, 8)
    Edd = np.diagonal(e_band[:nbc, 0], axis1=1, axis2=2).astype(np.float64)
    low = np.tril(np.ones((8, 8), bool), -1)
    rg, rc = [], []
    for J in range(nbc):
        tq = min(q, (Na_f + 7) // 8 - 1 - J)
        dj, Ej = d[J][None, :], Edd[J][None, :]
        # d on the diagonal, unit L strictly below it, X in the panel and border tiles
        parts = [(np.diagonal(g_band[J, 0]), np.diagonal(c_band[J, 0]), np.diagonal(l_band[J, 0]), EPS * Edd[J])]
        for g, c, l, e in ((g_band[J, 0][low], c_band[J, 0][low], l_band[J, 0][low], e_band[J, 0][low]),):
            Ll = np.abs(l).astype(np.float64)
            bound = EPS * (e.astype(np.float64) + Ll * np.broadcast_to(Ej, (8, 8))[low]) / np.broadcast_to(dj, (8, 8))[low]
            parts.append((g, c, l, bound))
        for g, c, l, e in ((g_band[J, 1:1 + tq], c_band[J, 1:1 + tq], l_band[J, 1:1 + tq], e_band[J, 1:1 + tq]),
                           (g_bord[J, :nbt_s], c_bord[J, :nbt_s], l_bord[J, :nbt_s], e_bord[J, :nbt_s])):
            bound = EPS * (e.astype(np.float64) + np.abs(l).astype(np.float64) * Ej) / dj
            parts.append((g, c, l, bound))
        rg.append(max((_col_ratio(g, l, b).max(initial=0) for g, c, l, b in parts), default=0))
        rc.append(max((_col_ratio(c, l, b).max(initial=0) for g, c, l, b in parts), default=0))
    growth = max(max(rc, default=0), 1.0)
    for J in range(nbc):
        assert rg[J] <= FACTOR_SLACK * growth, (where, "block column", J, "gpu", rg[J], "cpu fp64", rc[J], "cpu max", growth)
    return f64


def check_solution(res, b, s, where, factors=True):
    K, r, nbl, Qst = res["systems"][b]
    st = res["st"]
    assert res["fail"][b] == 0, (where, "pivot failure flagged")
    x = res["sol"][b, :s.Na + nbl]
    if factors:
        f64 = check_factors(st, res["K"][b], res["Kf"][b], s, nbl, Qst, where)
        x_cpu = f64["x"]
    else:
        x_cpu = R.ldl_solve(res["K"][b], s.Na, nbl, st, Qst)["x"]
    assert np.isfinite(x).all(), where
    be_gpu, be_cpu = R.backward_error(K, x, r), R.backward_error(K, x_cpu, r)
    assert be_gpu <= max(BERR_SLACK * be_cpu, BERR_FLOOR), (where, be_gpu, be_cpu)
    x_ref, kappa = R.refined_solution(K, r)
    fe = np.abs(x - x_ref).max() / max(np.abs(x_ref).max(), 1e-300)
    assert fe <= FWD_SLACK * kappa * max(be_gpu, be_cpu) + FWD_FLOOR, (where, fe, kappa, be_gpu)


def check_launch(H, dims, seqs, optin, kernel, name):
    res = run(H, dims, seqs, optin)
    print("%s: %s" % (name, res["kernel"]))
    assert res["kernel"] == kernel, (name, res["kernel"], kernel)
    for b, s in enumerate(seqs):
        check_solution(res, b, s, "%s seq %d (Na=%d nb=%d w=%d stage %s) on %s" % (
            name, b, s.Na, s.nb, s.w, "3" if s.opt_dur else "fixed", kernel))
    return res


def _dims_of(seqs, n_max=None):
    Na_max = max(s.Na for s in seqs)
    return (Na_max, max(s.nb for s in seqs), max(s.w for s in seqs), max(s.w_fix for s in seqs),
            n_max if n_max is not None else Na_max + max(s.nb for s in seqs))


def _param(name, seqs, n_max=None, marks=()):
    dims = _dims_of(seqs, n_max)
    return [pytest.param(name, dims, seqs, optin, kern, id="%s-%s" % (name, kern), marks=marks)
            for optin, kern in _modes(dims)]


# ---------------------------------------------------------------------------------------------------------------
# shape grid: every boundary value of Na, nb and w at least once, both stages
# ---------------------------------------------------------------------------------------------------------------
NAS = (5, 8, 9, 63, 64, 65, 1001)
NBS = (0, 6, 7, 8, 15, 31, 96)
WSS = (0, 1, 7, 8, 9, 64, 150)


def _grid():
    out = []
    for i in range(14):
        Na, nb, w, od = NAS[i % 7], NBS[(3 * i + 1) % 7], WSS[(5 * i + 2) % 7], i % 2
        s = Seq(Na, nb, w, opt_dur=od, nb_fix=nb if od else nb // 2, w_fix=w if od else w // 2, zero_tiles=i % 3 == 0,
                seed=i)
        out += _param("grid%02d-Na%d-nb%d-w%d-%s" % (i, Na, nb, w, "st3" if od else "fix"), [s])
    # windows wide enough for chd_k_kkt's shared-memory window, with fewer block columns than the band is wide
    for i, (Na, nb) in enumerate(zip((5, 8, 9, 64, 1001), (0, 7, 8, 15, 31))):
        od = 1 - i % 2
        s = Seq(Na, nb, 150, opt_dur=od, nb_fix=nb if od else nb // 2, w_fix=150 if od else 70, zero_tiles=i == 4,
                seed=20 + i)
        out += _param("wide%d-Na%d-nb%d-w150-%s" % (i, Na, nb, "st3" if od else "fix"), [s])
    return out


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _grid())
def test_shape_grid(H, name, dims, seqs, optin, kernel):
    check_launch(H, dims, seqs, optin, kernel, name)


# ---------------------------------------------------------------------------------------------------------------
# trailing-update paths of the global window: 64 panel groups (update_compact), 65 (update_wide), ~85 (banded
# stage 3), the 96-group limit
# ---------------------------------------------------------------------------------------------------------------
def _groups(w, nb):
    return (w + 7) // 8 + (nb + 1 + 7) // 8


UPDATE_CASES = [("groups64-compact", 504, 7, False), ("groups65-wide", 512, 7, True),
                ("groups85-wide", 600, 79, False), ("groups96-wide", 688, 79, True)]


@pytest.mark.parametrize("name,w,nb,zt", UPDATE_CASES, ids=[c[0] for c in UPDATE_CASES])
def test_update_paths(H, name, w, nb, zt):
    assert _groups(w, nb) == int(name[6:8])
    seqs = [Seq(1001, nb, w, zero_tiles=zt, seed=40 + len(name)), Seq(777, nb // 2, w - 40, seed=41)]
    dims = _dims_of(seqs)
    assert _kernel_for(dims, R_OPTIN) == "chd_k_kkt_gwin"
    check_launch(H, dims, seqs, 0, "chd_k_kkt_gwin", name + ("-update_wide" if _groups(w, nb) > 64 else "-update_compact"))


# ---------------------------------------------------------------------------------------------------------------
# the benchmark's batches (strides from the layout builder), both stages
# ---------------------------------------------------------------------------------------------------------------
PRODUCT = {"phys-120f-2ee": (dict(F=120, n_ee=2), None), "phys-120f-4ee": (dict(F=120, n_ee=4), None),
           "long-600f-4ee-dense": (dict(F=600, n_ee=4, dense=True), None),
           "banded-stage3-200f": (dict(F=200, n_ee=4, dense=True), 96)}


def _product_case(chd, key):
    kw, band = PRODUCT[key]
    ps = [chd.synth.make_problem(s, kw["F"], kw["n_ee"], dense=kw.get("dense", False)) for s in range(2)]
    b = chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=band)
    d, sz, fx = b.dims, b.sizes, b.sizes_fixed()
    dims = (d["na_max"], d["nb_max"], d["w_max"], int(fx[:, 1].max()), d["n_max"])
    seqs = [Seq(int(sz[i, 3]), int(sz[i, 4]), int(sz[i, 5]), opt_dur=1 - i, nb_fix=int(fx[i, 0]), w_fix=int(fx[i, 1]),
                seed=60 + i) for i in range(2)]
    b.close()
    return dims, seqs


@pytest.mark.parametrize("key", list(PRODUCT))
@pytest.mark.parametrize("force_gwin", [False, True], ids=["natural", "gwin"])
def test_product_shapes(H, chd, key, force_gwin):
    dims, seqs = _product_case(chd, key)
    modes = dict((k, o) for o, k in _modes(dims))
    if force_gwin and "chd_k_kkt" not in modes:
        pytest.skip("runs on chd_k_kkt_gwin already")
    kernel = "chd_k_kkt_gwin" if force_gwin else _kernel_for(dims, R_OPTIN)
    if kernel not in modes:
        pytest.skip("the plan does not allow %s here" % kernel)
    check_launch(H, dims, seqs, modes[kernel], kernel, "%s-%s" % (key, kernel))


# ---------------------------------------------------------------------------------------------------------------
# ragged batch: each sequence bitwise equal to itself solved alone at its own strides
# ---------------------------------------------------------------------------------------------------------------
RAGGED = [Seq(1001, 31, 150, seed=80), Seq(65, 6, 9, seed=81), Seq(300, 96, 64, opt_dur=0, nb_fix=40, w_fix=30, seed=82),
          Seq(9, 0, 1, seed=83), Seq(513, 15, 8, zero_tiles=True, seed=84)]


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _param("ragged", RAGGED))
def test_ragged_batch_bitwise(H, name, dims, seqs, optin, kernel):
    """Extra window groups of a narrower sequence only meet zero X tiles (skipped, or a zero product that leaves C
    unchanged), extra border tiles are never used, and every target tile gets one product per block column whatever
    the compacted list pairs it with: a sequence's solution does not depend on the batch it is solved in."""
    res = check_launch(H, dims, seqs, optin, kernel, name)
    for b, s in enumerate(seqs):
        alone_dims = (s.Na, s.nb, s.w, s.w_fix, s.Na + s.nb)
        # alone on the same kernel where the plan allows it (the arithmetic of the two kernels is the same too)
        alone_optin = 0
        if kernel == "chd_k_kkt_gwin" and _kernel_for(alone_dims, GWIN_OPTIN) == "chd_k_kkt_gwin":
            alone_optin = GWIN_OPTIN
        one = run(H, alone_dims, [s], alone_optin)
        n = s.Na + s.nbl
        assert one["fail"][0] == 0
        np.testing.assert_array_equal(res["sol"][b, :n], one["sol"][0, :n], err_msg="seq %d: %s vs alone on %s" % (
            b, kernel, one["kernel"]))


# ---------------------------------------------------------------------------------------------------------------
# storage a fixed-duration stage does not use: band tiles Qfix..Q-1, border rows past NBR, the corner beyond it
# ---------------------------------------------------------------------------------------------------------------
UNUSED = [Seq(1001, 31, 150, opt_dur=0, nb_fix=20, w_fix=60, seed=90), Seq(200, 15, 64, opt_dur=0, nb_fix=7, w_fix=9, seed=91),
          Seq(64, 8, 9, opt_dur=0, nb_fix=0, w_fix=0, seed=92)]


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _param("unused-storage", UNUSED))
def test_unused_storage_not_read(H, name, dims, seqs, optin, kernel):
    built = build(dims, seqs)
    st, Kbuf = built[0], built[1]
    junk = Kbuf.copy()
    rng = np.random.default_rng(7)
    for b, s in enumerate(seqs):
        band, bord, corn = R.views(junk[b], st)
        nbc = (s.Na + 7) // 8
        band[:nbc, st["Qfix"]:] = rng.uniform(0.5, 2.0, band[:nbc, st["Qfix"]:].shape)
        NBR = s.nbl
        rows = np.arange(8 * st["nbt"]) > NBR
        bv = bord.reshape(bord.shape[0], -1, 8)     # (block column, border row, column)
        bv[:nbc, rows] = rng.uniform(0.5, 2.0, bv[:nbc, rows].shape)
        corn[rows, :] = rng.uniform(0.5, 2.0, corn[rows, :].shape)
        corn[:, rows] = rng.uniform(0.5, 2.0, corn[:, rows].shape)
    clean = run(H, dims, seqs, optin, built=built)
    dirty = run(H, dims, seqs, optin, built=(st, junk) + built[2:])
    assert clean["kernel"] == dirty["kernel"] == kernel
    np.testing.assert_array_equal(clean["fail"], dirty["fail"])
    np.testing.assert_array_equal(clean["sol"], dirty["sol"])
    for b, s in enumerate(seqs):
        check_solution(clean, b, s, "%s seq %d" % (name, b))


# ---------------------------------------------------------------------------------------------------------------
# n_max at the alias boundary of the shared-memory window, and back-substitution chunks that do not divide nbc
# ---------------------------------------------------------------------------------------------------------------
def _alias_n_max(dims):
    lo, hi = 0, 1 << 20
    assert _kernel_for(dims[:4] + (lo,), R_OPTIN) == "chd_k_kkt"
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _kernel_for(dims[:4] + (mid,), R_OPTIN) == "chd_k_kkt":
            lo = mid
        else:
            hi = mid
    return lo


def _chunk_rows(p, n_max, Qst):
    """R of chd_kkt_backsub: block rows per staging chunk."""
    nbc, Q, nbt = p["nbc_max"], p["Q"], p["nbt"]
    win_region = p["win_tiles"] * 64 + Q * nbt * 64
    n_even, xs_len = (n_max + 1) & ~1, 8 * nbc + 8 * nbt
    return max(1, (win_region - (n_even + xs_len if p["win_smem"] else 0)) // 64 // (2 * Qst))


@pytest.mark.parametrize("force_gwin", [False, True], ids=["chd_k_kkt", "chd_k_kkt_gwin"])
def test_alias_boundary_and_chunks(H, force_gwin):
    Na_max, nb_max, w = 1001, 15, 150
    dims = _alias_n_max((Na_max, nb_max, w, w, 0))
    dims = (Na_max, nb_max, w, w, dims)
    optin = GWIN_OPTIN if force_gwin else 0
    kernel = _kernel_for(dims, GWIN_OPTIN if force_gwin else R_OPTIN)
    assert kernel == ("chd_k_kkt_gwin" if force_gwin else "chd_k_kkt")
    p = parent_plan(*dims, optin=GWIN_OPTIN if force_gwin else R_OPTIN)
    Rr = _chunk_rows(p, dims[4], p["Q"])
    nbcs = sorted({Rr, Rr + 1, 2 * Rr + 1, p["nbc_max"]})
    assert max(nbcs) <= p["nbc_max"], (Rr, p["nbc_max"])
    seqs = [Seq(8 * k - (3 if k % 2 else 0), nb_max, w, seed=100 + k, zero_tiles=k % 3 == 0) for k in nbcs]
    seqs[-1].Na = Na_max
    check_launch(H, dims, seqs, optin, kernel, "alias-n_max%d-R%d-nbc%s" % (dims[4], Rr, nbcs))


# ---------------------------------------------------------------------------------------------------------------
# determinism and failure flags
# ---------------------------------------------------------------------------------------------------------------
DET = [Seq(1001, 31, 150, seed=120), Seq(300, 96, 64, opt_dur=0, nb_fix=40, w_fix=30, seed=121)]


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _param("determinism", DET))
def test_two_launches_bitwise_equal(H, name, dims, seqs, optin, kernel):
    built = build(dims, seqs)
    a, b = run(H, dims, seqs, optin, built=built), run(H, dims, seqs, optin, built=built)
    assert a["kernel"] == b["kernel"] == kernel
    np.testing.assert_array_equal(a["Kf"], b["Kf"])
    np.testing.assert_array_equal(a["sol"], b["sol"])
    np.testing.assert_array_equal(a["fail"], b["fail"])


FAIL = [Seq(300, 15, 150, seed=130 + i) for i in range(5)]


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _param("pivot-failure", FAIL))
def test_pivot_failure_flags(H, name, dims, seqs, optin, kernel):
    """An exactly singular diagonal tile (band unknown 8k with no entry at all), a border unknown whose Schur pivot is 0,
    a NaN entry: each flags its own sequence only; the others solve correctly."""
    st, Kbuf, rhs0, rhs1, mu, systems = build(dims, seqs)
    band, bord, corn = R.views(Kbuf[1], st)               # band unknown 80: row and column zero
    k = 80
    band[k >> 3, :, :, k & 7] = 0.0
    band[k >> 3, 0, k & 7, :] = 0.0
    for t in range(1, st["Q"]):
        if (k >> 3) - t >= 0:
            band[(k >> 3) - t, t, k & 7, :] = 0.0
    bord[k >> 3, :, :, k & 7] = 0.0
    band, bord, corn = R.views(Kbuf[2], st)               # border unknown 3: row and column zero
    bv = bord.reshape(bord.shape[0], -1, 8)
    bv[:, 3, :] = 0.0
    corn[3, :] = 0.0
    corn[:, 3] = 0.0
    band, bord, corn = R.views(Kbuf[3], st)               # a NaN inside a panel tile
    band[10, 2, 3, 4] = np.nan
    band, bord, corn = R.views(Kbuf[4], st)               # a NaN in a border row
    bord[20, 1, 2, 5] = np.nan
    res = run(H, dims, seqs, optin, built=(st, Kbuf, rhs0, rhs1, mu, systems))
    assert res["kernel"] == kernel
    assert list(res["fail"]) == [0, 1, 1, 1, 1], res["fail"]
    for b in range(len(seqs)):
        ref = R.ldl_solve(Kbuf[b], seqs[b].Na, seqs[b].nbl, st, st["Q"])
        assert ref["fail"] == (b != 0), b
    check_solution(res, 0, seqs[0], name + " seq 0")


# ---------------------------------------------------------------------------------------------------------------
# regression: with one band tile per block column (half bandwidth 0 of the stage) the first panel group is a border
# tile, and the trailing update skipped its corner block as if it were the next diagonal tile (warp 0's): the border
# Schur complement missed every band contribution to its first 8 x 8 block.  And warp 0 only factors the next diagonal
# tile after updating it, so with no band tile below the diagonal the diagonal tiles after the first were never
# factored.  (The storage may still hold more band tiles: a fixed-duration stage with w_fix = 0.)
# ---------------------------------------------------------------------------------------------------------------
CORNER = [Seq(8, 15, 0, seed=140), Seq(61, 7, 0, seed=141), Seq(200, 31, 40, opt_dur=0, nb_fix=12, w_fix=0, seed=142)]
CORNER_WS = [Seq(1001, 15, 150, opt_dur=0, nb_fix=9, w_fix=0, seed=143), Seq(300, 7, 150, seed=144)]


@pytest.mark.parametrize("name,dims,seqs,optin,kernel", _param("corner-block-single-band-tile", CORNER) +
                         _param("corner-block-single-band-tile-window", CORNER_WS))
def test_regression_corner_block_single_band_tile(H, name, dims, seqs, optin, kernel):
    check_launch(H, dims, seqs, optin, kernel, name)
