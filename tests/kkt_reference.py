"""Reference of the KKT factorisation and solve (csrc/chd_kkt.cu, tile format of csrc/chd_kkt_tiles.cuh) for
tests/test_kkt_factor_gpu.py and tests/test_kkt_reference_cpu.py, written from the storage rules, not from the kernels:

* pack / unpack between a symmetric scipy.sparse matrix (band unknowns 0..Na-1, border unknowns Na..Na+nbl-1) with its
  right-hand side and one sequence's tile-format buffer  band | bord | corn;
* the unpivoted block LDL^T in the kernels' elimination order (8x8 block columns of the band, then the border Schur
  complement), in fp64 or np.longdouble, leaving its factors where the kernels leave theirs, plus |L||D||L^T| on the
  pattern for the rounding bounds;
* matrix generators in the regime the solver assembles (quasi-definite: PSD Gauss-Newton block + delta_w I on primal
  unknowns, -delta_c or -1/Sigma - delta_c on interleaved multipliers, dense border columns on primal unknowns);
* the ctypes loader of the harness (tests/kkt/libchd_kkt_harness.so), which __graft_entry__.build() makes."""
import ctypes as C
import os
import re

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "contact-human-dynamics_b200", "csrc")
HARNESS = os.path.join(HERE, "kkt", "libchd_kkt_harness.so")
DELTA_C, DW_MIN, DW_MAX = 1e-8, 1e-8, 1e4      # CHD_DELTA_C, CHD_DW_MIN, CHD_DW_MAX (csrc/chd_dev.h)


def _define(name):
    txt = open(os.path.join(CSRC, "chd_dev.h")).read()
    return float(re.search(r"#define %s (\S+)" % name, txt).group(1))


assert (_define("CHD_DELTA_C"), _define("CHD_DW_MIN"), _define("CHD_DW_MAX")) == (DELTA_C, DW_MIN, DW_MAX)


# ---------------------------------------------------------------------------------------------------------------
# strides and tile-format storage
# ---------------------------------------------------------------------------------------------------------------
def strides(Na_max, nb_max, w_max, w_fix_max):
    """The storage sizes of chd_kkt_plan (csrc/chd_kkt_plan.h) that do not depend on the device."""
    nbc, Q, Qfix, nbt = (Na_max + 7) // 8, (w_max + 7) // 8 + 1, (w_fix_max + 7) // 8 + 1, (nb_max + 1 + 7) // 8
    return dict(nbc_max=nbc, Q=Q, Qfix=Qfix, nbt=nbt, kstride=nbc * Q * 64 + nbc * nbt * 64 + 64 * nbt * nbt)


def views(buf, st):
    """band (nbc_max, Q, 8, 8): block column J, tile t = block row J + t;  bord (nbc_max, nbt, 8, 8): border tile of
    block column J, row b -> tile b >> 3, row b & 7;  corn (nbp8, nbp8) row major."""
    nbc, Q, nbt = st["nbc_max"], st["Q"], st["nbt"]
    nb_ = nbc * Q * 64
    no = nb_ + nbc * nbt * 64
    return (buf[:nb_].reshape(nbc, Q, 8, 8), buf[nb_:no].reshape(nbc, nbt, 8, 8),
            buf[no:no + 64 * nbt * nbt].reshape(8 * nbt, 8 * nbt))


def pack(K, r, Na, nbl, st, Qst, out=None):
    """Tile-format buffer of the symmetric matrix K (lower triangle read) of order Na + nbl and right-hand side r, for a
    stage whose band spans Qst tiles per block column: what chd_k_asm leaves in Kwork plus the right-hand-side row
    chd_kkt_assemble writes (border row NBR = nbl, corner row NBR), identity on the padding rows Na..Np-1."""
    buf = np.zeros(st["kstride"]) if out is None else out
    band, bord, corn = views(buf, st)
    L = sp.tril(sp.coo_matrix(K)).tocsr().tocoo()
    i, j, v = L.row, L.col, L.data
    m = i < Na
    t = (i[m] >> 3) - (j[m] >> 3)
    assert (t < Qst).all(), "entry outside the band of the stage"
    band[j[m] >> 3, t, i[m] & 7, j[m] & 7] = v[m]
    m = (i >= Na) & (j < Na)
    b = i[m] - Na
    bord[j[m] >> 3, b >> 3, b & 7, j[m] & 7] = v[m]
    m = j >= Na
    corn[i[m] - Na, j[m] - Na] = v[m]
    Np = (Na + 7) & ~7
    k = np.arange(Na, Np)
    band[k >> 3, 0, k & 7, k & 7] = 1.0
    NBR = nbl
    k = np.arange(Na)
    bord[k >> 3, NBR >> 3, NBR & 7, k & 7] = r[:Na]
    corn[NBR, :nbl] = r[Na:]
    return buf


def unpack(buf, Na, nbl, st, Qst):
    """Inverse of pack: (K as a symmetric csr matrix, r)."""
    band, bord, corn = views(buf, st)
    Np, NBR = (Na + 7) & ~7, nbl
    rows, cols, vals = [], [], []
    J, t, a, c = np.meshgrid(np.arange(Np // 8), np.arange(Qst), np.arange(8), np.arange(8), indexing="ij")
    i, j = 8 * (J + t) + a, 8 * J + c
    m = (i < Na) & (j < Na) & (i >= j)
    rows.append(i[m]), cols.append(j[m]), vals.append(band[:Np // 8, :Qst][m])
    bq, jq = np.meshgrid(np.arange(nbl), np.arange(Na), indexing="ij")
    rows.append(Na + bq.ravel()), cols.append(jq.ravel()), vals.append(bord[jq >> 3, bq >> 3, bq & 7, jq & 7].ravel())
    iq, jq = np.tril_indices(nbl)
    rows.append(Na + iq), cols.append(Na + jq), vals.append(corn[iq, jq])
    i, j, v = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    nz = v != 0
    i, j, v = i[nz], j[nz], v[nz]
    off = i != j
    K = sp.coo_matrix((np.concatenate([v, v[off]]), (np.concatenate([i, j[off]]), np.concatenate([j, i[off]]))),
                      shape=(Na + nbl,) * 2).tocsr()
    k = np.arange(Na)
    r = np.concatenate([bord[k >> 3, NBR >> 3, NBR & 7, k & 7], corn[NBR, :nbl]])
    return K, r


# ---------------------------------------------------------------------------------------------------------------
# reference elimination
# ---------------------------------------------------------------------------------------------------------------
def _tile_ldl(T):
    """LDL^T of the lower triangle of an 8x8 tile: (unit L, d)."""
    a = np.tril(T).copy()
    L, d = np.eye(8, dtype=T.dtype), np.zeros(8, T.dtype)
    for p in range(8):
        d[p] = a[p, p]
        L[p + 1:, p] = a[p + 1:, p] / d[p]
        a[p + 1:, p + 1:] -= np.outer(L[p + 1:, p], a[p + 1:, p])
    return L, d


def ldl_solve(buf, Na, nbl, st, Qst, dtype=np.float64):
    """The block LDL^T of chd_kkt_factor / chd_kkt_border and the solve of chd_kkt_border / chd_kkt_backsub on a packed
    buffer (right-hand side included), in `dtype`.  Returns dict: fac = the buffer with the factors where the kernel
    leaves them (diagonal tiles: unit L strictly below the diagonal, d on it; panel and border tiles: X = final L,
    border row NBR = the forward-substituted right-hand side over d), E = |L||D||L^T| on the same places (diagonal tiles:
    lower triangle), x = solution (Na + nbl), fail = a bad pivot (|d| <= 1e-300 or not finite in the band, not > 0 in
    the border), dS / ES = the border Schur pivots and their |L||D||L^T|."""
    fac = np.array(buf, dtype=dtype)
    E = np.zeros_like(fac)
    band, bord, corn = views(fac, st)
    Eb, Ebo, Ec = views(E, st)
    Np, q, NBR = (Na + 7) & ~7, Qst - 1, nbl
    nbc, nbt_s = Np // 8, (nbl + 1 + 7) // 8
    fail = False
    for Kc in range(nbc):
        tq = min(q, nbc - 1 - Kc)
        L0, d = _tile_ldl(band[Kc, 0])
        fail |= not (np.all(np.abs(d) > 1e-300) and np.all(np.isfinite(d)))
        W = np.eye(8, dtype=dtype)                  # L0^-1 by forward substitution on the rows
        for rr in range(1, 8):
            W[rr] -= L0[rr, :rr] @ W[:rr]
        A = np.concatenate([band[Kc, 1:1 + tq].reshape(-1, 8), bord[Kc, :nbt_s].reshape(-1, 8)])
        Y = A @ W.T
        X = Y * (1.0 / d)[None, :]
        band[Kc, 0] = np.tril(L0, -1) + np.diag(d)
        band[Kc, 1:1 + tq] = X[:8 * tq].reshape(tq, 8, 8)
        bord[Kc, :nbt_s] = X[8 * tq:].reshape(nbt_s, 8, 8)
        aL0, ad, aX = np.abs(L0), np.abs(d), np.abs(X)
        Eb[Kc, 0] = np.tril(Eb[Kc, 0] + (aL0 * ad) @ aL0.T)
        Ep = (aX * ad) @ aL0.T
        Eb[Kc, 1:1 + tq] += Ep[:8 * tq].reshape(tq, 8, 8)
        Ebo[Kc, :nbt_s] += Ep[8 * tq:].reshape(nbt_s, 8, 8)
        ng = tq + nbt_s
        P = X @ Y.T
        PA = aX @ (aX * ad).T
        P4 = P.reshape(ng, 8, ng, 8).transpose(0, 2, 1, 3)
        PA4 = PA.reshape(ng, 8, ng, 8).transpose(0, 2, 1, 3)
        for gj in range(tq):
            band[Kc + 1 + gj, :tq - gj] -= P4[gj:tq, gj]
            Eb[Kc + 1 + gj, :tq - gj] += PA4[gj:tq, gj]
        bord[Kc + 1:Kc + 1 + tq, :nbt_s] -= P4[tq:, :tq].transpose(1, 0, 2, 3)
        Ebo[Kc + 1:Kc + 1 + tq, :nbt_s] += PA4[tq:, :tq].transpose(1, 0, 2, 3)
        corn[:8 * nbt_s, :8 * nbt_s] -= P[8 * tq:, 8 * tq:]
        Ec[:8 * nbt_s, :8 * nbt_s] += PA[8 * tq:, 8 * tq:]
    # border Schur complement (rows 0..nbl-1 of the corner) and the forward substitution of its right-hand side (row NBR)
    cc, ec = corn.copy(), Ec.copy()
    dS = np.zeros(nbl, dtype)
    for k in range(nbl):
        dk = cc[k, k]
        fail |= not (dk > 0 and np.isfinite(dk))
        dS[k] = dk
        l = cc[k + 1:nbl, k] / dk
        cc[k + 1:nbl, k + 1:nbl] -= np.outer(l, cc[k + 1:nbl, k])
        ec[k + 1:nbl, k + 1:nbl] += np.outer(np.abs(l), np.abs(cc[k + 1:nbl, k]))
        cc[NBR, k + 1:nbl] -= l * cc[NBR, k]
    xb = np.zeros(nbl, dtype)
    acc = cc[NBR, :nbl].copy()
    for k in range(nbl - 1, -1, -1):
        xb[k] = acc[k] / cc[k, k]
        acc[:k] -= cc[k, :k] * xb[k]
    # band back-substitution: acc = u - Lb^T xb, then x_K = L0^-T acc_K, acc_J -= L(K, J)^T x_K
    xs = np.zeros(Np, dtype)
    Xb = bord[:nbc].transpose(0, 3, 1, 2).reshape(Np, -1)        # (band unknown, border row)
    acc = Xb[:, NBR] - Xb[:, :nbl] @ xb
    for Kc in range(nbc - 1, -1, -1):
        T0 = band[Kc, 0]
        a = acc[8 * Kc:8 * Kc + 8]
        xk = np.zeros(8, dtype)
        for cl in range(7, -1, -1):
            xk[cl] = a[cl] - T0[cl + 1:, cl] @ xk[cl + 1:]
        xs[8 * Kc:8 * Kc + 8] = xk
        nrow = min(q, Kc)
        for g in range(nrow):
            acc[8 * (Kc - 1 - g):8 * (Kc - g)] -= band[Kc - 1 - g, g + 1].T @ xk
    return dict(fac=fac, E=E, x=np.concatenate([xs[:Na], xb]), fail=fail, dS=dS, ES=np.diag(ec)[:nbl] + np.abs(dS))


# ---------------------------------------------------------------------------------------------------------------
# matrix generators
# ---------------------------------------------------------------------------------------------------------------
def make_kkt(rng, Na, nbl, w, mult_frac=0.35, zero_tiles=False, delta_w=None):
    """Quasi-definite KKT matrix of order Na + nbl as the solver assembles it (DESIGN.md section 3): primal unknowns get a
    banded PSD Gauss-Newton block R^T R + delta_w I (half bandwidth w, delta_w in [CHD_DW_MIN, CHD_DW_MAX]); multiplier
    unknowns, interleaved in the band, couple to primal ones within the band and carry -delta_c (equality rows) or
    -1/Sigma - delta_c (Sigma in 1e-8 .. 1e8) on the diagonal; the border unknowns are primal, with dense rows over a
    stretch of the band's primal unknowns and a corner that keeps the primal block positive definite (so the border
    Schur pivots are positive).  zero_tiles: residuals and couplings only inside a block or between blocks 1 or q apart,
    border rows over a range of block columns -- whole zero tiles in the band and the border, some of which receive
    fill-in.  Returns (K as a symmetric csr matrix, multiplier mask)."""
    q = (w + 7) // 8
    n = Na + nbl
    mult = rng.random(Na) < mult_frac
    if Na:
        mult[rng.integers(Na)] = False
    prim = np.flatnonzero(~mult)
    dw = 10.0 ** rng.uniform(np.log10(DW_MIN), np.log10(DW_MAX)) if delta_w is None else delta_w
    I, J, V = [], [], []

    def add(i, j, v):
        I.append(np.asarray(i)), J.append(np.asarray(j)), V.append(np.asarray(v, float))

    # Gauss-Newton residuals: one per primal unknown p, on p and up to five primal companions behind it
    res_r, res_c, res_v = [], [], []
    if len(prim):
        for k in range(6):
            if zero_tiles:
                off = rng.choice([0, 1, q], size=len(prim), p=[0.7, 0.05, 0.25]) if q else np.zeros(len(prim), int)
                blk = np.maximum((prim >> 3) - off, 0)
                c = 8 * blk + rng.integers(0, 8, len(prim))
            else:
                c = prim - rng.integers(0, w + 1, len(prim))
            c = np.clip(c, 0, Na - 1) if k else prim
            ok = ~mult[c] & (rng.random(len(prim)) < (1.0 if k == 0 else 0.6))
            res_r.append(np.flatnonzero(ok)), res_c.append(c[ok])
            res_v.append(rng.standard_normal(ok.sum()) * 10.0 ** rng.uniform(-1, 1, ok.sum()))
        R = sp.coo_matrix((np.concatenate(res_v), (np.concatenate(res_r), np.concatenate(res_c))), shape=(len(prim), Na))
        H = (R.T @ R).tocoo()
        add(H.row, H.col, H.data)
        add(prim, prim, 10.0 ** rng.uniform(-2, 2, len(prim)) + dw)
    # multipliers: couplings to primal unknowns in the band, -delta_c or -1/Sigma - delta_c on the diagonal
    mi = np.flatnonzero(mult)
    for k in range(4):
        if zero_tiles:
            c = 8 * (mi >> 3) + rng.integers(0, 8, len(mi))
        else:
            c = mi + rng.integers(-w, w + 1, len(mi))
        c = np.clip(c, 0, Na - 1)
        ok = ~mult[c]
        v = rng.standard_normal(ok.sum()) * 10.0 ** rng.uniform(-1, 1, ok.sum())
        add(mi[ok], c[ok], v), add(c[ok], mi[ok], v)
    eq = rng.random(len(mi)) < 0.3
    sig = 10.0 ** rng.uniform(-8, 8, len(mi))
    add(mi, mi, np.where(eq, -DELTA_C, -1.0 / sig - DELTA_C))
    Kb = sp.coo_matrix((np.concatenate(V), (np.concatenate(I), np.concatenate(J))), shape=(Na, Na)).tocsr()
    if nbl == 0:
        return _symmetric(Kb), mult
    # border: dense rows over a stretch of primal unknowns, corner = 1.5 B H^-1 B^T + a positive diagonal
    Bd = np.zeros((nbl, Na))
    for b in range(nbl):
        if zero_tiles:
            lo = 8 * rng.integers(0, max(1, (Na + 7) // 8)); hi = min(Na, lo + 8 * rng.integers(1, 4))
        else:
            lo = rng.integers(0, max(1, Na // 2)); hi = min(Na, lo + max(1, int(Na * rng.uniform(0.25, 1.0))))
        cols = prim[(prim >= lo) & (prim < hi)]
        Bd[b, cols] = rng.standard_normal(len(cols)) * (rng.random(len(cols)) < 0.7)
    Hp = Kb[prim][:, prim].tocsc()
    Bp = Bd[:, prim]
    HiB = spla.splu(Hp).solve(Bp.T) if len(prim) else np.zeros((0, nbl))
    Cn = 1.5 * (Bp @ HiB)
    Cn = 0.5 * (Cn + Cn.T) + np.diag(10.0 ** rng.uniform(-2, 1, nbl) + dw)
    K = sp.bmat([[Kb, sp.csr_matrix(Bd.T)], [sp.csr_matrix(Bd), sp.csr_matrix(Cn)]]).tocsr()
    return _symmetric(K), mult


def _symmetric(K):
    """Exactly symmetric copy of K from its lower triangle (R^T R in floating point need not be)."""
    L = sp.tril(K)
    K = (L + sp.tril(L, -1).T).tocsr()
    K.eliminate_zeros()
    return K


def inertia(K, Na, nbl, st, Qst):
    """(positive, negative) pivots of the reference elimination."""
    f = ldl_solve(pack(K, np.zeros(Na + nbl), Na, nbl, st, Qst), Na, nbl, st, Qst)
    band = views(f["fac"], st)[0]
    d = np.concatenate([np.diagonal(band[:(Na + 7) // 8, 0], axis1=1, axis2=2).ravel()[:Na], f["dS"]])
    return int((d > 0).sum()), int((d < 0).sum())


# ---------------------------------------------------------------------------------------------------------------
# reference solution and error measures
# ---------------------------------------------------------------------------------------------------------------
def refined_solution(K, r):
    """splu in fp64 plus two steps of iterative refinement with the residual in np.longdouble; also an estimate of
    kappa_inf(K) (= kappa_1, K symmetric)."""
    Kc = sp.csc_matrix(K)
    lu = spla.splu(Kc)
    x = lu.solve(r)
    Kl, rl = Kc.astype(np.longdouble), np.asarray(r, np.longdouble)
    for _ in range(2):
        res = rl - Kl @ np.asarray(x, np.longdouble)
        x = x + lu.solve(np.asarray(res, np.float64))
    inv = spla.LinearOperator(Kc.shape, matvec=lu.solve, rmatvec=lu.solve, dtype=np.float64)
    kappa = spla.onenormest(inv) * spla.norm(Kc, 1)
    return x, kappa


def backward_error(K, x, r):
    """Normwise backward error ||r - K x||_inf / (||K||_inf ||x||_inf + ||r||_inf), residual in np.longdouble."""
    Kl = sp.csr_matrix(K).astype(np.longdouble)
    res = np.asarray(r, np.longdouble) - Kl @ np.asarray(x, np.longdouble)
    den = spla.norm(sp.csr_matrix(K), np.inf) * np.abs(x).max(initial=0) + np.abs(r).max(initial=0)
    return float(np.abs(res).max(initial=0) / den) if den else 0.0


# ---------------------------------------------------------------------------------------------------------------
# the harness (tests/kkt/libchd_kkt_harness.so)
# ---------------------------------------------------------------------------------------------------------------
def _plan_type():
    body = re.search(r"struct ChdKktPlan \{(.*?)\};", open(os.path.join(CSRC, "chd_kkt_plan.h")).read(), re.S).group(1)
    fields = []
    for typ, names in re.findall(r"^\s*(int|size_t)\s+([^;]+);", body, re.M):
        fields += [(n.strip(), C.c_int if typ == "int" else C.c_size_t) for n in names.split(",")]
    return type("ChdKktPlan", (C.Structure,), {"_fields_": fields})


class Harness:
    """ctypes view of the harness: plan(...) and run(...); the library must have been built by build()."""

    def __init__(self):
        if not os.path.exists(HARNESS):
            raise RuntimeError("%s is missing: build it with __graft_entry__.build() (make -C tests/kkt)" % HARNESS)
        self.L = C.CDLL(HARNESS)
        self.T = _plan_type()
        assert self.L.chd_kkt_harness_plan_size() == C.sizeof(self.T)
        self.L.chd_kkt_harness_plan.argtypes = [C.c_int] * 5 + [C.c_longlong, C.POINTER(self.T), C.c_char_p, C.c_int]
        self.L.chd_kkt_harness_run.argtypes = [C.c_int] * 6 + [C.c_longlong] + [C.c_void_p] * 11 + [C.c_char_p, C.c_int]

    def plan(self, Na_max, nb_max, w_max, w_fix_max, n_max, optin=0):
        p, err = self.T(), C.create_string_buffer(256)
        rc = self.L.chd_kkt_harness_plan(Na_max, nb_max, w_max, w_fix_max, n_max, optin, C.byref(p), err, 256)
        assert rc == 0, err.value.decode()
        return {k: getattr(p, k) for k, _ in self.T._fields_}

    def run(self, dims, seqs, K, rhs0, rhs1, mu, optin=0):
        """dims = (Na_max, nb_max, w_max, w_fix_max, n_max); seqs = list of (Na, nb, nb_fix, opt_dur); K: (B, kstride),
        rhs0 / rhs1: (B, Na_max + nb_max); mu: (B,).  Returns (factored K, sol, fail, kernel name)."""
        B = len(seqs)
        ints = [np.ascontiguousarray([s[k] for s in seqs], np.int32) for k in range(4)]
        Kf = np.array(K, np.float64, order="C")
        r0, r1 = np.ascontiguousarray(rhs0, np.float64), np.ascontiguousarray(rhs1, np.float64)
        mu = np.ascontiguousarray(mu, np.float64)
        sol = np.zeros((B, dims[0] + dims[1]))
        fail = np.zeros(B, np.int32)
        which = C.c_int(-1)
        err = C.create_string_buffer(256)
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        rc = self.L.chd_kkt_harness_run(B, *dims, optin, *[ptr(a) for a in ints], ptr(Kf), ptr(r0), ptr(r1), ptr(mu),
                                        ptr(sol), ptr(fail), C.byref(which), err, 256)
        assert rc == 0, err.value.decode()
        return Kf, sol, fail, "chd_k_kkt" if which.value == 1 else "chd_k_kkt_gwin"
