"""CPU tests of the host-side NLP layout (chd_layout.cpp, reached through the C ABI in host-only mode)
against the oracle's independent TOWR-style construction."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.util import master_to_oracle_perm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n_ee,seed", [(2, 0), (2, 3), (4, 1)])
def test_layout_matches_oracle(chd, n_ee, seed):
    from oracle.phys import OracleProblem
    p = chd.synth.make_problem(seed, n_ee=n_ee)
    b = chd.phys.PhysBatch([p], host_only=True)
    o = OracleProblem(p)
    # stage 3 (phys_optim.cpp:663-711) adds the PhaseDurations sets and the TotalTime rows; the product keeps one layout
    # for all stages and additionally carries the duration bounds (0, 500) of parameters.cpp:60 as rows
    o.set_stage("3")
    n_dur = sum(len(d) - 1 for d in p.ee_durations)
    assert b.sizes[0, 0] == o.n and b.sizes[0, 1] == o.m + n_dur
    np.testing.assert_allclose(b.get_x()[0, :o.n], o.get_x(), rtol=0, atol=1e-14)
    o.set_stage("2.2")
    n, m = o.n, o.m
    assert n == b.sizes[0, 0] - n_dur and m == b.sizes[0, 1] - n_dur - p.n_ee
    # initial point (nlp_formulation.cpp:106-203)
    x0 = b.get_x()[0, :n]
    xlo, xhi = o.var_bounds()
    xo = o.get_x()
    np.testing.assert_allclose(x0, xo, rtol=0, atol=1e-14)
    lay = b.layout()
    # fixed variables = equality-bounded ones (start / final base velocity)
    assert np.array_equal(lay["var_kkt"][0, :n] < 0, xlo == xhi)
    assert (lay["var_kkt"][0, n:n + n_dur] >= b.sizes[0, 3]).all()      # durations: border unknowns (stage 3)
    # row bounds
    sl = chd.phys.master_row_slices(b, 0, lay)
    im, io = master_to_oracle_perm(sl, o)
    cl, cu = o.con_bounds()
    np.testing.assert_allclose(lay["row_lo"][0, im], cl[io], rtol=0, atol=0)
    np.testing.assert_allclose(lay["row_hi"][0, im], cu[io], rtol=0, atol=0)
    # Jacobian pattern: every oracle nonzero is covered by a slot of the same row
    J = o.jac().tocsr()
    ptr, col = lay["ent_ptr"][0], lay["ent_col"][0]
    for rm, ro in zip(im, io):
        mine = set(col[ptr[rm]:ptr[rm + 1]].tolist())
        theirs = set(J.indices[J.indptr[ro]:J.indptr[ro + 1]][np.abs(J.data[J.indptr[ro]:J.indptr[ro + 1]]) > 0].tolist())
        assert theirs <= mine, (rm, ro, sorted(theirs - mine))
    # KKT ordering: unknowns are a permutation, bandwidth covers every equality coupling
    Na, nb, w = b.sizes[0, 3], b.sizes[0, 4], b.sizes[0, 5]
    n, m = b.sizes[0, 0], b.sizes[0, 1]
    vk, rk = lay["var_kkt"][0, :n], lay["row_kkt"][0, :m]
    used = np.concatenate([vk[vk >= 0], rk[rk >= 0]])
    assert len(np.unique(used)) == len(used) == Na + nb
    lo_, hi_ = lay["row_lo"][0, :m], lay["row_hi"][0, :m]
    assert (rk[lo_ == hi_] >= 0).all()          # every equality row is a KKT unknown
    for r in np.nonzero(rk >= 0)[0]:
        c = col[ptr[r]:ptr[r + 1]]
        k = vk[c[c >= 0]]
        k = k[(k >= 0) & (k < Na)]
        if len(k):
            assert np.abs(k - rk[r]).max() <= w


def test_ragged_batch_padding(chd):
    ps = [chd.synth.make_problem(s, n_ee=2) for s in range(4)]
    b = chd.phys.PhysBatch(ps, host_only=True)
    assert b.dims["batch"] == 4
    assert b.dims["n_max"] == b.sizes[:, 0].max() and b.dims["m_max"] == b.sizes[:, 1].max()
    singles = [chd.phys.PhysBatch([p], host_only=True) for p in ps]
    for i, s in enumerate(singles):
        assert np.array_equal(s.sizes[0], b.sizes[i])
        n = s.sizes[0, 0]
        np.testing.assert_array_equal(s.get_x()[0, :n], b.get_x()[i, :n])


def _header_prototypes(path):
    """{name: (return type, [parameter types])} of every chd_ function a C header declares."""
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(path).read(), flags=re.S)
    src = "\n".join(l for l in src.splitlines() if not l.lstrip().startswith("#"))
    out = {}
    for stmt in src.split(";"):
        stmt = " ".join(re.split(r"[{}]", stmt)[-1].split())
        m = re.fullmatch(r"(.+?)\s*\b(chd_\w+)\s*\((.*)\)", stmt)
        if m:
            params = m.group(3).strip()
            out[m.group(2)] = (m.group(1).replace(" *", "*"),
                               [] if params in ("", "void") else [re.sub(r"\w+$", "", p).strip() for p in params.split(",")])
    return out


def test_binding_table_matches_header_and_exports(chd):
    """include/chd.h, the ctypes table of phys.py and the dynamic symbols of libchd.so agree: the same functions, and
    each declared to ctypes with the header's return type and parameter list."""
    import ctypes as C
    proto = _header_prototypes(os.path.join(ROOT, "include", "chd.h"))
    table = chd.phys.SIGNATURES
    assert set(proto) == set(table), (sorted(set(proto) - set(table)), sorted(set(table) - set(proto)))
    scalar = {"int32_t": C.c_int32, "int64_t": C.c_int64, "int": C.c_int, "double": C.c_double, "float": C.c_float}
    ret = {"int": C.c_int, "int64_t": C.c_int64, "const char*": C.c_char_p, "void": None}
    for name, (rtype, params) in proto.items():
        restype, argtypes = table[name]
        assert restype is ret[rtype], (name, rtype, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for p, a in zip(params, argtypes):
            if "*" in p:
                assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (name, p, a)
            else:
                assert a is scalar[p.replace("const ", "")], (name, p, a)
    chd.phys.load_lib()          # applies the table: every declared function resolves
    nm = subprocess.run(["nm", "-D", "--defined-only", chd.phys.lib_path()], check=True, capture_output=True, text=True)
    exported = {w[-1] for w in map(str.split, nm.stdout.splitlines()) if w and re.fullmatch(r"chd_\w+", w[-1])}
    assert exported == set(proto), ("exported, not declared", sorted(exported - set(proto)),
                                    "declared, not exported", sorted(set(proto) - exported))


def test_column_oriented_slot_index(chd):
    """ent_row / col_ptr / col_ent (used by the device to gather J^T y per variable) describe exactly the slots of
    ent_ptr / ent_col: every slot with a variable appears once, under its own column, with its own row."""
    ps = [chd.synth.make_problem(s, n_ee=ne) for s, ne in ((0, 2), (3, 4))]
    b = chd.phys.PhysBatch(ps, host_only=True)
    lay, idx = b.layout(), b.slot_index()
    for i in range(len(ps)):
        n, m, nslots = (int(v) for v in b.sizes[i, :3])
        ep, ec = lay["ent_ptr"][i], lay["ent_col"][i]
        er, cp, ce = idx["ent_row"][i], idx["col_ptr"][i], idx["col_ent"][i]
        for r in range(m):
            assert (er[ep[r]:ep[r + 1]] == r).all()
        assert cp[0] == 0 and (np.diff(cp[:n + 1]) >= 0).all()
        used = np.flatnonzero(ec[:nslots] >= 0)
        assert cp[n] == len(used)
        assert sorted(ce[:cp[n]].tolist()) == used.tolist()
        for v in range(n):
            assert (ec[ce[cp[v]:cp[v + 1]]] == v).all()


def test_adaptive_band_border_split(chd):
    """The layout builder chooses per sequence which stance variables go to the dense border: walking gaits keep
    a border of a few dozen columns, densely switching contacts (0.13-0.33 s stances) fit in the band (DESIGN.md 2)."""
    walk = chd.phys.PhysBatch([chd.synth.make_problem(0, n_ee=2)], host_only=True).dims
    dense = chd.phys.PhysBatch([chd.synth.make_problem(0, n_frames=300, n_ee=4, dense=True)], host_only=True).dims
    assert 12 <= walk["nb_max"] <= 60 and walk["w_max"] <= 160
    assert dense["nb_max"] <= 40 and dense["w_max"] <= 400
    # every KKT unknown index is used exactly once (band + border)
    b = chd.phys.PhysBatch([chd.synth.make_problem(1, n_frames=150, n_ee=4, dense=True)], host_only=True)
    lay = b.layout()
    Na, nb = int(b.sizes[0, 3]), int(b.sizes[0, 4])
    ks = np.concatenate([lay["var_kkt"][0][lay["var_kkt"][0] >= 0], lay["row_kkt"][0][lay["row_kkt"][0] >= 0]])
    assert sorted(ks.tolist()) == list(range(Na + nb))
