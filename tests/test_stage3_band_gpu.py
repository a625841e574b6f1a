"""GPU tests of banded switch times (`PhysBatch(stage3_band_above=...)`): the same problems solved with the switch
times in the dense border and in the band, and -- above the dense border's limit of 96 phase durations -- a 200-frame
densely switching gait against the CPU oracle and the long-horizon configuration at full size."""
import numpy as np
import pytest

from tests.util import duration_blocks, master_to_oracle_perm, to_tau

pytestmark = pytest.mark.gpu

TRUST = 0.04   # CHD_TAU_TRUST [s]


def _close(got, exp, n_ee):
    """max |diff| of positions / angles, forces; asserts the tolerances of test_solved_trajectories_match_cpu_oracle."""
    npos, nfrc = 6 + 3 * n_ee, 6 + 6 * n_ee
    dp, df = np.abs(got[:, :npos] - exp[:, :npos]).max(), np.abs(got[:, npos:nfrc] - exp[:, npos:nfrc]).max()
    assert dp <= 1e-5 and df <= 1e-3, (dp, df)
    np.testing.assert_array_equal(got[:, nfrc:], exp[:, nfrc:])
    return dp, df


def test_banded_and_border_forms_agree(chd):
    """Benchmark seeds (2 feet) with every sequence's switch times banded (0) against the default dense border."""
    ps = [chd.synth.make_problem(s, n_ee=2) for s in range(16)]
    ref = chd.phys.PhysBatch(ps).solve()
    bb = chd.phys.PhysBatch(ps, stage3_band_above=0)
    assert (bb.sizes_fixed()[:, 0] == bb.sizes[:, 4]).all()        # no switch time in the border
    got = bb.solve()
    st, it = got["stage_status"], got["stage_iters"]
    np.testing.assert_array_equal(st[:4], ref["stage_status"][:4])
    np.testing.assert_array_equal(it[:4], ref["stage_iters"][:4])
    fixed = [[_close(got["samples"][snap, i, :120], ref["samples"][snap, i, :120], 2) for i in range(16)] for snap in (0, 1)]
    print("stages 1.1-2.2: max |diff| positions %.2e, forces %.2e" % (np.max([f[0] for s in fixed for f in s]),
                                                                     np.max([f[1] for s in fixed for f in s])))
    np.testing.assert_array_equal(st[4], ref["stage_status"][4])
    np.testing.assert_array_equal(st[5], ref["stage_status"][5])
    same = np.nonzero(it[4] == ref["stage_iters"][4])[0]
    print("stage 3: iteration counts equal for %d / 16 sequences" % len(same))
    assert len(same) >= 0.9 * 16
    d3 = [_close(got["samples"][2, i, :120], ref["samples"][2, i, :120], 2) for i in same]
    print("stage 3: max |diff| positions %.2e, forces %.2e" % (max(d[0] for d in d3), max(d[1] for d in d3)))


def _kkt_residuals_ok(chd, b, i, p):
    """IPOPT's termination test at the final point of stage 3, residuals recomputed with the oracle's callbacks
    (as test_kkt_conditions_recomputed_independently)."""
    from oracle.phys import OracleProblem
    x, du, lay = b.get_x(), b.duals(), b.layout()
    o = OracleProblem(p)
    o.set_stage("3")
    n = o.n
    o.set_x(x[i, :n])
    sl = chd.phys.master_row_slices(b, i, lay)
    im, io = master_to_oracle_perm(sl, o)
    c, J, g = o.cons(), o.jac().tocsr(), o.grad()
    cl, cu = o.con_bounds()
    sc, sf = du["row_scale"][i], du["obj_scale"][i]
    y, zL, zU, s = du["y"][i], du["zL"][i], du["zU"][i], du["s"][i]
    nd = sum(len(d) - 1 for d in p.ee_durations)
    assert max(np.maximum(cl - c, c - cu).max(), (-x[i, n - nd:n]).max(), 0.0) <= 1e-4
    lam = np.zeros(o.m)
    lam[io] = (sc * y)[im]
    r = sf * g + J.T @ lam
    rows_dp = np.concatenate([np.arange(a, e) for nm, a, e in sl if nm == "durpos"])
    r[n - nd:n] += (sc * y)[rows_dp]
    r_tau = to_tau(r, duration_blocks(p, n))
    free = lay["var_kkt"][i, :n] >= 0
    rows_all = np.concatenate([im, rows_dp])
    lo, hi = lay["row_lo"][i, rows_all], lay["row_hi"][i, rows_all]
    ineq = lo != hi
    nbnd = int((lo[ineq] > -1e19).sum() + (hi[ineq] < 1e19).sum())
    s_d = max(100.0, (np.abs(y[rows_all]).sum() + (zL[rows_all][ineq] + zU[rows_all][ineq]).sum()) / (len(rows_all) + nbnd)) / 100.0
    assert np.abs(r_tau[free]).max() / s_d <= 1e-3
    cm = np.zeros(len(y))
    cm[im] = c[io]
    cm[rows_dp] = x[i, n - nd:n]
    ri = rows_all[ineq]
    assert np.abs(sc[ri] * cm[ri] - s[ri]).max() <= 1e-3
    lo_s, hi_s = lay["row_lo"][i, ri] * sc[ri], lay["row_hi"][i, ri] * sc[ri]
    relax = lambda v: 1e-8 * np.maximum(1.0, np.abs(v))
    hasl, hasu = lay["row_lo"][i, ri] > -1e19, lay["row_hi"][i, ri] < 1e19
    comp = np.concatenate([((s[ri] - (lo_s - relax(lo_s))) * zL[ri])[hasl], (((hi_s + relax(hi_s)) - s[ri]) * zU[ri])[hasu]])
    s_c = max(100.0, (zL[ri][hasl].sum() + zU[ri][hasu].sum()) / max(len(comp), 1)) / 100.0
    assert (comp >= 0).all() and comp.max() / s_c <= 1e-3
    assert np.abs(-y[ri] - zL[ri] + zU[ri]).max() / s_d <= 1e-3


def test_banded_above_limit_matches_oracle(chd):
    """200 frames, 4 feet, dense switches: more phase durations (113) than the dense border holds, so stage 3 runs only
    with banded switch times.  Compared with the CPU oracle, which keeps the durations in its own dense border; its
    staged solve takes 691 s of one CPU core, so its result is a golden file (tests/golden/make_stage3_band_golden.py).
    Assertions of test_dense_switch_long_horizon_matches_oracle, plus IPOPT's termination test recomputed with the
    oracle's callbacks when stage 3 converged on the GPU."""
    import os
    p = chd.synth.make_problem(0, n_frames=200, n_ee=4, dense=True)
    assert sum(len(d) - 1 for d in p.ee_durations) > 96
    b = chd.phys.PhysBatch([p], stage3_band_above=96)
    assert b.sizes_fixed()[0, 0] == b.sizes[0, 4] and b.sizes_fixed()[0, 2] > 96   # switch times are band unknowns
    out = b.solve()
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stage3_band", "oracle_dense200.npz"))
    ids = [str(k) for k in g["stage_ids"]]
    ref = {"stage_ids": ids, "success": g["success"], "durations": g["durations"],
           "stages": [{"status": int(a), "iters": int(i), "f": float(f)} for a, i, f in zip(g["status"], g["iters"], g["f"])]}
    print("GPU status %s iters %s" % (out["stage_status"][:, 0].tolist(), out["stage_iters"][:, 0].tolist()))
    print("oracle %s %s %s" % (ids, g["status"].tolist(), g["iters"].tolist()))
    assert (out["stage_status"][[0, 1, 2, 3], 0] == 0).all()
    # attempted, and not ended by a coupling outside the band the layout sized (that shows as -2, then stage 4 runs)
    assert out["stage_status"][4, 0] not in (-3, -2) and ref["stage_ids"][4] == "3"
    assert out["success"][0, 1] == 1 and ref["success"][1]
    stats = b.stage_stats()
    if out["stage_status"][4, 0] == 0 and ref["stages"][4]["status"] == 0:
        f_gpu, f_ref = stats[4, 0, 0], ref["stages"][4]["f"]
        assert abs(f_gpu - f_ref) <= 0.03 * abs(f_ref), (f_gpu, f_ref)
        assert stats[4, 0, 2] <= 1e-4
    nf = out["frames"][0]
    got, exp = out["samples"][2, 0, :nf], ref["durations"]
    assert np.abs(got[:, :3] - exp[:, :3]).max() < 0.02
    assert (got[:, 30:] != exp[:, 30:]).mean() < 0.02
    if out["stage_status"][4, 0] == 0:
        _kkt_residuals_ok(chd, b, 0, p)


def test_long_horizon_full_size_banded(chd):
    """test_long_horizon_full_size_properties's problems with banded switch times: stage 3 is attempted everywhere."""
    ps = [chd.synth.make_problem(s, n_frames=600, n_ee=4, dense=True) for s in range(2)]
    b = chd.phys.PhysBatch(ps, stage3_band_above=96)
    out = b.solve()
    st = out["stage_status"]
    print("stage status", st.tolist(), "iterations", out["stage_iters"].tolist())
    assert (st[[0, 1, 2, 3]] == 0).all(), st
    assert (st[4] != -3).all() and (st[4] != -9).all()
    assert (st[4] != -2).all()                          # no coupling left the band the layout sized
    assert ((st[4] == 0) == (st[5] == -9)).all()        # stage 4 runs exactly where stage 3 did not succeed
    assert (out["success"] == 1).all()
    x = b.get_x()
    for i, p in enumerate(ps):
        s = out["samples"][2, i, :600]
        pos, frc, flag = s[:, 6:18].reshape(600, 4, 3), s[:, 18:30].reshape(600, 4, 3), s[:, 30:34]
        nrm = np.asarray(p.floor_normal, float)
        nrm /= np.linalg.norm(nrm)
        assert np.abs(frc[flag == 0]).max() == 0.0
        assert np.isfinite(s).all() and np.abs(frc @ nrm).max() < 5000.0
        h = (pos - np.asarray(p.floor_point, float)) @ nrm
        assert np.abs(h[flag == 1]).max() <= 2e-4
        if st[4, i] != 0:
            continue
        n, T = int(b.sizes[i, 0]), sum(p.ee_durations[0])
        xo = n - sum(len(d) - 1 for d in p.ee_durations)
        for d0 in p.ee_durations:
            d = x[i, xo:xo + len(d0) - 1]
            xo += len(d0) - 1
            assert (d >= -1e-4).all()
            assert d.sum() <= T + 1e-4                     # the last phase (T - sum) is not negative either
            tau, tau0 = np.cumsum(d), np.cumsum(np.asarray(d0[:-1], float))
            assert np.abs(tau - tau0).max() <= TRUST + 1e-6
