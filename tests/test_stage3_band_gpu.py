"""GPU tests of banded switch times (`PhysBatch(stage3_band_above=...)`): the same problems solved with the switch
times in the dense border and in the band, and -- above the dense border's limit of 96 phase durations -- a 200-frame
densely switching gait against the CPU oracle and the long-horizon configuration at full size."""
import numpy as np
import pytest

from tests.util import assert_ipopt_termination, assert_loosely_close, assert_solves_agree

pytestmark = pytest.mark.gpu

TRUST = 0.04   # CHD_TAU_TRUST [s]


def test_banded_and_border_forms_agree(chd):
    """Benchmark seeds (2 feet) with every sequence's switch times banded (0) against the default dense border."""
    ps = [chd.synth.make_problem(s, n_ee=2) for s in range(16)]
    ref = chd.phys.PhysBatch(ps).solve()
    bb = chd.phys.PhysBatch(ps, stage3_band_above=0)
    assert (bb.sizes_fixed()[:, 0] == bb.sizes[:, 4]).all()        # no switch time in the border
    assert_solves_agree(ref, bb.solve(), 2)


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
    assert_loosely_close(out["samples"][2, 0, :nf], ref["durations"], 4)
    if out["stage_status"][4, 0] == 0:
        assert_ipopt_termination(chd, b, 0, p, "3")


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
    _, pc, fc, cc = chd.phys.sample_columns(4, 4)
    for i, p in enumerate(ps):
        s = out["samples"][2, i, :600]
        pos, frc, flag = s[:, pc].reshape(600, 4, 3), s[:, fc].reshape(600, 4, 3), s[:, cc]
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
