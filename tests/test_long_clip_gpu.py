"""GPU tests of clips whose iterate is longer than the evaluation and line-search kernels can hold in shared memory
(n_max > 14 208 at 227 KB of opt-in shared memory; tests/test_long_clip_cpu.py checks the sizes): batch creation takes
them and runs the global-memory form of chd_k_eval / chd_k_linesearch.  The long clip is 1100 frames of a 4-foot walk
(`chd.synth.make_problem(0, n_frames=1100, n_ee=4)`, n = 15 240, 338 phase durations: stage 3 is not attempted, stage 4
runs), checked against the CPU oracle's staged solve (tests/golden/make_long_clip_golden.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.util import (assert_ipopt_termination, assert_loosely_close, assert_samples_close, assert_solves_agree,
                        master_to_oracle_perm)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "long_clip", "oracle_walk1100.npz")
FRAMES, N_EE = 1100, 4
SMEM_N_MAX = 14208
RTOL = 1e-10


def _long(chd):
    return chd.synth.make_problem(0, n_frames=FRAMES, n_ee=N_EE)


@pytest.fixture(scope="module")
def solved(chd):
    """The 16 benchmark seeds (120 frames, 2 feet) solved alone (shared-memory form) and with the long clip appended
    (the batch's n_max then selects the global-memory form for all 17 sequences)."""
    short = [chd.synth.make_problem(s, n_ee=2) for s in range(16)]
    alone = chd.phys.PhysBatch(short)
    assert alone.dims["n_max"] <= SMEM_N_MAX
    mixed = chd.phys.PhysBatch(short + [_long(chd)])
    assert mixed.dims["n_max"] > SMEM_N_MAX
    return alone, alone.solve(), mixed, mixed.solve()


def test_batch_creation_past_the_shared_memory_limit(chd):
    """Failed with -5 ("problem too large for the shared-memory staged kernels") before the global-memory form."""
    for p in (_long(chd), chd.synth.make_problem(0, n_frames=700, n_ee=4, dense=True)):
        b = chd.phys.PhysBatch([p])
        assert b.dims["n_max"] > SMEM_N_MAX
        ev = b.eval("2.2")
        assert np.isfinite(ev["cost"]).all() and np.isfinite(ev["grad"]).all()
        b.close()


@pytest.mark.parametrize("stage", ["1.2", "2.1", "2.2"])
def test_long_clip_eval_parity(chd, stage):
    """cost / gradient / constraint values / Jacobian of the global-memory evaluation kernel against the oracle at two
    random points, as tests/test_phys_gpu.py::test_eval_parity."""
    from oracle.phys import OracleProblem
    p = _long(chd)
    b = chd.phys.PhysBatch([p])
    lay = b.layout()
    o = OracleProblem(p)
    n = int(b.sizes[0, 0])
    nd = sum(len(d) - 1 for d in p.ee_durations)
    free = lay["var_kkt"][0, :n] >= 0
    free[n - nd:] = False
    rng = np.random.default_rng(321)
    x0 = b.get_x()
    for _ in range(2):
        x = x0.copy()
        x[0, :n] += np.where(free, rng.normal(0, 0.01, n), 0.0)
        b.set_x(x)
        ev = b.eval(stage)
        o.set_stage(stage)
        no = o.n
        o.set_x(x[0, :no])
        np.testing.assert_allclose(ev["cost"][0], o.cost(), rtol=RTOL)
        go = o.grad()
        np.testing.assert_allclose(ev["grad"][0, :no], go, rtol=RTOL, atol=RTOL * np.abs(go).max())
        assert (ev["grad"][0, no:n] == 0).all()
        sl = chd.phys.master_row_slices(b, 0, lay)
        im, io = master_to_oracle_perm(sl, o)
        assert len(io) == o.m
        co = o.cons()
        np.testing.assert_allclose(ev["g"][0, im], co[io], rtol=RTOL, atol=RTOL * max(1.0, np.abs(co).max()))
        J = b.jac_csr(0, ev["jac"], lay).tocsr()[im][:, :no]     # sparse: the dense Jacobian would take 1.7 GB
        Jo = o.jac().tocsr()[io]
        assert J.shape == Jo.shape
        assert np.abs((J - Jo).data).max(initial=0.0) <= RTOL * np.abs(Jo.data).max()


def test_shared_and_global_forms_agree(solved):
    """The benchmark seeds solved by the shared-memory form (alone) and by the global-memory form (long clip appended):
    the same algorithm with the same arithmetic, up to the order of the gradient's atomic additions."""
    _, ref, mixed, got = solved
    assert_solves_agree(ref, got, 2, n_ee_max=mixed.n_ee_max)


def test_long_clip_matches_oracle(chd, solved):
    """The long clip (in the batch of test_shared_and_global_forms_agree, index 16) against the oracle's staged solve:
    1.1, 1.2, 2.1, 2.2, then 4 (more than 96 phase durations: stage 3 is not attempted on either side)."""
    _, _, b, out = solved
    i = 16
    p = _long(chd)
    g = np.load(GOLDEN)
    ids = [str(k) for k in g["stage_ids"]]
    assert ids == ["1.1", "1.2", "2.1", "2.2", "4"]
    st, it = out["stage_status"][:, i], out["stage_iters"][:, i]
    print("GPU status %s iters %s" % (st.tolist(), it.tolist()))
    print("oracle %s %s %s (%.0f s)" % (ids, g["status"].tolist(), g["iters"].tolist(), float(g["seconds"])))
    assert st[chd.phys.STAGES["3"]] == -3
    assert [int(st[chd.phys.STAGES[k]]) for k in ids] == [int(v) for v in g["status"]]
    for k in range(4):
        assert int(it[chd.phys.STAGES[ids[k]]]) == int(g["iters"][k]), (ids[k], it.tolist(), g["iters"].tolist())
    nf = out["frames"][i]
    assert nf == FRAMES
    for snap, key in enumerate(["no_dynamics", "dynamics"]):
        dp, df = assert_samples_close(out["samples"][snap, i, :nf], g[key], N_EE)
        print("%s: max |diff| positions %.2e, forces %.2e" % (key, dp, df))
    # stage 4 replaces stage 3: the loose check of a stage that takes its own path on either side
    print("stage 4: iterations GPU %d oracle %d" % (it[chd.phys.STAGES["4"]], g["iters"][4]))
    dcom = assert_loosely_close(out["samples"][2, i, :nf], g["durations"], N_EE)
    print("stage 4: max |diff| COM %.2e" % dcom)
    assert out["success"][i].tolist() == [int(v) for v in g["success"]]
    if st[chd.phys.STAGES["4"]] == 0:
        assert_ipopt_termination(chd, b, i, p, "4")


def test_long_clip_through_phys_optim_files(chd, tmp_path):
    """The long clip's four input files -> scripts/phys_optim.py -> the output files -> chd.prepare.load_results."""
    p = _long(chd)
    ind, outd = str(tmp_path / "phys_optim_in"), str(tmp_path / "phys_optim_out")
    os.makedirs(outd)
    chd.io_formats.write_phys_inputs(p, ind)
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "phys_optim.py"), "--in_dir", ind,
                           "--nframes", str(FRAMES), "--out_dir", outd])
    r = chd.prepare.load_results(outd)
    assert set(r) == {"no_dynamics", "dynamics", "durations", "success"}
    g = np.load(GOLDEN)
    for key in ("no_dynamics", "dynamics", "durations"):
        assert r[key]["num_frames"] == FRAMES and r[key]["num_feet"] == N_EE
        assert all(np.isfinite(np.asarray(v, float)).all() for v in r[key].values() if isinstance(v, np.ndarray))
        assert np.abs(r[key]["base_lin"] - g[key][:, :3]).max() < 0.02
    assert r["success"] == {"dynamics": int(g["success"][0]), "durations": int(g["success"][1])}
