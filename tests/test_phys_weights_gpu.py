"""GPU tests of per-clip cost weights and of the cost terms (chd_phys_cost_terms, `solve(cost_terms=True)`): a list of
equal tuples is the scalar argument; in a batch of mixed weights each clip solves as in a batch that gives every clip
its weights; the CPU oracle agrees with non-default weights; the ten terms weight up to the evaluated cost and agree
with the oracle's, bitwise repeatably; a queue (refills included) and two processes sharing one counter return every
clip's terms; weight_sweep.py writes its rows and files."""
import json
import os
import sys

import numpy as np
import pytest

from tests.test_phys_weights_cpu import SETTINGS, oracle_cost_terms
from tests.util import assert_loosely_close, assert_samples_close, assert_solves_agree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clips(chd, seed0=300, n=4):
    return [chd.synth.make_problem(seed0 + i, n_frames=60 + 20 * i, n_ee=2) for i in range(n)]


def _same_loop(ra, rb):
    """two solves ran the same number of schedule iterations when every stage's iteration counts agree (stage 3's may
    differ from run to run: shared-memory fp64 atomics)"""
    return (ra["stage_iters"] == rb["stage_iters"]).all() and (ra["stage_status"] == rb["stage_status"]).all()


def test_uniform_list_is_the_scalar(chd):
    """A list of equal tuples gives what the scalar argument gives, with the same launches; asking for the terms adds
    exactly one launch (chd_k_cost_terms), whose result is chd_phys_cost_terms at the final iterate."""
    ps = _clips(chd, 10, 6)
    a = chd.phys.PhysBatch(ps, weights=SETTINGS[1])
    b = chd.phys.PhysBatch(ps, weights=[SETTINGS[1]] * len(ps))
    for s in ("2.1", "2.2"):                                          # deterministic stages: launches equal
        sa, sb = a.solve_stage(s), b.solve_stage(s)
        np.testing.assert_array_equal(sa["iters"], sb["iters"])
    assert a.launch_count() == b.launch_count()
    a.reset(), b.reset()
    n0 = a.launch_count()
    ra, rb = a.solve(), b.solve()
    np.testing.assert_array_equal(ra["stage_status"], rb["stage_status"])
    np.testing.assert_array_equal(ra["stage_iters"][:4], rb["stage_iters"][:4])
    assert_solves_agree(ra, rb, 2)
    if _same_loop(ra, rb):
        assert a.launch_count() == b.launch_count()
    a.reset()
    n1 = a.launch_count()
    rt = a.solve(cost_terms=True)
    if _same_loop(ra, rt):
        assert a.launch_count() - n1 == (n1 - 1 - n0) + 1
    assert rt["cost_terms"].tobytes() == a.cost_terms().tobytes()
    assert rt["cost_terms"].shape == (len(ps), 10) and (rt["cost_terms"][:, :9] > 0).all()


def test_mixed_weights_match_uniform_batches(chd):
    """4 clips x 4 settings in one batch: clip k as in a batch of the same clips that all use setting k."""
    ps = _clips(chd)
    mixed = chd.phys.PhysBatch(ps, weights=SETTINGS).solve()
    for k, w in enumerate(SETTINGS):
        ref = chd.phys.PhysBatch(ps, weights=w).solve()
        np.testing.assert_array_equal(mixed["stage_status"][:4, k], ref["stage_status"][:4, k])
        np.testing.assert_array_equal(mixed["stage_iters"][:4, k], ref["stage_iters"][:4, k])
        nf = ref["frames"][k]
        for snap in (0, 1):
            assert_samples_close(mixed["samples"][snap, k, :nf], ref["samples"][snap, k, :nf], 2)
        assert_loosely_close(mixed["samples"][2, k, :nf], ref["samples"][2, k, :nf], 2)


def test_oracle_with_non_default_weights(chd):
    """w_com_ang = 0.5, w_ee = 1.0, w_dur = 1.0: the same stage statuses and stage 1.1-2.2 iterations as the oracle, the
    same trajectories after stages 1.2 and 2.2, and the final one loosely."""
    from oracle.phys import OracleProblem
    w = (0.4, 0.5, 1.0, 0.1, 1.0)
    ps = [chd.synth.make_problem(s, n_frames=90, n_ee=2) for s in (1, 2)]
    out = chd.phys.PhysBatch(ps, weights=[w] * 2).solve()
    for i, p in enumerate(ps):
        ref = OracleProblem(p, weights=w).solve()
        st, it = out["stage_status"][:, i], out["stage_iters"][:, i]
        assert [s["status"] for s in ref["stages"]] == [int(st[chd.phys.STAGES[k]]) for k in ref["stage_ids"]]
        for k, s in zip(ref["stage_ids"], ref["stages"]):
            if k in ("1.1", "1.2", "2.1", "2.2"):
                assert s["iters"] == it[chd.phys.STAGES[k]], k
        nf = out["frames"][i]
        for snap, name in enumerate(("no_dynamics", "dynamics")):
            print("clip %d %s: max |diff| positions %.2e, forces %.2e" % ((i, name) + assert_samples_close(
                out["samples"][snap, i, :nf], ref[name], 2)))
        # stage 3 takes its own path on the GPU (fp64 atomics in shared memory, DESIGN §3, §7)
        print("clip %d durations: COM within %.2e" % (i, assert_loosely_close(out["samples"][2, i, :nf], ref["durations"], 2)))


@pytest.mark.parametrize("n_ee", [2, 4])
def test_terms_weight_up_to_the_cost_and_match_the_oracle(chd, n_ee):
    """At random points (stage 3 with moved durations too) and in every stage: the stage's weights times the ten terms
    add up to chd_phys_eval's cost, each term is the oracle's, and two calls give the same bits."""
    from oracle.phys import OracleProblem
    ps = [chd.synth.make_problem(40 + i, n_frames=50 + 10 * i, n_ee=n_ee) for i in range(3)]
    b = chd.phys.PhysBatch(ps, weights=SETTINGS[1:4])
    sw = b.stage_weights()
    rng = np.random.default_rng(8)
    x = b.get_x()
    for i, p in enumerate(ps):
        n, nd = b.sizes[i, 0], sum(len(d) - 1 for d in p.ee_durations)
        x[i, :n - nd] += rng.normal(0, 0.005, n - nd)
        x[i, n - nd:n] += rng.uniform(-0.01, 0.01, nd)
    b.set_x(x)
    t = b.cost_terms()
    assert t.tobytes() == b.cost_terms().tobytes()
    for name, st in chd.phys.STAGES.items():
        ev = b.eval(name)
        np.testing.assert_allclose((t * sw[:, st]).sum(axis=1), ev["cost"], rtol=1e-12)
    assert t.tobytes() == b.cost_terms().tobytes()
    for i, p in enumerate(ps):
        o = OracleProblem(p, weights=SETTINGS[1 + i])
        for name in ("3", "2.2"):                                    # stage 3 first: 2.2 keeps its durations
            o.set_stage(name)
            o.set_x(x[i, :o.n])
            ot = oracle_cost_terms(o, sw[i, chd.phys.STAGES[name]])
            have = ~np.isnan(ot)
            np.testing.assert_allclose(t[i, have], ot[have], rtol=1e-10, err_msg=name)


def test_queue_refills_with_other_weights(chd):
    """6 clips with different weights through 2 slots: each clip's stages 1.1-2.2 as in the mixed batch, and its terms
    returned in its place (those of the batch where stages 3 and 4 took the same path)."""
    ps = _clips(chd, 500, 6)
    W = [SETTINGS[i % 4] for i in range(6)]
    ref = chd.phys.PhysBatch(ps, weights=W).solve(cost_terms=True)
    got = chd.phys.PhysQueue(ps, 2, weights=W).solve(cost_terms=True)
    np.testing.assert_array_equal(got["stage_status"][:4], ref["stage_status"][:4])
    np.testing.assert_array_equal(got["stage_iters"][:4], ref["stage_iters"][:4])
    for i in range(6):
        nf = ref["frames"][i]
        assert_samples_close(got["samples"][1, i, :nf], ref["samples"][1, i, :nf], 2)
        same = (got["stage_status"][:, i] == ref["stage_status"][:, i]).all() and got["stage_iters"][4, i] == ref["stage_iters"][4, i]
        if same:
            np.testing.assert_allclose(got["cost_terms"][i], ref["cost_terms"][i], rtol=1e-4, atol=1e-9)
    assert (got["cost_terms"][:, :9] > 0).all()


def _two_ranks(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = _clips(chd, 600, 8)
    store = dist.FileStore(os.path.join(tmp, "claims"), world)
    s = chd.parallel.ShardedSolver(ps, weights=[SETTINGS[i % 4] for i in range(8)], device=0, rank=rank, world=world,
                                   slots=2, store=store, tensor_device=torch.device("cpu"))
    try:
        out = s.solve(cost_terms=True)
    finally:
        s.close()
    np.savez(os.path.join(tmp, "r%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    dist.destroy_process_group()


def test_two_processes_merge_the_terms(chd, tmp_path):
    import torch.multiprocessing as mp
    port = 38500 + (os.getpid() % 2000)
    mp.spawn(_two_ranks, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "r0.npz")), np.load(str(tmp_path / "r1.npz"))
    for k in r0.files:
        assert r0[k].tobytes() == r1[k].tobytes(), k
    assert r0["solved"].all()
    ps = _clips(chd, 600, 8)
    W = [SETTINGS[i % 4] for i in range(8)]
    ref = chd.phys.PhysQueue(ps, 2, weights=W).solve(cost_terms=True)
    np.testing.assert_array_equal(r0["stage_iters"][:4], ref["stage_iters"][:4])
    for i in range(8):
        if (r0["stage_status"][:, i] == ref["stage_status"][:, i]).all() and r0["stage_iters"][4, i] == ref["stage_iters"][4, i]:
            np.testing.assert_allclose(r0["cost_terms"][i], ref["cost_terms"][i], rtol=1e-4, atol=1e-9)
    assert (r0["cost_terms"][:, :9] > 0).all()


def test_weight_sweep_script(chd, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import weight_sweep
    p = chd.synth.make_problem(3, n_frames=60, n_ee=2)
    clip = str(tmp_path / "clip")
    os.makedirs(clip)
    chd.io_formats.write_phys_inputs(p, clip)
    res, od = str(tmp_path / "sweep.json"), str(tmp_path / "out")
    weight_sweep.main(["--in_dir", clip, "--nframes", "60", "--n_ee", "2", "--w_ee", "0.3,1", "--w_dur", "0.1,1",
                       "--slots", "2", "--results", res, "--out_dir", od])
    rows = json.load(open(res))
    assert len(rows) == 4 and [(r["w_ee"], r["w_dur"]) for r in rows] == [(0.3, 0.1), (0.3, 1.0), (1.0, 0.1), (1.0, 1.0)]
    for r in rows:
        assert all(r[t] >= 0 for t in chd.phys.COST_TERMS) and r["status_1.1"] == 0
        d = os.path.join(od, "clip", "setting_%d" % r["setting"])
        assert sorted(os.listdir(d)) == sorted(list(chd.phys.SOLUTION_FILES) + ["success_log.txt"])
