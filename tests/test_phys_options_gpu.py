"""GPU tests of per-clip solver options (`chd.phys.SolverOptions`): explicit defaults are the default solve; in a batch,
a queue and two processes sharing one claim counter every clip solves as with its options alone; a clip stopped after
`no_dynamics` or `dynamics` keeps its earlier stages and frees its queue slot at once; converged stages meet each clip's
own tolerances; a capped stage ends at its cap and the schedule goes on.

Two solves of the same clips can differ in the last bits of their snapshots (fp64 atomics, DESIGN §3, §7): statuses and
stage 1.1-2.2 iteration counts are compared exactly, NaN snapshots bit for bit, the other snapshots within
`assert_samples_close`'s tolerances (stage 3 and 4 within `assert_loosely_close`'s)."""
import os
import sys

import numpy as np
import pytest

from tests.util import assert_loosely_close, assert_samples_close, assert_solves_agree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clips(chd, seed0=700, n=4):
    return [chd.synth.make_problem(seed0 + i, n_frames=60 + 20 * i, n_ee=2) for i in range(n)]


def _mixed(chd, n):
    S = chd.phys.SolverOptions
    base = [S(last_stage="no_dynamics"), S(tol=1e-2), S(last_stage="dynamics", constr_viol_tol=1e-5),
            S(max_iter=(0, 0, 4, 0, 0, 0)), S(tol=1e-4, compl_inf_tol=1e-5)]
    return [base[i % len(base)] for i in range(n)]


def _early(out, i):
    """1 + the stage id after which clip i's schedule ended early, else None"""
    st = out["stage_status"][:, i]
    return None if st[4] != -9 else (2 if st[2] == -9 else 4)


def _assert_snaps_same(got, ref, n_ee=2):
    """two stacks of snapshot rows: NaN in the same places and bit for bit there (a snapshot not taken), the rest
    within assert_samples_close's tolerances (two solves of the same clips can differ in the last bits)"""
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(got), nan)
    assert got[nan].tobytes() == ref[nan].tobytes()
    for g, r in zip(got.reshape(-1, *got.shape[-2:]), ref.reshape(-1, *ref.shape[-2:])):
        if not np.isnan(r).all():
            assert_samples_close(g, r, n_ee)


def _assert_clip_same(got, ref, i, j=None, n_ee=2):
    """clip i of `got` is clip j of `ref`: equal statuses and iterations of stages 1.1-2.2 and the first two snapshots
    (NaN included); a clip that stopped early equal in every status and snapshot; otherwise stages 3 and 4 as
    assert_loosely_close."""
    j = i if j is None else j
    np.testing.assert_array_equal(got["stage_status"][:4, i], ref["stage_status"][:4, j])
    np.testing.assert_array_equal(got["stage_iters"][:4, i], ref["stage_iters"][:4, j])
    assert got["frames"][i] == ref["frames"][j]
    nf = ref["frames"][j]
    _assert_snaps_same(got["samples"][:2, i, :nf], ref["samples"][:2, j, :nf], n_ee)
    if _early(ref, j) is not None:
        _assert_snaps_same(got["samples"][:, i, :nf], ref["samples"][:, j, :nf], n_ee)
        np.testing.assert_array_equal(got["stage_status"][:, i], ref["stage_status"][:, j])
        np.testing.assert_array_equal(got["success"][i], ref["success"][j])
    else:
        np.testing.assert_array_equal(got["stage_status"][4, i], ref["stage_status"][4, j])
        assert_loosely_close(got["samples"][2, i, :nf], ref["samples"][2, j, :nf], n_ee)


def test_explicit_defaults_are_the_default_solve(chd):
    """SolverOptions() for every clip gives the solve without options: a batch and a queue (2 slots)."""
    ps = _clips(chd, 10, 5)
    P = chd.phys
    a = P.PhysBatch(ps).solve(cost_terms=True)
    b = P.PhysBatch(ps, options=P.SolverOptions()).solve(cost_terms=True)
    assert_solves_agree(a, b, 2)
    for i in range(len(ps)):
        _assert_clip_same(b, a, i)
        if (a["stage_iters"][:, i] == b["stage_iters"][:, i]).all():
            np.testing.assert_allclose(b["cost_terms"][i], a["cost_terms"][i], rtol=1e-4, atol=1e-9)
    qa = P.PhysQueue(ps, 2).solve()
    qb = P.PhysQueue(ps, 2, options=[P.SolverOptions()] * len(ps)).solve()
    assert_solves_agree(qa, qb, 2)
    for i in range(len(ps)):
        _assert_clip_same(qb, qa, i)


def test_mixed_options_match_uniform_batches(chd):
    """5 clips with 5 option records in one batch, and in a queue of 2 slots: clip k as in a batch of the same clips
    that all use record k."""
    P = chd.phys
    ps = _clips(chd, 720, 5)
    opts = _mixed(chd, 5)
    mixed = P.PhysBatch(ps, options=opts).solve()
    queue = P.PhysQueue(ps, 2, options=opts).solve()
    assert queue["solved"].all()
    for k, o in enumerate(opts):
        ref = P.PhysBatch(ps, options=o).solve()
        _assert_clip_same(mixed, ref, k)
        _assert_clip_same(queue, ref, k)
    # the records as the solver resolved them
    got = P.PhysBatch(ps, options=opts).solver_options()
    assert [g.last_stage for g in got] == [o.last_stage for o in opts] and got[3].max_iter[2] == 4


def test_last_stage_keeps_the_earlier_stages(chd):
    """A clip stopped after no_dynamics / dynamics: the statuses, iterations and snapshots of the stages it ran are
    those of the full run, its later stages report -9 and 0 iterations, its later snapshots are NaN and its success flags
    0 for the stages it did not run."""
    P = chd.phys
    ps = _clips(chd, 740, 3)
    full = P.PhysBatch(ps).solve()
    for last, ran in (("no_dynamics", 2), ("dynamics", 4)):
        out = P.PhysBatch(ps, options=P.SolverOptions(last_stage=last)).solve()
        k = P.LAST_STAGES.index(last)
        _assert_snaps_same(out["samples"][:k + 1], full["samples"][:k + 1])
        assert np.isnan(out["samples"][k + 1:]).all()
        np.testing.assert_array_equal(out["stage_status"][:ran], full["stage_status"][:ran])
        np.testing.assert_array_equal(out["stage_iters"][:ran], full["stage_iters"][:ran])
        assert (out["stage_status"][ran:] == -9).all() and (out["stage_iters"][ran:] == 0).all()
        np.testing.assert_array_equal(out["success"][:, 0], full["success"][:, 0] if ran == 4 else 0)
        assert (out["success"][:, 1] == 0).all()


def test_stopped_clip_frees_its_slot_at_once(chd):
    """A queue of 2 slots: the longest clip runs the whole schedule in one slot while three short clips stopped after
    no_dynamics pass through the other one, so the queue takes no longer than the long clip; its results are those of
    the long clip alone."""
    P = chd.phys
    S = P.SolverOptions
    ps = [chd.synth.make_problem(760, n_frames=160, n_ee=2)] + [chd.synth.make_problem(761 + i, n_frames=40, n_ee=2)
                                                                for i in range(3)]
    opts = [S()] + [S(last_stage="no_dynamics")] * 3
    q = P.PhysQueue(ps, 2, options=opts)
    assert q.order[0] == 0
    out = q.solve()
    loop = q.kernel_times()["kkt"][1]                                        # one KKT launch per schedule iteration
    it = out["stage_iters"].astype(int)
    long_clip = int(it[:, 0].sum()) + 2 * 6
    print("queue iterations %d, long clip %d, short clips %s" % (loop, long_clip, it[:, 1:].sum(axis=0).tolist()))
    assert int(it[:, 1:].sum()) + 3 * 2 * 2 < long_clip                      # the short clips fit beside the long one
    assert loop <= long_clip + 16                                            # refills happen at check points, every 8
    assert (out["stage_status"][2:, 1:] == -9).all()
    alone = P.PhysBatch(ps, options=opts).solve()
    for i in range(4):
        _assert_clip_same(out, alone, i)


def test_converged_stages_meet_each_clips_tolerances(chd):
    """tol 1e-2, the default and 1e-4 side by side on the same clips: every converged stage's scaled error, constraint
    violation and dual infeasibility are within its clip's own tolerances."""
    P = chd.phys
    S = P.SolverOptions
    base = _clips(chd, 780, 2)
    ps = [p for p in base for _ in range(3)]
    opts = [S(tol=1e-2), S(), S(tol=1e-4, constr_viol_tol=1e-5, dual_inf_tol=1e-1)] * 2
    b = P.PhysBatch(ps, options=opts)
    out = b.solve()
    stats = b.stage_stats()
    checked = 0
    for i, o in enumerate(opts):
        for s in range(6):
            if out["stage_status"][s, i] == 0:
                E0, viol, dual = stats[s, i, 1:4]
                assert E0 <= o.tol and viol <= o.constr_viol_tol and dual <= o.dual_inf_tol, (i, s, E0, viol, dual)
                checked += 1
    assert checked >= 4 * len(opts)
    print("stage 1.1-2.2 iterations at tol 1e-2 / 1e-3 / 1e-4:", out["stage_iters"][:4].sum(axis=0).reshape(2, 3).tolist())


def test_capped_stage_goes_on_like_a_capped_stage(chd):
    """Stage 2.1 capped at 4: it ends with status -1 after 4 iterations and stages 2.2 onwards follow, as in the
    stage-by-stage solve with the same cap (chd_phys_solve_stage's override)."""
    P = chd.phys
    ps = _clips(chd, 800, 3)
    out = P.PhysBatch(ps, options=P.SolverOptions(max_iter=(0, 0, 4, 0, 0, 0))).solve()
    assert (out["stage_status"][2] == -1).all() and (out["stage_iters"][2] == 4).all()
    assert (out["stage_status"][3] != -9).all() and (out["stage_status"][4] != -9).all()
    step = P.PhysBatch(ps)
    for name, cap in (("1.1", 0), ("1.2", 0), ("2.1", 4), ("2.2", 0)):
        r = step.solve_stage(name, max_iter=cap)
        np.testing.assert_array_equal(r["status"], out["stage_status"][P.STAGES[name]])
        np.testing.assert_array_equal(r["iters"], out["stage_iters"][P.STAGES[name]])
    smp, frames = step.sample()
    for i in range(3):
        nf = frames[i]
        assert_samples_close(out["samples"][1, i, :nf], smp[i, :nf], 2)


def _two_ranks(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = _clips(chd, 820, 6)
    store = dist.FileStore(os.path.join(tmp, "claims"), world)
    s = chd.parallel.ShardedSolver(ps, device=0, rank=rank, world=world, slots=2, store=store,
                                   tensor_device=torch.device("cpu"), options=_mixed(chd, 6))
    try:
        out = s.solve()
    finally:
        s.close()
    np.savez(os.path.join(tmp, "r%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    dist.destroy_process_group()


def test_two_processes_merge_every_clips_options(chd, tmp_path):
    """Two processes claiming from one counter: both return the same bytes, and every clip is what one queue with the
    same options computes, its NaN snapshots bit for bit."""
    import torch.multiprocessing as mp
    port = 39500 + (os.getpid() % 2000)
    mp.spawn(_two_ranks, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "r0.npz")), np.load(str(tmp_path / "r1.npz"))
    for k in r0.files:
        assert r0[k].tobytes() == r1[k].tobytes(), k
    assert r0["solved"].all()
    ps = _clips(chd, 820, 6)
    ref = chd.phys.PhysQueue(ps, 2, options=_mixed(chd, 6)).solve()
    got = {k: r0[k] for k in r0.files}
    early = [i for i in range(6) if _early(ref, i) is not None]
    assert early and all(np.isnan(got["samples"][2, i]).all() for i in early)
    for i in range(6):
        _assert_clip_same(got, ref, i)
