"""GPU tests of the claim source of the physics solve queue (`PhysQueue(claim=...)`, `chd_phys_queue_set_claim`) and
of `ShardedSolver(slots=...)`: clips handed out in any chunks and any order give, clip by clip, the results of a queue
in its own order; a source that runs dry leaves the rest unsolved; a failing source fails the solve and leaves the handle
usable; two processes sharing one GPU and one FileStore counter solve every clip once and merge to the one-process
result, and rank 0 writes the files the one-process run writes."""
import os
import sys

import numpy as np
import pytest

from tests.util import assert_samples_close, assert_solves_agree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mixed(chd, n, seed0):
    F = [40 + (29 * i) % 81 for i in range(n)]                     # 40 .. 120 frames
    return [chd.synth.make_problem(seed0 + i, n_frames=f, n_ee=2) for i, f in enumerate(F)]


class _Back:
    """Hands out the last `want` positions not handed out yet (at most `stop` in all), recording every chunk."""

    def __init__(self, n, stop=None):
        self.n, self.stop, self.chunks = n, n if stop is None else stop, []

    def __call__(self, want):
        k = min(want, self.stop - sum(self.chunks))
        self.chunks.append(k)
        return self.n - sum(self.chunks), k


def test_irregular_chunks_match_own_order(chd):
    """The library asks for as many positions as slots have finished at a check point, so the chunks are as uneven
    as the clips' finishing times (4 at the start, then 1, 3, 2, ...); served from the back of the queue they still
    give every clip the result of the queue in its own order."""
    ps = _mixed(chd, 14, 100)
    ref = chd.phys.PhysQueue(ps, 4).solve()
    src = _Back(len(ps))
    got = chd.phys.PhysQueue(ps, 4, claim=src).solve()
    print("chunks", src.chunks)
    assert src.chunks[0] == 4 and sum(src.chunks) == len(ps) and len(src.chunks) > 2
    assert got["solved"].all() and ref["solved"].all()
    assert_solves_agree(ref, got, 2)
    np.testing.assert_array_equal(got["frames"], ref["frames"])
    np.testing.assert_array_equal(got["success"], ref["success"])


def test_source_that_stops_leaves_the_rest_unsolved(chd):
    ps = _mixed(chd, 12, 200)
    N = len(ps)
    ref = chd.phys.PhysQueue(ps, 3).solve()
    handed = []

    def first_half(want):
        f = sum(handed)
        k = min(want, N // 2 - f)
        handed.append(k)
        return f, k

    q = chd.phys.PhysQueue(ps, 3, claim=first_half)
    got = q.solve()                                                   # returns normally: rc 0
    mine = np.sort(q.order[:N // 2])                                  # the first N/2 queue positions, as input clips
    rest = np.setdiff1d(np.arange(N), mine)
    np.testing.assert_array_equal(np.nonzero(got["solved"])[0], mine)
    a, b = chd.phys.take_clips(ref, mine), chd.phys.take_clips(got, mine)
    assert_solves_agree(a, b, 2)
    np.testing.assert_array_equal(b["frames"], a["frames"])
    np.testing.assert_array_equal(b["success"], a["success"])
    assert (got["frames"][rest] == 0).all() and (got["samples"][:, rest] == 0).all()
    assert (got["stage_iters"][:, rest] == 0).all()


def test_failing_source_fails_the_solve_and_the_handle_still_solves(chd):
    """-1 from the source at the first refill, a range beyond n at the start and a position handed out twice at the
    first refill each make the solve fail (code -1); the next solve on the same handle is the queue's own result."""
    ps = _mixed(chd, 6, 300)
    N = len(ps)
    ref = chd.phys.PhysQueue(ps, 2).solve()
    mode = {"m": None, "calls": 0, "next": 0}

    def claim(want):
        mode["calls"] += 1
        m, first_call = mode["m"], mode["calls"] == 1
        if m == "negative" and not first_call:
            return 0, -1
        if m == "range" and first_call:
            return N - 1, want
        if m == "twice" and not first_call:
            return 0, want
        f = mode["next"]
        k = min(want, N - f)
        mode["next"] += k
        return f, k

    q = chd.phys.PhysQueue(ps, 2, claim=claim)
    for m in ("negative", "range", "twice"):
        mode.update(m=m, calls=0, next=0)
        with pytest.raises(RuntimeError, match="code -1"):
            q.solve()
        assert mode["calls"] == (1 if m == "range" else 2), m
    mode.update(m=None, calls=0, next=0)
    got = q.solve()
    assert got["solved"].all()
    assert_solves_agree(ref, got, 2)
    np.testing.assert_array_equal(got["frames"], ref["frames"])
    np.testing.assert_array_equal(got["success"], ref["success"])


def _two_ranks(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import torch
    import torch.distributed as dist
    import chd
    import phys_optim
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = _mixed(chd, 16, 400)
    store = dist.FileStore(os.path.join(tmp, "claims"), world)
    s = chd.parallel.ShardedSolver(ps, device=0, rank=rank, world=world, slots=4, store=store,
                                   tensor_device=torch.device("cpu"))
    try:
        out = s.solve()
    finally:
        s.close()
    np.savez(os.path.join(tmp, "r%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    if rank == 0:
        dirs = [os.path.join(tmp, "rank0", "c%d" % i) for i in range(len(ps))]
        for d in dirs:
            os.makedirs(d)
        phys_optim.write_results(out, ps, dirs, 2)
    dist.destroy_process_group()


def _rows(chd, path):
    r = chd.io_formats.read_solution(path)
    n = r["num_frames"]
    cat = lambda a: a.transpose(1, 0, 2).reshape(n, -1)
    return np.concatenate([r["base_lin"], r["base_ang_deg"], cat(r["foot_pos"]), cat(r["foot_force"]),
                           r["foot_contact"].T.astype(np.float64)], axis=1)


def test_two_processes_share_one_counter(chd, tmp_path):
    """Two processes on cuda:0 (gloo, CPU tensors for the merge, one FileStore counter), ShardedSolver(slots=4) over 16
    mixed 2-foot clips: every clip solved exactly once, the merged result that of one process's queue, and rank 0's
    files those write_outputs makes of it (the final file and success log where stages 3 and 4 ended the same way)."""
    import torch.multiprocessing as mp
    port = 37500 + (os.getpid() % 2000)
    mp.spawn(_two_ranks, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "r0.npz")), np.load(str(tmp_path / "r1.npz"))
    for k in r0.files:
        assert r0[k].tobytes() == r1[k].tobytes(), k
    ps = _mixed(chd, 16, 400)
    got = {k: r0[k] for k in r0.files}
    print("clips solved by rank 0 / 1: %d / %d" % ((got["solved_by"] == 0).sum(), (got["solved_by"] == 1).sum()))
    assert got["solved"].all() and set(got["solved_by"].tolist()) <= {0, 1}
    ref = chd.phys.PhysQueue(ps, 4).solve()
    assert_solves_agree(ref, got, 2)
    np.testing.assert_array_equal(got["frames"], ref["frames"])
    np.testing.assert_array_equal(got["success"], ref["success"])
    for i, p in enumerate(ps):
        d = str(tmp_path / "ref" / ("c%d" % i))
        os.makedirs(d)
        chd.phys.write_outputs(ref, i, p, d, 2)
        g = str(tmp_path / "rank0" / ("c%d" % i))
        names = list(chd.phys.SOLUTION_FILES[:2])
        if (ref["stage_status"][:, i] == got["stage_status"][:, i]).all() and ref["stage_iters"][4, i] == got["stage_iters"][4, i]:
            names.append(chd.phys.SOLUTION_FILES[2])
            assert open(os.path.join(d, "success_log.txt")).read() == open(os.path.join(g, "success_log.txt")).read()
        assert sorted(os.listdir(g)) == sorted(list(chd.phys.SOLUTION_FILES) + ["success_log.txt"])
        for name in names:
            assert_samples_close(_rows(chd, os.path.join(g, name)), _rows(chd, os.path.join(d, name)), 2)
