"""CPU tests of the claim source of the physics solve queue (`chd_phys_queue_set_claim`, `PhysQueue(claim=...)`), of
`chd.parallel.StoreClaim` over a FileStore shared by several processes, of the merge of queue results across gloo ranks
(`merge_solved`, `ShardedSolver(slots=...)`) and of the writer rank 0 of `phys_optim.py --slots` uses under torchrun."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests.util import QueueLib, random_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_claim_refuses_batch_and_null_handles(chd):
    P = chd.phys
    L = P.load_lib()
    fn = P.CLAIM_FN(lambda ctx, want, first: 0)
    cb, null = C.cast(fn, C.c_void_p), None
    assert L.chd_phys_queue_set_claim(None, cb, None) == -1
    assert L.chd_phys_queue_set_claim(None, null, None) == -1
    b = P.PhysBatch([chd.synth.make_problem(0)], host_only=True)
    assert L.chd_phys_queue_set_claim(b.h, cb, None) == -1
    assert L.chd_phys_queue_set_claim(b.h, null, None) == -1
    ps = [chd.synth.make_problem(s, n_frames=40, n_ee=2) for s in range(3)]
    arr, _ = P.make_problem_array(ps)
    h = C.c_void_p()
    assert L.chd_phys_queue_create(arr, 3, 2, None, -2, None, C.byref(h)) == 0
    try:
        assert L.chd_phys_queue_set_claim(h, cb, None) == 0        # a queue handle takes a source, and NULL clears it
        assert L.chd_phys_queue_set_claim(h, null, None) == 0
    finally:
        L.chd_phys_batch_destroy(h)


def _from_the_back(n, stop=None):
    """claim source handing out the last `want` positions not yet handed out (at most `stop` in all)"""
    left = [n if stop is None else stop]

    def claim(want):
        k = min(want, left[0])
        left[0] -= k
        return (n - (n if stop is None else stop)) + left[0], k
    return claim


@pytest.mark.parametrize("stop", [None, 5])
def test_claim_chunks_give_input_order_and_solved_mask(chd, monkeypatch, stop):
    """Uneven chunks (3 at the start, then 1, 2, 1, 3, ...) taken from the back of the queue: every clip handed out is
    answered in its input place, `solved` marks exactly those clips, the others' rows stay zero."""
    fake = QueueLib([1, 2, 1, 3, 2, 2, 1, 3])
    monkeypatch.setattr(chd.phys, "load_lib", lambda: fake)
    F = [50, 90, 40, 120, 90, 70, 66, 48, 101, 75]
    N = len(F)
    ps = [chd.synth.make_problem(i, n_frames=f, n_ee=2) for i, f in enumerate(F)]
    q = chd.phys.PhysQueue(ps, slots=3, claim=_from_the_back(N, stop))
    out = q.solve()
    est = chd.parallel.work_estimate(ps)
    expect = sorted(range(N), key=lambda i: (-est[i], i))          # queue position -> input clip
    pos = {i: k for k, i in enumerate(expect)}
    handed = set(range(N)) if stop is None else set(range(N - stop, N))
    assert fake.asked[0] == 3 and len(set(fake.asked)) > 1
    for i, f in enumerate(F):
        if pos[i] in handed:
            assert out["solved"][i]
            assert out["frames"][i] == f
            assert (out["samples"][:, i, :f, 0] == f).all() and (out["samples"][:, i, f:, 0] == 0).all()
            assert (out["stage_status"][:, i] == pos[i]).all() and tuple(out["success"][i]) == (pos[i], f)
            assert (out["stage_stats"][:, i] == f).all()
        else:
            assert not out["solved"][i]
            assert out["frames"][i] == 0 and (out["samples"][:, i] == 0).all() and (out["stage_iters"][:, i] == 0).all()
    assert out["solved"].dtype == bool and out["solved"].sum() == len(handed)


def test_claim_exception_is_raised_by_solve(chd, monkeypatch):
    fake = QueueLib([2])
    monkeypatch.setattr(chd.phys, "load_lib", lambda: fake)
    ps = [chd.synth.make_problem(i, n_frames=40 + i, n_ee=2) for i in range(4)]
    calls = []

    def claim(want):
        calls.append(want)
        if len(calls) == 2:
            raise ValueError("store went away")
        return 0, want

    q = chd.phys.PhysQueue(ps, slots=2, claim=claim)
    with pytest.raises(RuntimeError, match="claim source") as e:
        q.solve()
    assert isinstance(e.value.__cause__, ValueError)


def _claimer(rank, path, n, seed, tmp):
    import random
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import chd
    store = dist.FileStore(path, 3)
    claim = chd.parallel.StoreClaim(store, "test", n)
    rng = random.Random(seed + rank)
    got = []
    for gen in range(2):                                              # a restart starts the counter over
        if gen:
            claim.restart()
        while True:
            want = rng.randint(1, 9)
            f, k = claim(want)
            assert 0 <= k <= want and (k == 0 or 0 <= f <= n - k)
            got.append((gen, f, k))
            if k < want:
                break
    np.save(os.path.join(tmp, "claims%d.npy" % rank), np.array(got, np.int64))


def test_store_claim_hands_out_every_position_once(tmp_path):
    import torch.multiprocessing as mp
    n = 157
    mp.spawn(_claimer, args=(str(tmp_path / "store"), n, 11, str(tmp_path)), nprocs=3, join=True)
    for gen in range(2):
        seen = np.zeros(n, np.int64)
        for r in range(3):
            for g, f, k in np.load(str(tmp_path / ("claims%d.npy" % r))):
                if g == gen:
                    seen[f:f + k] += 1
        np.testing.assert_array_equal(seen, np.ones(n, np.int64))


N_MERGE = 11


def _subset(rank, world, n):
    """interleaved random subsets: a random owner for every clip (rank 1 gets clip 0 so that both ranks hold some)"""
    owner = np.random.default_rng(9).integers(0, world, n)
    owner[0] = 1
    return owner == rank


def _merge_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = [chd.synth.make_problem(s, n_frames=40 + 3 * s, n_ee=2) for s in range(N_MERGE)]

    def solve_fn(problems):
        assert len(problems) == N_MERGE
        full = random_result(len(problems), 7)
        mine = _subset(rank, world, len(problems))
        out = {k: v.copy() for k, v in full.items()}
        for k in out:
            np.moveaxis(out[k], chd.phys.clip_axis(k), 0)[~mine] = 0   # rows of clips another rank solved stay zero
        out["solved"] = mine
        return out

    s = chd.parallel.ShardedSolver(ps, rank=rank, world=world, solve_fn=solve_fn, slots=4)
    out = s.solve()
    s.close()
    np.savez(os.path.join(tmp, "m%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    dist.destroy_process_group()


def test_merge_is_bitwise_union_in_input_order(tmp_path):
    import torch.multiprocessing as mp
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_merge_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "m0.npz")), np.load(str(tmp_path / "m1.npz"))
    full = random_result(N_MERGE, 7)
    owner = np.where(_subset(1, 2, N_MERGE), 1, 0)
    for k in r0.files:                                                  # every rank returns the same bits
        assert r0[k].tobytes() == r1[k].tobytes(), k
    for k, v in full.items():
        assert r0[k].dtype == v.dtype and r0[k].tobytes() == v.tobytes(), k   # bitwise, -0.0 included
    assert (np.signbit(r0["samples"]) == np.signbit(full["samples"])).all()
    np.testing.assert_array_equal(r0["solved"], np.ones(N_MERGE, bool))
    np.testing.assert_array_equal(r0["solved_by"], owner)


def test_merge_on_one_rank_keeps_unsolved_rows_empty(chd):
    full = random_result(6, 7)
    local = dict(full, solved=np.array([1, 0, 1, 1, 0, 0], bool))
    out = chd.parallel.merge_solved(local, 1)
    np.testing.assert_array_equal(out["solved_by"], [0, -1, 0, 0, -1, -1])
    assert out["samples"][:, [0, 2, 3]].tobytes() == full["samples"][:, [0, 2, 3]].tobytes()
    assert (out["samples"][:, [1, 4, 5]] == 0).all() and (out["frames"][[1, 4, 5]] == 0).all()


def test_rank0_writer_writes_four_files_per_clip(chd, tmp_path):
    """phys_optim.write_results (rank 0 of a `--slots` run under torchrun, and the one-GPU run): the four files of
    every clip, each solution file from its own snapshot, feet padding of a mixed batch stripped."""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import phys_optim
    ps = [chd.synth.make_problem(0, n_frames=40, n_ee=2), chd.synth.make_problem(1, n_frames=50, n_ee=4)]
    fo, stride = 30, chd.phys.sample_stride(4)
    rng = np.random.default_rng(3)
    out = dict(samples=np.round(rng.standard_normal((3, 2, fo, stride)), 3), frames=np.array([21, 30], np.int32),
               success=np.array([[1, 0], [0, 1]], np.int32), stage_status=np.zeros((6, 2), np.int32),
               stage_iters=np.ones((6, 2), np.int32))
    for s in range(3):
        out["samples"][s, :, :, 6 + 6 * 4:] = rng.integers(0, 2, (2, fo, 4))
    dirs = [str(tmp_path / ("clip%d" % i)) for i in range(2)]
    for d in dirs:
        os.makedirs(d)
    phys_optim.write_results(out, ps, dirs, 4)
    for i, (p, d) in enumerate(zip(ps, dirs)):
        assert sorted(os.listdir(d)) == sorted(list(chd.phys.SOLUTION_FILES) + ["success_log.txt"])
        base, pos, frc, flag = chd.phys.sample_columns(p.n_ee, 4)
        nf = int(out["frames"][i])
        for snap, name in enumerate(chd.phys.SOLUTION_FILES):
            r = chd.io_formats.read_solution(os.path.join(d, name))
            rows = out["samples"][snap, i, :nf]
            assert r["num_frames"] == nf and r["num_feet"] == p.n_ee
            np.testing.assert_allclose(r["base_lin"], rows[:, base[:3]], atol=1e-9)
            np.testing.assert_allclose(r["foot_pos"].transpose(1, 0, 2).reshape(nf, -1), rows[:, pos], atol=1e-9)
            np.testing.assert_array_equal(r["foot_contact"].T, rows[:, flag])
        log = open(os.path.join(d, "success_log.txt")).read()
        assert log == "dynamics %d\ndurations %d\n" % tuple(out["success"][i])
