"""Multi-process (gloo, world_size 2) test of the sharding + gather plumbing used on N > 1 GPUs."""
import os

import numpy as np
import pytest


def _worker(rank, world, port, tmp):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B = 5
    ps = chd.synth.make_batch(B, 40, 2)
    full = chd.phys.PhysBatch(ps, host_only=True)
    shards = chd.parallel.shard_by_work(full.sizes[:, 0], world)
    slots = chd.parallel.pad_to(shards)
    mine = shards[rank]
    local = chd.phys.PhysBatch([ps[i] for i in mine], host_only=True)
    # stand-in for the sampled solution block: the initial iterate, padded to a fixed width
    width = 1500
    x = np.zeros((slots, 1, width))
    x0 = local.get_x()
    x[:len(mine), 0, :x0.shape[1]] = x0
    g = chd.parallel.gather_samples(torch.from_numpy(x), world).numpy()
    out = chd.parallel.unshard(g, shards, slots)
    if rank == 0:
        np.save(os.path.join(tmp, "gathered.npy"), out)
        np.save(os.path.join(tmp, "ref.npy"), full.get_x())
    dist.destroy_process_group()


def test_shard_and_gather_gloo(tmp_path):
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    got = np.load(str(tmp_path / "gathered.npy"))
    ref = np.load(str(tmp_path / "ref.npy"))
    for i in range(ref.shape[0]):
        n = ref.shape[1]
        np.testing.assert_array_equal(got[i, 0, :n][ref[i] != 0], ref[i][ref[i] != 0])


def test_shard_by_work_balanced(chd):
    work = [10, 1, 9, 2, 8, 3, 7, 4]
    s = chd.parallel.shard_by_work(work, 2)
    assert sorted(s[0] + s[1]) == list(range(8))
    assert abs(sum(work[i] for i in s[0]) - sum(work[i] for i in s[1])) <= 2
    assert chd.parallel.shard_by_work([5, 5, 5], 4)[3] == []


def _oracle_solve_fn(problems):
    """stand-in for the CUDA solve of a shard in the CPU test: the oracle solves the same NLPs (test infrastructure)"""
    import chd
    from oracle.phys import OracleProblem
    finals, frames, succ = [], [], []
    sstat, siter = np.full((6, len(problems)), -9, np.int32), np.zeros((6, len(problems)), np.int32)
    for i, p in enumerate(problems):
        r = OracleProblem(p).solve()
        finals.append(r["durations"]), frames.append(len(r["durations"])), succ.append(r["success"])
        for k, s in zip(r["stage_ids"], r["stages"]):
            sstat[chd.phys.STAGES[k], i], siter[chd.phys.STAGES[k], i] = s["status"], s["iters"]
    fo = max(frames)
    blk = np.zeros((len(problems), fo, finals[0].shape[1]))
    for i, f in enumerate(finals):
        blk[i, :len(f)] = f
    return dict(final=blk, frames=np.array(frames), success=np.array(succ, np.int32), stage_status=sstat, stage_iters=siter)


def _worker_solve(rank, world, port, tmp):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = [chd.synth.make_problem(s, n_frames=40 + 4 * s, n_ee=2) for s in range(3)]     # ragged lengths
    out = chd.parallel.solve_sharded(ps, rank=rank, world=world, solve_fn=_oracle_solve_fn)
    np.savez(os.path.join(tmp, "rank%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    dist.destroy_process_group()


def test_solve_sharded_gloo(tmp_path, chd):
    """chd.parallel.solve_sharded (the path bench.py and scripts/phys_optim.py use on N > 1 GPUs) with world size 2 on
    gloo: both ranks end up with every sequence's solved trajectory and status, in the original order."""
    import torch.multiprocessing as mp
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_worker_solve, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "rank0.npz")), np.load(str(tmp_path / "rank1.npz"))
    for k in r0.files:
        np.testing.assert_array_equal(r0[k], r1[k])
    ps = [chd.synth.make_problem(s, n_frames=40 + 4 * s, n_ee=2) for s in range(3)]
    ref = _oracle_solve_fn(ps)
    for i in range(3):
        nf = ref["frames"][i]
        assert r0["frames"][i] == nf == chd.parallel.frames_out(ps[i])
        np.testing.assert_array_equal(r0["samples"][i, :nf], ref["final"][i, :nf])
    np.testing.assert_array_equal(r0["stage_status"], ref["stage_status"])
    np.testing.assert_array_equal(r0["stage_iters"], ref["stage_iters"])
    assert (r0["success"] == 1).all()


def _oracle_detect_fn(sd):
    def fn(raws):
        from oracle import contact as oc
        frames, lens = oc.preprocess_videos(raws)
        logits = oc.forward_torch(sd, oc.windows_from_frames(frames))
        return [oc.vote(logits[i], int(lens[i])) for i in range(len(raws))]
    return fn


def _worker_contacts(rank, world, port, tmp):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import torch.distributed as dist
    import chd
    from make_contact_golden import contact_weights, synth_keypoints
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    raw = [synth_keypoints(40 + i, 30 + 7 * i) for i in range(5)]                  # ragged lengths, odd count
    out = chd.parallel.detect_contacts_sharded(raw, rank=rank, world=world, detect_fn=_oracle_detect_fn(contact_weights(0)))
    np.savez(os.path.join(tmp, "c%d.npz" % rank), *out)
    dist.destroy_process_group()


def test_detect_contacts_sharded_gloo(tmp_path, chd):
    """Contact path across ranks (SURVEY 8(e)): videos sharded by length, one gather of the int64 labels, input order restored."""
    import sys
    import torch.multiprocessing as mp
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_contact_golden import contact_weights, synth_keypoints
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_worker_contacts, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "c0.npz")), np.load(str(tmp_path / "c1.npz"))
    raw = [synth_keypoints(40 + i, 30 + 7 * i) for i in range(5)]
    ref = _oracle_detect_fn(contact_weights(0))(raw)
    for i in range(5):
        a, b = r0["arr_%d" % i], r1["arr_%d" % i]
        assert a.dtype == np.int64 and a.shape == (30 + 7 * i, 4)
        np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(a, ref[i])
