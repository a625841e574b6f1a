"""Multi-GPU plumbing of the phys-optim path: sequences are independent NLPs (the reference runs them as separate
processes, scripts/run_phys_mocap.py:80), so they shard embarrassingly -- one process per GPU, no collective inside
the solver, one gather of the fixed-size sampled solutions at the end (SURVEY.md 8(e)).

Everything here is backend agnostic (`nccl` on the GPU box, `gloo` in the CPU tests).
"""
from __future__ import annotations

import itertools
from typing import List, Sequence, Tuple

import numpy as np

from . import phys


def shard_by_work(work: Sequence[float], world: int) -> List[List[int]]:
    """Deals sequence indices to ranks: sorted by estimated work (number of variables ~ iterations x size),
    largest first, round robin with reversal every other pass (snake order) so that ragged batches balance.
    Deterministic; every rank computes the same assignment."""
    order = sorted(range(len(work)), key=lambda i: (-float(work[i]), i))
    shards: List[List[int]] = [[] for _ in range(world)]
    for k, idx in enumerate(order):
        r = k % world
        if (k // world) % 2 == 1:
            r = world - 1 - r
        shards[r].append(idx)
    for s in shards:
        s.sort()
    return shards


def pad_to(shards: List[List[int]]) -> int:
    """Per-rank slot count so that the gather has equal receive counts."""
    return max((len(s) for s in shards), default=0)


def gather_samples(local, world: int, group=None):
    """all_gather of a (slots, frames, stride) tensor -> (world*slots, frames, stride).  `local` is a torch tensor
    on the device the process group's backend expects (cuda for nccl, cpu for gloo)."""
    import torch
    import torch.distributed as dist
    if world == 1 or not dist.is_initialized():
        return local
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out.view(-1), local.contiguous().view(-1), group=group)
    return out


def unshard(gathered: np.ndarray, shards: List[List[int]], slots: int) -> np.ndarray:
    """Reorders gathered rows (rank major, `slots` rows per rank) back to the original sequence order."""
    n = sum(len(s) for s in shards)
    out = np.zeros((n,) + gathered.shape[1:], dtype=gathered.dtype)
    for r, s in enumerate(shards):
        for k, idx in enumerate(s):
            out[idx] = gathered[r * slots + k]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# The product's multi-GPU entry point: shard -> solve -> sample into the send buffer -> ONE gather -> unshard.
# ---------------------------------------------------------------------------------------------------------------------
# per-sequence trailer of the gathered block: these fields (`phys.pack_rows`, 15 columns), zero-padded to N_EXTRA
TRAILER_KEYS = ("frames", "success", "stage_status", "stage_iters")
N_EXTRA = 16


def work_estimate(problems) -> List[float]:
    """Predicted solver work of a sequence: interior-point iterations grow with the number of contact phases (every
    switch adds free swing / stance nodes and, in stage 3, a duration), the cost of one iteration with the frame count."""
    return [float(p.n_frames) * float(sum(len(d) for d in p.ee_durations)) * (p.n_ee / 2.0) for p in problems]


def frames_out(p) -> int:
    """SaveSolution frame count of a problem (phys_optim.cpp:84: t accumulates dt while t <= T + 1e-5)."""
    T = float(np.sum(np.asarray(p.ee_durations[0], dtype=np.float64)))
    return int((T + 1e-5) / p.dt) + 1


class StoreClaim:
    """Claim source of a `PhysQueue` (its `claim`) shared by processes through a c10d store (`torch.distributed.Store`:
    the process group's store under torchrun, or a `FileStore`).  A claim of `want` positions is one atomic
    `store.add(key, want)`, which returns the new total t, and hands out [t - want, t) ∩ [0, n): every position of
    [0, n) goes to exactly one claim of one process.  `restart()` moves to a fresh counter (the key's next generation) so
    that a repeated solve starts over; every process must restart as often as the others."""

    def __init__(self, store, key: str, n: int):
        self.store, self.key, self.n, self.generation = store, key, int(n), 0

    def restart(self):
        self.generation += 1

    def __call__(self, want: int) -> Tuple[int, int]:
        t = int(self.store.add("%s/%d" % (self.key, self.generation), int(want)))
        lo, hi = min(t - int(want), self.n), min(t, self.n)
        return lo, hi - lo


# Fields of a row of a rank's block in the merge of queue results (merge_solved), after the clip index
# (`phys.pack_rows`); the cost terms follow when the results carry them.
MERGE_KEYS = phys.SOLVE_KEYS + ("stage_stats",)


def merge_solved(local: dict, world: int, group=None, tensor_device=None) -> dict:
    """Merges the `PhysQueue.solve()` results of `world` ranks that each solved some of the same N clips (`solved`;
    every rank's arrays have the same shapes) into every clip's result, by clip index.  The ranks' solved counts are
    all-gathered, every rank's block of solved rows is padded to the largest count, and one `all_gather_into_tensor`
    moves the blocks, each row carrying its clip index, the three snapshots and the status trailer.  Rows are copied,
    never summed, so every bit of a result (a -0.0 too) arrives as its rank computed it.  Returns `PhysQueue.solve()`'s
    keys over all N clips in input order, plus `solved_by` (N, the rank that solved each clip, -1: none) and
    `d2h_bytes` (the gathered block).  `cost_terms`, when every rank's results have them, travel in the row next to
    the stage statistics.  `tensor_device`: where the collective's tensors live (cuda for nccl, the default cpu for
    gloo)."""
    import torch
    import torch.distributed as dist
    dev = tensor_device or torch.device("cpu")
    _, N, fo, stride = local["samples"].shape
    keys = MERGE_KEYS + (("cost_terms",) if "cost_terms" in local else ())
    mine = np.nonzero(local["solved"])[0]
    n = len(mine)
    packed = phys.pack_rows(local, keys, mine)
    width = 1 + packed.shape[1]
    collective = world > 1 and dist.is_initialized()
    counts = torch.tensor([n], dtype=torch.int64, device=dev)
    if collective:
        counts = torch.empty(world, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(counts, torch.tensor([n], dtype=torch.int64, device=dev), group=group)
    counts = counts.cpu().numpy()
    cmax = int(counts.max())
    blk = np.zeros((cmax, width))
    blk[:n, 0] = mine
    blk[:n, 1:] = packed
    g = blk
    if collective and cmax > 0:
        send = torch.from_numpy(blk).to(dev)
        recv = torch.empty((world * cmax, width), dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(recv, send, group=group)
        g = recv.cpu().numpy()
    rows = np.concatenate([g[r * cmax:r * cmax + int(counts[r])] for r in range(len(counts))])
    rank_of = np.repeat(np.arange(len(counts)), counts)
    idx = rows[:, 0].astype(np.int64)
    if len(np.unique(idx)) != len(idx) or (len(idx) and (idx.min() < 0 or idx.max() >= N)):
        raise RuntimeError("merge of queue results: a clip was solved by more than one rank, or a clip index is out of range")
    out = phys.result_arrays(N, keys + ("solved",), fo, stride)
    phys.unpack_rows(rows[:, 1:], out, keys, idx)
    out["solved"][idx] = True
    out["solved_by"] = np.full(N, -1, np.int32)
    out["solved_by"][idx] = rank_of
    out["d2h_bytes"] = int(g.nbytes)
    return out


_QUEUE_KEYS = itertools.count()   # one counter key per queue-mode ShardedSolver, created in the same order on every rank


class ShardedSolver:
    """One process per GPU (torchrun).  Every rank holds the same problem list, solves its shard on its device and
    takes part in a single all_gather of the fixed-size result block (final SaveSolution snapshot + status trailer).

    `solve_fn(problems) -> dict(final=(n, fo, stride) array, frames, success, stage_status (6,n), stage_iters (6,n))`
    replaces the CUDA solve in the CPU (gloo) tests; the default drives `PhysBatch` on `device` (`stage3_band_above`:
    see `PhysBatch`).

    `slots`: instead of a static shard, every rank runs a `PhysQueue` of `slots` device slots over all N clips (so
    every clip fits every slot on every rank and its result does not depend on the rank that solved it), and all
    ranks claim their next clips from one counter (`StoreClaim`) in `store`, by default the process group's store.  A
    rank that finishes early simply claims more.  `solve()` then merges the ranks' results by clip index
    (`merge_solved`) and returns `PhysQueue.solve()`'s keys over all N clips, including all three snapshots, plus
    `solved_by`.  Every rank keeps the page-locked record store of all N clips (about 106 MB per 256 clips of 120
    frames, 2 feet), and every rank must call `solve()` as often as the others.  With `slots`, `solve_fn(problems)`
    stands in for `PhysQueue.solve()` over all N problems and returns its dict, `solved` marking the clips this rank
    solved.

    `weights`: one 5-tuple for every problem or one per problem (`phys.clip_weights`); `options`: one
    `phys.SolverOptions` for every problem or one per problem (`phys.clip_options`).  Without `slots` only the final
    iterate travels, which for a clip that stopped early (`SolverOptions.last_stage`) is that of its last stage.
    `solve(cost_terms=True)` (with `slots` only) also returns every clip's unweighted cost terms (`phys.COST_TERMS`),
    merged by clip index."""

    def __init__(self, problems, weights=phys.DEFAULT_WEIGHTS, device: int = 0, rank: int = 0, world: int = 1,
                 group=None, solve_fn=None, tensor_device=None, stage3_band_above=None, slots=None, store=None,
                 options=None):
        self.problems, self.rank, self.world, self.group = list(problems), rank, world, group
        self.queue_slots, self.queue = slots, None
        per = phys.clip_weights(weights, len(self.problems))
        per_opt = phys.clip_options(options, len(self.problems))
        if slots is not None:
            self._init_queue(weights, device, solve_fn, tensor_device, stage3_band_above, slots, store, options)
            return
        self.shards = shard_by_work(work_estimate(self.problems), world)
        self.slots = pad_to(self.shards)
        self.mine = self.shards[rank]
        self.n_ee_max = max(p.n_ee for p in self.problems)
        self.stride = phys.sample_stride(self.n_ee_max)
        self.fo = max(frames_out(p) for p in self.problems)
        self.width = self.fo * self.stride + N_EXTRA
        self.solve_fn = solve_fn
        self.batch = None
        import torch
        if solve_fn is None:
            self.batch = phys.PhysBatch([self.problems[i] for i in self.mine], device=device,
                                        weights=weights if per is None else per[self.mine],
                                        options=None if per_opt is None else [per_opt[i] for i in self.mine],
                                        stage3_band_above=stage3_band_above) if self.mine else None
            tensor_device = tensor_device or torch.device("cuda", device)
        self.tdev = tensor_device or torch.device("cpu")
        self.send = torch.zeros((self.slots, self.width), dtype=torch.float64, device=self.tdev)
        self.recv = torch.zeros((world * self.slots, self.width), dtype=torch.float64, device=self.tdev) if world > 1 else None
        self.last_ms = {}

    def _init_queue(self, weights, device, solve_fn, tensor_device, stage3_band_above, slots, store, options):
        import torch
        self.solve_fn, self.batch, self.last_ms = solve_fn, None, {}
        self.n_ee_max = max(p.n_ee for p in self.problems)
        if solve_fn is None:
            if store is None:
                from torch.distributed import distributed_c10d
                store = distributed_c10d._get_default_store()
            self.claim = StoreClaim(store, "chd/phys_queue/%d" % next(_QUEUE_KEYS), len(self.problems))
            self.queue = phys.PhysQueue(self.problems, slots, weights=weights, device=device,
                                        stage3_band_above=stage3_band_above, claim=self.claim, options=options)
            tensor_device = tensor_device or torch.device("cuda", device)
        self.tdev = tensor_device or torch.device("cpu")

    def close(self):
        if self.batch is not None:
            self.batch.close()
            self.batch = None
        if self.queue is not None:
            self.queue.close()
            self.queue = None

    def _solve_queue(self, cost_terms: bool) -> dict:
        import time
        t0 = time.perf_counter()
        if self.solve_fn is not None:
            local = self.solve_fn(self.problems)
        else:
            self.claim.restart()
            local = self.queue.solve(cost_terms=cost_terms)
        t1 = time.perf_counter()
        out = merge_solved(local, self.world, self.group, self.tdev)
        t2 = time.perf_counter()
        self.last_ms = {"solve_ms": 1e3 * (t1 - t0), "gather_ms": 1e3 * (t2 - t1)}
        return out

    def _solve_local(self, resident: bool):
        """fills self.send; returns the local status arrays"""
        import torch
        n = len(self.mine)
        trailer = np.zeros((self.slots, N_EXTRA))
        if n == 0:
            return trailer
        if self.solve_fn is not None:
            r = self.solve_fn([self.problems[i] for i in self.mine])
            blk = np.zeros((self.slots, self.fo, self.stride))
            f = np.asarray(r["final"])
            blk[:n, :f.shape[1], :f.shape[2]] = f
            self.send[:, :self.fo * self.stride] = torch.from_numpy(blk.reshape(self.slots, -1)).to(self.tdev)
        else:
            b = self.batch
            if resident:
                b.reset()
            keys = phys.SOLVE_KEYS[2:]               # the snapshots are sampled below, the frame counts known
            r = phys.result_arrays(b.B, keys)
            b._chk(b.L.chd_phys_solve(b.h, None, None, *[r[k].ctypes.data for k in keys]))
            # final iterate sampled on the device straight into the send buffer (no host round trip)
            fo_l, st_l = b.dims["frames_out_max"], phys.sample_stride(b.n_ee_max)
            if fo_l == self.fo and st_l == self.stride:
                view = self.send[:n, :self.fo * self.stride]
                if view.is_contiguous():
                    b._chk(b.L.chd_phys_sample_device(b.h, view.data_ptr(), torch.cuda.current_stream().cuda_stream))
                else:
                    tmp = torch.zeros((n, self.fo * self.stride), dtype=torch.float64, device=self.tdev)
                    b._chk(b.L.chd_phys_sample_device(b.h, tmp.data_ptr(), torch.cuda.current_stream().cuda_stream))
                    self.send[:n, :self.fo * self.stride] = tmp
            else:   # ragged shards: local frame / stride padding differs from the global one
                tmp = torch.zeros((n, fo_l, st_l), dtype=torch.float64, device=self.tdev)
                b._chk(b.L.chd_phys_sample_device(b.h, tmp.data_ptr(), torch.cuda.current_stream().cuda_stream))
                blk = torch.zeros((n, self.fo, self.stride), dtype=torch.float64, device=self.tdev)
                blk[:, :fo_l, :st_l] = tmp
                self.send[:n, :self.fo * self.stride] = blk.reshape(n, -1)
            r["frames"] = np.array([frames_out(self.problems[i]) for i in self.mine], np.int32)
        trailer[:n] = phys.pack_rows(r, TRAILER_KEYS, np.arange(n), N_EXTRA)
        self.send[:, self.fo * self.stride:] = torch.from_numpy(trailer).to(self.tdev)
        return trailer

    def solve(self, resident: bool = False, cost_terms: bool = False) -> dict:
        """Solves the shard (resident=True: device-side reset of an already uploaded batch) and gathers.  Every rank
        returns the full result in the original sequence order.  With `slots`: the queue solve and the merge of every
        clip's results (resident does not apply: a queue always starts over), with `cost_terms` as
        `PhysQueue.solve`'s."""
        if self.queue_slots is not None:
            return self._solve_queue(cost_terms)
        if cost_terms:
            raise ValueError("cost_terms needs the queue form of the sharded solve (slots=S)")
        import time
        import torch
        import torch.distributed as dist
        t0 = time.perf_counter()
        self._solve_local(resident)
        if self.tdev.type == "cuda":
            torch.cuda.synchronize()
        t1 = time.perf_counter()
        if self.world > 1:
            dist.all_gather_into_tensor(self.recv.view(-1), self.send.view(-1), group=self.group)
            if self.tdev.type == "cuda":
                torch.cuda.synchronize()
            g = self.recv
        else:
            g = self.send
        t2 = time.perf_counter()
        self.last_ms = {"solve_ms": 1e3 * (t1 - t0), "gather_ms": 1e3 * (t2 - t1)}
        g = g.cpu().numpy()
        full = unshard(g, self.shards, self.slots)
        N = len(self.problems)
        out = dict(samples=full[:, :self.fo * self.stride].reshape(N, self.fo, self.stride))
        out.update(phys.result_arrays(N, TRAILER_KEYS))
        phys.unpack_rows(full[:, self.fo * self.stride:], out, TRAILER_KEYS, np.arange(N))
        out["d2h_bytes"] = int(g.nbytes)
        return out


def solve_sharded(problems, weights=phys.DEFAULT_WEIGHTS, device: int = 0, rank: int = 0, world: int = 1, group=None,
                  solve_fn=None, tensor_device=None, stage3_band_above=None, slots=None, store=None,
                  cost_terms: bool = False, options=None) -> dict:
    """shard -> solve -> one gather -> unshard for a list of `PhysProblem`s (see ShardedSolver; `slots`: a queue on
    every rank, claimed from one shared counter, merged by clip index; `weights`, `options` and `cost_terms` as
    there)."""
    s = ShardedSolver(problems, weights, device, rank, world, group, solve_fn, tensor_device, stage3_band_above, slots,
                      store, options)
    try:
        return s.solve(cost_terms=cost_terms)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# Contact classifier: videos are independent too (SURVEY.md 8(e)): shard by frame count, one gather of the int64 labels.
# ---------------------------------------------------------------------------------------------------------------------
def detect_contacts_sharded(raw, state_dict=None, device: int = 0, rank: int = 0, world: int = 1, group=None, detect_fn=None,
                            gather_device=None, precision: str = "fp32"):
    """`raw`: list of (F_i, 25, 3) OpenPose keypoint arrays, identical on every rank.  Every rank runs
    `ContactNet.detect` (`chd_contact_detect`: preprocessing, windows, network, votes on its GPU) on its shard, the
    (slots, F_max, 4) int64 label blocks are gathered once and put back in input order.  Returns the list of (F_i, 4) labels.
    `precision`: numerical mode of every rank's `ContactNet` ("fp32" or "tf32x3").
    `detect_fn(list_of_raw) -> list of (F_i, 4)` replaces the CUDA path in the CPU tests."""
    import torch
    n = len(raw)
    shards = shard_by_work([float(r.shape[0]) for r in raw], world)
    slots = pad_to(shards)
    f_max = max(int(r.shape[0]) for r in raw)
    mine = shards[rank]
    # The reference pads every video of a batch to the batch's longest one by repeating the last frame
    # (real_video_dataset.py:165-191) and votes over the padded windows before trimming, so the last labels of a video
    # depend on the longest video it is batched with.  To return exactly what one unsharded call returns, a shard that does
    # not hold the globally longest video carries it along (its labels are dropped).
    longest = max(range(n), key=lambda i: (raw[i].shape[0], -i))
    batch = [raw[i] for i in mine] + ([raw[longest]] if mine and longest not in mine else [])
    if detect_fn is None:
        from .contact import ContactNet
        net = ContactNet(state_dict, device=device, precision=precision)
        labels = net.detect(batch)[0][:len(mine)] if mine else []
        net.close()
    else:
        labels = detect_fn(batch)[:len(mine)] if mine else []
    dev = gather_device if gather_device is not None else (torch.device("cuda", device) if detect_fn is None else torch.device("cpu"))
    block = torch.zeros((slots, f_max, 4), dtype=torch.int64, device=dev)
    for k, lab in enumerate(labels):
        block[k, :lab.shape[0]] = torch.as_tensor(np.asarray(lab, dtype=np.int64), device=dev)
    gathered = gather_samples(block, world, group).cpu().numpy()
    full = unshard(gathered, shards, slots)
    return [full[i, :raw[i].shape[0]] for i in range(n)]
