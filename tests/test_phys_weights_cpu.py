"""CPU tests of per-clip cost weights (chd_phys_options.clip_weights, the `weights` of PhysBatch / PhysQueue /
ShardedSolver, the `--w_*` lists of phys_optim.py and weight_sweep.py) and of the column order of the cost terms
(chd_phys_cost_terms, `chd.phys.COST_TERMS`) against the CPU oracle's cost terms."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")

SETTINGS = [(0.4, 1.7, 0.3, 0.1, 0.1), (1.0, 0.5, 1.0, 0.3, 1.0), (0.2, 2.5, 0.05, 0.02, 0.4), (0.7, 1.0, 2.0, 0.5, 0.01)]


def oracle_cost_terms(o, stage_weights):
    """The ten unweighted cost terms (`chd.phys.COST_TERMS`) of the oracle problem `o` at its stage and x, from its
    weighted cost terms (chdo_cost_term, phys_optim.cpp's AddCostSet order: data, position smoothing, velocity
    smoothing or the durations; base lin, base ang, then every foot) divided by the weights of that stage
    (`stage_weights`: the stage's row of `PhysBatch.stage_weights()`).  NaN for a term the stage does not have."""
    ne = o.n_ee
    c = o.cost_terms()
    has_dur = len(c) == 2 * (2 + ne) + ne                             # stage 3: DurationCost, no velocity smoothing
    out = np.full(10, np.nan)
    k = 0
    for b0 in range(0, 3 * ((len(c) - (ne if has_dur else 0)) // (2 + ne)), 3):
        out[b0] = c[k] / stage_weights[b0]
        out[b0 + 1] = c[k + 1] / stage_weights[b0 + 1]
        out[b0 + 2] = c[k + 2:k + 2 + ne].sum() / stage_weights[b0 + 2]
        k += 2 + ne
    if has_dur:
        out[9] = c[k:k + ne].sum() / stage_weights[9]
        k += ne
    assert k == len(c)
    return out


@pytest.mark.parametrize("n_ee", [2, 4])
def test_oracle_terms_weighted_add_up_to_the_cost(chd, n_ee):
    """At random points of every stage the oracle's terms, split into the ten columns and weighted with the stage's row
    of the product's stage table, add up to chdo_cost; the columns a stage has are those with a nonzero weight in that
    row; and the unweighted terms of one point agree between the stages that have them, which pins the column order."""
    from oracle.phys import OracleProblem, STAGES
    w = SETTINGS[1]
    p = chd.synth.make_problem(3, n_frames=40, n_ee=n_ee)
    sw = chd.phys.PhysBatch([p], weights=w, host_only=True).stage_weights()[0]
    o = OracleProblem(p, weights=w)
    rng = np.random.default_rng(4)
    o.set_stage("3")
    x3 = o.get_x() + rng.normal(0, 0.005, o.n)
    nd = o.n_dur
    x3[o.n - nd:] = np.concatenate([np.asarray(d[:-1]) for d in p.ee_durations]) + rng.uniform(-0.005, 0.005, nd)
    seen = {}
    for name in ("3", "1.1", "1.2", "2.1", "2.2", "4"):        # stage 3 first: the others keep its durations
        st = STAGES[name]
        o.set_stage(name)
        o.set_x(x3[:o.n])
        t = oracle_cost_terms(o, sw[st])
        have = ~np.isnan(t)
        np.testing.assert_array_equal(have, sw[st] != 0, err_msg=name)
        np.testing.assert_allclose((sw[st][have] * t[have]).sum(), o.cost(), rtol=1e-12)
        for j in np.nonzero(have)[0]:
            if j in seen:
                np.testing.assert_allclose(t[j], seen[j], rtol=1e-12, err_msg="%s column %d" % (name, j))
            seen[j] = t[j]
    assert sorted(seen) == list(range(10))


def test_host_layout_rows_carry_each_clips_weights(chd):
    """A batch (and a queue) built with one tuple per clip has, in every row of its stage table, the weights of a batch
    of the same clips that all use that clip's tuple; every other table is the same."""
    P = chd.phys
    ps = [chd.synth.make_problem(s, n_frames=40 + 7 * s, n_ee=2 + 2 * (s % 2)) for s in range(4)]
    mixed = P.PhysBatch(ps, weights=SETTINGS, host_only=True)
    for k, w in enumerate(SETTINGS):
        one = P.PhysBatch(ps, weights=w, host_only=True)
        np.testing.assert_array_equal(mixed.stage_weights()[k], one.stage_weights()[k])
        assert mixed.dims == one.dims
        np.testing.assert_array_equal(mixed.sizes, one.sizes)
        np.testing.assert_array_equal(mixed.sizes_fixed(), one.sizes_fixed())
        for a, b in ((mixed.layout(), one.layout()), (mixed.slot_index(), one.slot_index())):
            for key in a:
                np.testing.assert_array_equal(a[key], b[key], err_msg=key)
        np.testing.assert_array_equal(mixed.get_x(), one.get_x())
    sw = mixed.stage_weights()
    for k, (wl, wa, we, ws, wd) in enumerate(SETTINGS):
        for st in (0, 1):                                            # stages 1.1 / 1.2: fixed weights
            np.testing.assert_array_equal(sw[k, st], [1, 1, 1, 0.1, 0.1, 0.1, 0, 0, 0, 0])
        for st in (2, 3, 5):
            np.testing.assert_array_equal(sw[k, st], [wl, wa, we, 0.001, 0.001, ws, 1e-4, 1e-4, 1e-4, 0])
        np.testing.assert_array_equal(sw[k, 4], [wl, wa, we, 0.001, 0.001, ws, 0, 0, 0, wd])
    # a queue's slots describe its first clips in queue (work-estimate) order
    arr, _ = P.make_problem_array(ps)
    w, opt, keep = P._create_args(SETTINGS, 4, None)
    h = C.c_void_p()
    assert P.load_lib().chd_phys_queue_create(arr, 4, 2, w, -2, opt, C.byref(h)) == 0
    try:
        out = np.zeros((2, 6, 10))
        assert P.load_lib().chd_phys_get_stage_weights(h, out.ctypes.data) == 0
        np.testing.assert_array_equal(out, sw[:2])
    finally:
        P.load_lib().chd_phys_batch_destroy(h)


@pytest.mark.parametrize("bad", [-0.1, float("nan"), float("inf"), -float("inf")])
@pytest.mark.parametrize("which", [0, 2, 4])
def test_bad_weights_are_refused(chd, bad, which):
    P = chd.phys
    L = P.load_lib()
    ps = [chd.synth.make_problem(s, n_frames=40, n_ee=2) for s in range(3)]
    arr, _ = P.make_problem_array(ps)
    w = list(SETTINGS[0])
    w[which] = bad
    h = C.c_void_p()
    per = [SETTINGS[1], tuple(w), SETTINGS[2]]
    for weights in (tuple(w), per):
        wa, opt, keep = P._create_args(weights, 3, None)
        assert L.chd_phys_batch_create(arr, 3, wa, -2, opt, C.byref(h)) == -1
        assert L.chd_phys_queue_create(arr, 3, 2, wa, -2, opt, C.byref(h)) == -1
    # the scalar argument is not looked at when every clip has its own tuple
    wa, opt, keep = P._create_args(SETTINGS[:3], 3, None)
    bad_w = P._Weights(*w)
    assert L.chd_phys_batch_create(arr, 3, C.byref(bad_w), -2, opt, C.byref(h)) == 0
    L.chd_phys_batch_destroy(h)
    with pytest.raises(RuntimeError, match="code -1"):
        P.PhysBatch(ps, weights=per, host_only=True)


def test_miscounted_weights_are_refused(chd):
    ps = [chd.synth.make_problem(s, n_frames=40, n_ee=2) for s in range(3)]
    for weights in (SETTINGS[:2], SETTINGS, (0.4, 1.7, 0.3, 0.1), [SETTINGS[0][:4]] * 3):
        with pytest.raises(ValueError):
            chd.phys.PhysBatch(ps, weights=weights, host_only=True)
        with pytest.raises(ValueError):
            chd.phys.clip_weights(weights, 3)
    assert chd.phys.clip_weights(SETTINGS[0], 3) is None
    np.testing.assert_array_equal(chd.phys.clip_weights(SETTINGS[:3], 3), np.array(SETTINGS[:3]))


def _args(**kw):
    import argparse
    d = dict(w_com_lin="0.4", w_com_ang="1.7", w_ee="0.3", w_smooth="0.1", w_dur="0.1")
    d.update(kw)
    return argparse.Namespace(**d)


def test_phys_optim_weight_lists():
    sys.path.insert(0, SCRIPTS)
    import phys_optim
    assert phys_optim.parse_weights(_args(), 3) == (0.4, 1.7, 0.3, 0.1, 0.1)      # single values: one tuple, as before
    assert phys_optim.parse_weights(_args(w_ee="1"), 1) == (0.4, 1.7, 1.0, 0.1, 0.1)
    got = phys_optim.parse_weights(_args(w_ee="1,2,3", w_dur="0.5,0.6,0.7"), 3)
    assert got == [(0.4, 1.7, 1.0, 0.1, 0.5), (0.4, 1.7, 2.0, 0.1, 0.6), (0.4, 1.7, 3.0, 0.1, 0.7)]
    with pytest.raises(ValueError, match="w_ee"):
        phys_optim.parse_weights(_args(w_ee="1,2"), 3)


def test_weight_sweep_grid_and_rows(chd):
    sys.path.insert(0, SCRIPTS)
    import weight_sweep
    grid = weight_sweep.weight_grid(_args(w_ee="0.3,1", w_dur="0.1,1,2"))
    assert len(grid) == 6 and grid[0] == (0.4, 1.7, 0.3, 0.1, 0.1) and grid[1] == (0.4, 1.7, 0.3, 0.1, 1.0)
    assert grid[5] == (0.4, 1.7, 1.0, 0.1, 2.0)
    assert weight_sweep.weight_grid(_args()) == [(0.4, 1.7, 0.3, 0.1, 0.1)]
    n = 2 * len(grid)
    rng = np.random.default_rng(0)
    st = np.zeros((6, n), np.int32)
    st[5, ::2] = -9                                                   # stage 4 not run: the final iterate is stage 3's
    out = dict(stage_status=st, stage_iters=rng.integers(0, 99, (6, n)).astype(np.int32),
               success=np.ones((n, 2), np.int32), cost_terms=rng.random((n, 10)), stage_stats=rng.random((6, n, 4)))
    rows = weight_sweep.sweep_rows(out, ["a", "b"], grid)
    assert len(rows) == n and [r["clip"] for r in rows] == ["a"] * 6 + ["b"] * 6
    for i, r in enumerate(rows):
        assert r["setting"] == i % 6 and (r["w_ee"], r["w_dur"]) == grid[i % 6][2:5:2]
        assert [r[t] for t in chd.phys.COST_TERMS] == out["cost_terms"][i].tolist()
        fin = 4 if i % 2 == 0 else 5
        assert r["final_stage"] == ("3" if fin == 4 else "4") and r["final_error"] == out["stage_stats"][fin, i, 1]
        assert r["iters_2.2"] == out["stage_iters"][3, i]


class _TermsLib:
    """Stands in for libchd's queue: writes every clip's cost terms as (queue position, column) into the buffer set
    with chd_phys_set_cost_terms_out, and records the per-clip weights it was created with."""

    def __init__(self):
        self.terms_ptr, self.set_calls = None, []

    def chd_phys_queue_create(self, arr, n, slots, w, dev, opt, out):
        self.n, self.slots = n, min(slots, n)
        self.frames_in = [arr[k].n_frames for k in range(n)]
        self.weights = [tuple(getattr(opt._obj.clip_weights[k], f) for f, _ in opt._obj.clip_weights[k]._fields_)
                        for k in range(n)]
        out._obj.value = 1
        return 0

    def chd_phys_get_dims(self, h, d):
        d._obj.batch, d._obj.frames_out_max = self.slots, max(self.frames_in)
        return 0

    def chd_phys_set_cost_terms_out(self, h, p):
        self.terms_ptr = p
        self.set_calls.append(p is not None)
        return 0

    def chd_phys_queue_solve(self, h, *outs):
        if self.terms_ptr is not None:
            t = np.ctypeslib.as_array(C.cast(self.terms_ptr, C.POINTER(C.c_double)), shape=(self.n, 10))
            t[:] = np.arange(self.n)[:, None] * 100 + np.arange(10)
        return 0

    def chd_phys_batch_destroy(self, h):
        pass


def test_queue_terms_and_weights_follow_the_clips(chd, monkeypatch):
    """PhysQueue hands each clip's weights to the library in queue order and returns the terms in input order; the
    output pointer is cleared after the solve."""
    fake = _TermsLib()
    monkeypatch.setattr(chd.phys, "load_lib", lambda: fake)
    F = [50, 90, 40, 120, 70]
    ps = [chd.synth.make_problem(i, n_frames=f, n_ee=2) for i, f in enumerate(F)]
    W = [(0.1 * (i + 1), 1.0, 0.3, 0.1, 0.1) for i in range(5)]
    q = chd.phys.PhysQueue(ps, slots=2, weights=W)
    assert fake.weights == [W[i] for i in q.order]
    out = q.solve(cost_terms=True)
    pos = np.argsort(q.order)
    np.testing.assert_array_equal(out["cost_terms"], pos[:, None] * 100 + np.arange(10))
    assert fake.set_calls == [True, False]
    assert "cost_terms" not in q.solve()


N_MERGE = 9


def _fake_result(n):
    rng = np.random.default_rng(5)
    terms = rng.random((n, 10))
    terms[rng.random(terms.shape) < 0.2] = -0.0
    return dict(samples=rng.standard_normal((3, n, 5, 20)), frames=rng.integers(1, 6, n).astype(np.int32),
                success=rng.integers(0, 2, (n, 2)).astype(np.int32), stage_status=rng.integers(-3, 2, (6, n)).astype(np.int32),
                stage_iters=rng.integers(0, 3000, (6, n)).astype(np.int32), stage_stats=rng.standard_normal((6, n, 4)),
                cost_terms=terms)


def _merge_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import chd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ps = [chd.synth.make_problem(s, n_frames=40 + 3 * s, n_ee=2) for s in range(N_MERGE)]
    mine = np.random.default_rng(2).integers(0, world, N_MERGE) == rank
    mine[0] = rank == 1

    def solve_fn(problems):
        out = {k: v.copy() for k, v in _fake_result(len(problems)).items()}
        for k, ax in dict(samples=1, frames=0, success=0, stage_status=1, stage_iters=1, stage_stats=1, cost_terms=0).items():
            np.moveaxis(out[k], ax, 0)[~mine] = 0
        out["solved"] = mine
        return out

    s = chd.parallel.ShardedSolver(ps, weights=[SETTINGS[i % 4] for i in range(N_MERGE)], rank=rank, world=world,
                                   solve_fn=solve_fn, slots=3)
    out = s.solve(cost_terms=True)
    s.close()
    np.savez(os.path.join(tmp, "m%d.npz" % rank), **{k: v for k, v in out.items() if k != "d2h_bytes"})
    dist.destroy_process_group()


def test_merge_carries_the_terms_bitwise(tmp_path):
    import torch.multiprocessing as mp
    port = 37600 + (os.getpid() % 2000)
    mp.spawn(_merge_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(str(tmp_path / "m0.npz")), np.load(str(tmp_path / "m1.npz"))
    full = _fake_result(N_MERGE)
    for k in r0.files:
        assert r0[k].tobytes() == r1[k].tobytes(), k
    for k, v in full.items():
        assert r0[k].dtype == v.dtype and r0[k].tobytes() == v.tobytes(), k
    assert (np.signbit(r0["cost_terms"]) == np.signbit(full["cost_terms"])).all()


def test_merge_without_terms_keeps_its_row(chd):
    full = _fake_result(4)
    local = {k: v for k, v in full.items() if k != "cost_terms"}
    local["solved"] = np.ones(4, bool)
    out = chd.parallel.merge_solved(local, 1)
    assert "cost_terms" not in out
    assert out["d2h_bytes"] == 4 * (1 + 3 * 5 * 20 + chd.parallel.Q_EXTRA) * 8
    with_terms = chd.parallel.merge_solved(dict(full, solved=np.ones(4, bool)), 1)
    assert with_terms["d2h_bytes"] == 4 * (1 + 3 * 5 * 20 + chd.parallel.Q_EXTRA + 10) * 8


def test_unsharded_terms_need_slots(chd):
    ps = [chd.synth.make_problem(s, n_frames=40, n_ee=2) for s in range(2)]
    s = chd.parallel.ShardedSolver(ps, solve_fn=lambda p: None, tensor_device=None)
    with pytest.raises(ValueError, match="slots"):
        s.solve(cost_terms=True)
