"""CPU tests of per-clip solver options (chd_phys_options.clip_options, `chd.phys.SolverOptions`, the `options` of
PhysBatch / PhysQueue / ShardedSolver, the option flags of phys_optim.py and weight_sweep.py) on host-only layouts, and of
the files write_outputs writes for a clip that stopped early."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")
STAGE_CAPS = (7000, 7000, 7000, 2500, 2000, 7000)   # phys_optim.cpp's caps of stages 1.1 .. 4


def _problems(chd, n=3):
    return [chd.synth.make_problem(s, n_frames=40 + 5 * s, n_ee=2) for s in range(n)]


def test_defaults_resolve_to_the_reference(chd):
    """Without options, and with explicit default ones, every sequence reports phys_optim's tolerances and caps, and
    the stage table is the same."""
    P = chd.phys
    ps = _problems(chd)
    none = P.PhysBatch(ps, host_only=True)
    explicit = P.PhysBatch(ps, host_only=True, options=P.SolverOptions())
    ref = P.SolverOptions(1e-3, 1e-4, 1.0, 1e-4, STAGE_CAPS, "durations")
    assert none.solver_options() == [ref] * 3 == explicit.solver_options()
    np.testing.assert_array_equal(none.stage_weights(), explicit.stage_weights())


def test_each_sequence_keeps_its_options(chd):
    """Mixed options: every sequence reports its own, caps of 0 resolved to the stage's own; the weights and every layout
    table are those of a batch without options; a queue's slots report the options of its first clips in queue order."""
    P = chd.phys
    ps = _problems(chd, 4)
    opts = [P.SolverOptions(tol=1e-2, last_stage="no_dynamics"),
            P.SolverOptions(constr_viol_tol=1e-6, dual_inf_tol=0.5, compl_inf_tol=1e-5, max_iter=(0, 0, 0, 7, 0, 0)),
            P.SolverOptions(max_iter=(11, 12, 13, 14, 15, 16), last_stage="dynamics"),
            P.SolverOptions(tol=1e-4)]
    b = P.PhysBatch(ps, host_only=True, options=opts)
    plain = P.PhysBatch(ps, host_only=True)
    got = b.solver_options()
    for o, g in zip(opts, got):
        caps = tuple(k or d for k, d in zip(o.max_iter, STAGE_CAPS))
        assert g == P.SolverOptions(o.tol, o.constr_viol_tol, o.dual_inf_tol, o.compl_inf_tol, caps, o.last_stage)
    np.testing.assert_array_equal(b.stage_weights(), plain.stage_weights())
    for x, y in ((b.layout(), plain.layout()), (b.slot_index(), plain.slot_index())):
        for k in x:
            np.testing.assert_array_equal(x[k], y[k], err_msg=k)
    # a queue: options travel in queue (work-estimate) order with the clips
    order = np.argsort(-np.asarray(chd.parallel.work_estimate(ps)), kind="stable")
    arr, _ = P.make_problem_array([ps[i] for i in order])
    w, opt, keep = P._create_args(P.DEFAULT_WEIGHTS, 4, None, order, opts)
    h = C.c_void_p()
    L = P.load_lib()
    assert L.chd_phys_queue_create(arr, 4, 2, w, -2, opt, C.byref(h)) == 0
    try:
        out = (P._SolverOptions * 2)()
        assert L.chd_phys_get_solver_options(h, out) == 0
        assert [o.value() for o in out] == [got[i] for i in order[:2]]
    finally:
        L.chd_phys_batch_destroy(h)


BAD = [dict(tol=0.0), dict(tol=-1e-3), dict(tol=float("nan")), dict(constr_viol_tol=float("inf")),
       dict(dual_inf_tol=0.0), dict(compl_inf_tol=-float("inf")), dict(max_iter=(0, 0, 0, -1, 0, 0)),
       dict(max_iter=(-5, 0, 0, 0, 0, 0))]


@pytest.mark.parametrize("bad", BAD, ids=[str(b) for b in BAD])
def test_bad_options_are_refused(chd, bad):
    """A tolerance that is not finite or not > 0, or a negative cap, in any clip: -1 from the batch and the queue."""
    P = chd.phys
    L = P.load_lib()
    ps = _problems(chd)
    arr, _ = P.make_problem_array(ps)
    opts = [P.SolverOptions(), P.SolverOptions(**bad), P.SolverOptions(tol=1e-2)]
    w, opt, keep = P._create_args(P.DEFAULT_WEIGHTS, 3, None, options=opts)
    h = C.c_void_p()
    assert L.chd_phys_batch_create(arr, 3, w, -2, opt, C.byref(h)) == -1
    assert L.chd_phys_queue_create(arr, 3, 2, w, -2, opt, C.byref(h)) == -1
    with pytest.raises(RuntimeError, match="code -1"):
        P.PhysBatch(ps, host_only=True, options=opts)


@pytest.mark.parametrize("last", [-1, 3, 99])
def test_unknown_last_stage_is_refused(chd, last):
    P = chd.phys
    L = P.load_lib()
    ps = _problems(chd, 2)
    arr, _ = P.make_problem_array(ps)
    rec = (P._SolverOptions * 2)(P._SolverOptions.of(P.SolverOptions()), P._SolverOptions.of(P.SolverOptions()))
    rec[1].last_stage = last
    opt = P._Options(-1, None, C.cast(rec, C.POINTER(P._SolverOptions)))
    h = C.c_void_p()
    assert L.chd_phys_batch_create(arr, 2, None, -2, C.byref(opt), C.byref(h)) == -1
    assert L.chd_phys_queue_create(arr, 2, 1, None, -2, C.byref(opt), C.byref(h)) == -1
    with pytest.raises(ValueError, match="last_stage"):
        P.SolverOptions(last_stage="preview")


def test_option_lists_are_checked(chd):
    P = chd.phys
    assert P.clip_options(None, 3) is None
    assert P.clip_options(P.SolverOptions(tol=0.1), 2) == [P.SolverOptions(tol=0.1)] * 2
    for bad in ([P.SolverOptions()] * 2, [P.SolverOptions(), None, P.SolverOptions()], (1e-3,)):
        with pytest.raises(ValueError):
            P.clip_options(bad, 3)
    with pytest.raises(ValueError, match="max_iter"):
        P.SolverOptions(max_iter=(1, 2, 3))


def _args(**kw):
    import argparse
    sys.path.insert(0, SCRIPTS)
    import phys_optim
    ap = argparse.ArgumentParser()
    phys_optim.add_option_flags(ap)
    return ap.parse_args(sum([["--" + k, v] for k, v in kw.items()], []))


def test_phys_optim_option_lists(chd):
    sys.path.insert(0, SCRIPTS)
    import phys_optim
    S = chd.phys.SolverOptions
    assert phys_optim.parse_options(_args(), 3) is None                     # no flag: the library's defaults
    assert phys_optim.parse_options(_args(tol="0.01"), 2) == [S(tol=0.01)] * 2
    got = phys_optim.parse_options(_args(**{"tol": "0.01,0.001,0.0001", "last_stage": "dynamics,durations,no_dynamics",
                                            "max_iter_3": "50", "max_iter_2.2": "0,7,9", "compl_inf_tol": "1e-5"}), 3)
    assert got == [S(tol=0.01, compl_inf_tol=1e-5, max_iter=(0, 0, 0, 0, 50, 0), last_stage="dynamics"),
                   S(tol=0.001, compl_inf_tol=1e-5, max_iter=(0, 0, 0, 7, 50, 0), last_stage="durations"),
                   S(tol=0.0001, compl_inf_tol=1e-5, max_iter=(0, 0, 0, 9, 50, 0), last_stage="no_dynamics")]
    with pytest.raises(ValueError, match="tol"):
        phys_optim.parse_options(_args(tol="0.1,0.2"), 3)
    with pytest.raises(ValueError, match="last_stage"):
        phys_optim.parse_options(_args(last_stage="dynamics,later"), 2)


def test_weight_sweep_options(chd):
    import argparse
    sys.path.insert(0, SCRIPTS)
    import weight_sweep
    S = chd.phys.SolverOptions
    ns = lambda **kw: argparse.Namespace(**dict(dict(tol=None, last_stage=None), **kw))
    assert weight_sweep.sweep_options(ns()) is None
    assert weight_sweep.sweep_options(ns(tol=0.01, last_stage="dynamics")) == S(tol=0.01, last_stage="dynamics")
    st = np.full(6, -9, np.int32)
    st[:4] = 0
    assert weight_sweep.final_stage(st) == 3                                 # stopped after 2.2
    st[4] = -1
    st[5] = 0
    assert weight_sweep.final_stage(st) == 5


@pytest.mark.parametrize("last", ["no_dynamics", "dynamics", "durations"])
def test_write_outputs_writes_the_snapshots_taken(chd, tmp_path, last):
    """A clip stopped after `last` writes the solution files of the snapshots it took and always success_log.txt, with 0
    for a stage that did not run."""
    P = chd.phys
    p = chd.synth.make_problem(1, n_frames=40, n_ee=2)
    nf = 10
    k = P.LAST_STAGES.index(last)
    out = P.result_arrays(1, P.SOLVE_KEYS, nf, P.sample_stride(2))
    out["frames"][0] = nf
    out["samples"][:] = 1.0
    out["samples"][k + 1:] = np.nan
    ran = [2, 4, 6][k]                                                       # stages 1.1 .. 1.2 / 2.2 / 4 ran
    out["stage_status"][:, 0] = [0] * ran + [-9] * (6 - ran)
    if last == "durations":
        out["stage_status"][4:, 0] = (-1, 0)                                 # stage 3 capped, stage 4 converged
    out["success"][0] = (out["stage_status"][3, 0] == 0, 1 if last == "durations" else 0)
    P.write_outputs(out, 0, p, str(tmp_path), 2)
    assert sorted(os.listdir(tmp_path)) == sorted(list(P.SOLUTION_FILES[:k + 1]) + ["success_log.txt"])
    log = open(tmp_path / "success_log.txt").read()
    assert log == "dynamics %d\ndurations %d\n" % (last != "no_dynamics", last == "durations")
    assert P.snapshots_taken(out, 0) == [s <= k for s in range(3)]
