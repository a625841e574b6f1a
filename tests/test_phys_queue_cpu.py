"""CPU tests of the physics solve queue (`chd_phys_queue_create`, `chd.phys.PhysQueue`): argument checks, the slot-sized
layout of a host-only queue handle, and the queue order / un-permutation of `PhysQueue` against a stand-in library."""
import ctypes as C

import numpy as np
import pytest

from tests.util import QueueLib


def _create(chd, problems, n, slots, device=-2, band=None):
    P = chd.phys
    L = P.load_lib()
    arr, keep = P.make_problem_array(problems) if problems else (None, None)
    h = C.c_void_p()
    opt = None if band is None else C.byref(P._Options(band))
    rc = L.chd_phys_queue_create(arr, n, slots, None, device, opt, C.byref(h))
    return rc, h


def test_queue_create_rejects_bad_arguments(chd):
    ps = [chd.synth.make_problem(s) for s in range(3)]
    assert _create(chd, None, 3, 2)[0] == -1
    assert _create(chd, ps, 0, 2)[0] == -1
    assert _create(chd, ps, -1, 2)[0] == -1
    assert _create(chd, ps, 3, 0)[0] == -1
    assert _create(chd, ps, 3, -4)[0] == -1
    assert _create(chd, ps, 3, 2, band=97)[0] == -1
    L = chd.phys.load_lib()
    assert L.chd_phys_queue_create(chd.phys.make_problem_array(ps)[0], 3, 2, None, -2, None, None) == -1


@pytest.mark.parametrize("slots", [1, 2, 5, 9])
def test_host_only_queue_has_slot_rows_and_clip_strides(chd, slots):
    """A queue's batch dimension is its slot count (clamped to n); its strides are those of a batch of all n clips, so
    every clip fits every slot.  Calls that address slots return -1 on it."""
    P = chd.phys
    L = P.load_lib()
    ps = [chd.synth.make_problem(0, n_frames=40, n_ee=2), chd.synth.make_problem(1, n_frames=120, n_ee=4),
          chd.synth.make_problem(2, n_frames=80, n_ee=2), chd.synth.make_problem(3, n_frames=60, n_ee=4, dense=True),
          chd.synth.make_problem(4, n_frames=100, n_ee=2)]
    rc, h = _create(chd, ps, len(ps), slots)
    assert rc == 0
    try:
        d = P._Dims()
        assert L.chd_phys_get_dims(h, C.byref(d)) == 0
        full = P.PhysBatch(ps, host_only=True)
        S = min(slots, len(ps))
        assert d.batch == S
        for k, _ in P._Dims._fields_:
            if k != "batch":
                assert getattr(d, k) == full.dims[k], k
        sz = np.zeros((S, 6), np.int32)
        assert L.chd_phys_get_sizes(h, sz.ctypes.data_as(C.c_void_p)) == 0
        np.testing.assert_array_equal(sz, full.sizes[:S])
        buf = np.zeros(len(ps) * full.dims["n_max"] * full.dims["frames_out_max"] * 40 * 3)
        p = buf.ctypes.data_as(C.c_void_p)
        assert L.chd_phys_get_x(h, p) == -1
        assert L.chd_phys_set_x(h, p) == -1
        assert L.chd_phys_eval(h, 0, p, None, None, None) == -1
        assert L.chd_phys_solve_stage(h, 0, 0, None, None, None) == -1
        assert L.chd_phys_solve(h, p, None, None, None, None) == -1
        assert L.chd_phys_sample(h, p, None) == -1
        assert L.chd_phys_sample_device(h, p, None) == -1
        assert L.chd_phys_reset(h) == -1
        assert L.chd_phys_get_duals(h, p, None, None, None, None, None) == -1
        assert L.chd_phys_queue_solve(h, p, None, None, None, None, None) == -1      # host-only: nothing to run
    finally:
        L.chd_phys_batch_destroy(h)


def test_batch_handle_refuses_queue_solve(chd):
    b = chd.phys.PhysBatch([chd.synth.make_problem(0)], host_only=True)
    assert b.L.chd_phys_queue_solve(b.h, None, None, None, None, None, None) == -1


def test_queue_orders_by_work_and_returns_input_order(chd, monkeypatch):
    fake = QueueLib()
    monkeypatch.setattr(chd.phys, "load_lib", lambda: fake)
    F = [50, 90, 40, 120, 90, 70]
    ps = [chd.synth.make_problem(i, n_frames=f, n_ee=2) for i, f in enumerate(F)]
    q = chd.phys.PhysQueue(ps, slots=4)
    est = chd.parallel.work_estimate(ps)
    expect = sorted(range(len(ps)), key=lambda i: (-est[i], i))
    assert fake.frames_in == [F[i] for i in expect]              # the library sees the longest clips first
    assert q.slots == 4
    out = q.solve()
    pos = {i: k for k, i in enumerate(expect)}                     # queue position of every input clip
    for i, f in enumerate(F):
        assert out["frames"][i] == f
        assert (out["samples"][:, i, :f, 0] == f).all() and (out["samples"][:, i, f:, 0] == 0).all()
        assert (out["stage_status"][:, i] == pos[i]).all() and (out["stage_iters"][:, i] == f).all()
        assert tuple(out["success"][i]) == (pos[i], f)
        assert (out["stage_stats"][:, i] == f).all()
    assert out["samples"].shape == (3, len(F), max(F), 20) and out["stage_stats"].shape == (6, len(F), 4)
