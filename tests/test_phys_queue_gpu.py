"""GPU tests of the physics solve queue (`chd.phys.PhysQueue`, `chd_phys_queue_solve`): clips streamed through fewer
device slots than clips give, clip by clip, the results of one `PhysBatch` of the same clips (which has the same
strides), also where a slot passes from a longer, 4-foot or stage-3-rewritten clip to a shorter 2-foot one."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.util import assert_samples_close, assert_solves_agree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _agree(chd, ps, slots, n_ee, band=None):
    ref = chd.phys.PhysBatch(ps, stage3_band_above=band).solve()
    q = chd.phys.PhysQueue(ps, slots, stage3_band_above=band)
    got = q.solve()
    assert q.slots == min(slots, len(ps))
    assert_solves_agree(ref, got, n_ee)
    np.testing.assert_array_equal(got["frames"], ref["frames"])
    np.testing.assert_array_equal(got["success"], ref["success"])
    return q, ref, got


def test_mixed_lengths_through_eight_slots(chd):
    F = [40 + (37 * i) % 81 for i in range(24)]                  # 40 .. 120 frames
    ps = [chd.synth.make_problem(i, n_frames=f, n_ee=2) for i, f in enumerate(F)]
    q, _, got = _agree(chd, ps, 8, 2)
    _, n = q.kernel_times()["admit"]
    assert n >= 1 + (24 - 8) // 8                                  # refilled at check points, several slots at a time
    assert (got["stage_stats"][3, :, 1] <= 1e-3).all()           # stage 2.2 converged: scaled NLP error within tol


@pytest.mark.parametrize("slots", [1, 3, 10])
def test_one_slot_and_more_slots_than_clips(chd, slots):
    ps = [chd.synth.make_problem(20 + i, n_frames=f, n_ee=2) for i, f in enumerate((60, 100, 45))]
    q, _, _ = _agree(chd, ps, slots, 2)
    assert q.slots == min(slots, 3)


def test_refilled_slot_keeps_nothing_of_its_previous_clip(chd):
    """Slots pass from a 200-frame 4-foot densely switching clip (more than 96 phase durations: stage 3 not attempted,
    status -3) and from 120-frame 2-foot clips whose stage 3 moved their switch times (spline tables and Jacobian
    columns rewritten on the device) to short 2-foot clips."""
    ps = [chd.synth.make_problem(0, n_frames=200, n_ee=4, dense=True)]
    ps += [chd.synth.make_problem(s, n_frames=120, n_ee=2) for s in (1, 2)]
    ps += [chd.synth.make_problem(30 + s, n_frames=40 + 8 * s, n_ee=2) for s in range(7)]
    q, ref, got = _agree(chd, ps, 2, 4)
    assert ref["stage_status"][4, 0] == -3
    assert (ref["stage_status"][4, 1:3] == 0).all()              # stage 3 ran and moved the durations
    # queue order: the dense clip, the two 120-frame clips, then the short ones, which take over the slots they held
    order = q.order.tolist()
    assert order[0] == 0 and set(order[:3]) == {0, 1, 2}


def test_banded_switch_times(chd):
    ps = [chd.synth.make_problem(40 + i, n_frames=f, n_ee=2) for i, f in enumerate((120, 60, 90, 45, 110, 75))]
    _agree(chd, ps, 2, 2, band=0)


def test_second_solve_starts_over(chd):
    ps = [chd.synth.make_problem(50 + i, n_frames=f, n_ee=2) for i, f in enumerate((80, 50, 120, 65, 100))]
    q = chd.phys.PhysQueue(ps, 2)
    a, b = q.solve(), q.solve()
    np.testing.assert_array_equal(a["stage_status"], b["stage_status"])
    np.testing.assert_array_equal(a["stage_iters"][:4], b["stage_iters"][:4])
    np.testing.assert_array_equal(a["frames"], b["frames"])
    for i, p in enumerate(ps):
        nf = a["frames"][i]
        assert_samples_close(b["samples"][1, i, :nf], a["samples"][1, i, :nf], 2)


def test_slot_addressed_calls_refused(chd):
    ps = [chd.synth.make_problem(60 + i, n_frames=50, n_ee=2) for i in range(3)]
    q = chd.phys.PhysQueue(ps, 2)
    L, h, d = q.L, q.h, q.dims
    buf = np.zeros(3 * 3 * d["n_max"] * d["frames_out_max"] * 20)
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
    assert q.solve()["frames"].tolist() == [50, 50, 50]              # the handle still solves


def _rows(chd, path):
    r = chd.io_formats.read_solution(path)
    n = r["num_frames"]
    cat = lambda a: a.transpose(1, 0, 2).reshape(n, -1)
    return np.concatenate([r["base_lin"], r["base_ang_deg"], cat(r["foot_pos"]), cat(r["foot_force"]),
                           r["foot_contact"].T.astype(np.float64)], axis=1), r["num_feet"]


def test_phys_optim_slots_matches_batch(chd, tmp_path):
    """scripts/phys_optim.py --slots 2 on the three golden clips (4 feet) writes what the batch run writes: the files of
    stages 1.1-2.2 for every clip, the final one and the success log where stages 3 and 4 ended the same way.  On these
    clips stage 3 runs for up to its 2000-iteration cap, a path long enough for the run-to-run rounding of the kernels'
    fp64 atomic sums (DESIGN §7) to change how stages 3 and 4 end: two batch runs of them differ there too."""
    import json
    import re
    cases = {"combined": 38, "ybot": 36, "ybot_noheel": 36}
    ind = ",".join(os.path.join(ROOT, "tests", "golden", "towr", c, "phys_in") for c in cases)
    nfr = ",".join(str(f) for f in cases.values())
    runs, logs = {}, {}
    for tag, extra in (("batch", []), ("queue", ["--slots", "2"])):
        outs = [str(tmp_path / tag / c) for c in cases]
        for o in outs:
            os.makedirs(o)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "phys_optim.py"), "--in_dir", ind,
                            "--nframes", nfr, "--out_dir", ",".join(outs)] + extra, check=True, capture_output=True, text=True)
        print(r.stdout)
        logs[tag] = [(json.loads(m.group(1)), json.loads(m.group(2)))
                     for m in re.finditer(r"stages status (\[.*?\]) iterations (\[.*?\])", r.stdout)]
        runs[tag] = outs
    assert len(logs["batch"]) == len(logs["queue"]) == len(cases)
    for (sa, ia), (sb, ib), a, b in zip(logs["batch"], logs["queue"], runs["batch"], runs["queue"]):
        assert sa[:4] == sb[:4] and ia[:4] == ib[:4]
        names = list(chd.phys.SOLUTION_FILES[:2])
        if sa == sb and ia == ib:
            names.append(chd.phys.SOLUTION_FILES[2])
            assert open(os.path.join(a, "success_log.txt")).read() == open(os.path.join(b, "success_log.txt")).read()
        for name in names:
            exp, ne = _rows(chd, os.path.join(a, name))
            got, _ = _rows(chd, os.path.join(b, name))
            assert_samples_close(got, exp, ne)
