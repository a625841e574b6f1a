"""File-format tests at the reference's process/file boundary (towr_utils.py:51-122,435-449,585-777;
phys_optim.cpp:63-267)."""
import os

import numpy as np


def test_find_contact_durations_reference_semantics(chd):
    f = chd.io_formats.find_contact_durations
    dt = 1.0 / 30
    c = np.array([1, 1, 1, 0, 0, 1, 1, 1, 1, 0])
    d = f(c, dt)
    # the last frame is ignored, runs are 3,2,4 frames (towr_utils.py:435-449)
    np.testing.assert_allclose(d, [3 * dt, 2 * dt, 4 * dt])
    assert abs(sum(d) - (len(c) - 1) * dt) < 1e-12
    assert f(np.ones(5), dt) == [4 * dt] or abs(f(np.ones(5), dt)[0] - 4 * dt) < 1e-15


def test_input_files_round_trip(chd, tmp_path):
    for n_ee in (2, 4):
        p = chd.synth.make_problem(7, n_frames=60, n_ee=n_ee)
        d = str(tmp_path / ("in%d" % n_ee))
        chd.io_formats.write_phys_inputs(p, d)
        for name in ("skel_info.txt", "motion_info.txt", "terrain_info.txt", "contact_info.txt"):
            assert os.path.exists(os.path.join(d, name))
        q = chd.io_formats.read_phys_inputs(d, 60, n_ee=n_ee)
        # python repr(float) round-trips exactly
        for a in ("hip_left", "hip_right", "inertia", "base_lin", "base_ang", "ee_pos", "floor_normal", "floor_point"):
            np.testing.assert_array_equal(getattr(p, a), getattr(q, a))
        assert (p.dt, p.max_leg_length, p.max_heel_length, p.heel_dist, p.body_mass) == \
               (q.dt, q.max_leg_length, q.max_heel_length, q.heel_dist, q.body_mass)
        assert list(p.ee_start_contact) == list(q.ee_start_contact)
        for a, b in zip(p.ee_durations, q.ee_durations):
            np.testing.assert_array_equal(a, b)
    # motion_info.txt layout: dt line + 6 lines of F*3 numbers (towr_utils.py:640-683)
    lines = open(os.path.join(d, "motion_info.txt")).read().strip().split("\n")
    assert len(lines) == 7 and all(len(l.split()) == 180 for l in lines[1:])


def test_solution_file_layout(chd, tmp_path):
    rng = np.random.default_rng(0)
    n_ee, N = 4, 17
    base, _, frc, flag = chd.phys.sample_columns(n_ee, n_ee)
    s = rng.normal(size=(N, chd.phys.sample_stride(n_ee)))
    s[:, flag] = rng.integers(0, 2, size=(N, n_ee))
    path = str(tmp_path / "sol_out_dynamics.txt")
    chd.io_formats.write_solution(path, 1.0 / 30, s, n_ee)
    lines = open(path).read().split("\n")
    # label / value alternation that towr_utils.load_results indexes by line number (towr_utils.py:64-98)
    assert lines[0] == "dt" and lines[2] == "num_frames" and lines[4] == "num_feet" and lines[6] == "base_lin"
    assert lines[8] == "base_ang" and lines[10] == "foot0_pos" and lines[10 + 2 * n_ee] == "foot0_force"
    assert lines[10 + 4 * n_ee] == "foot0_contact"
    assert not lines[7].endswith(" ") and len(lines[7].split()) == 3 * N
    r = chd.io_formats.read_solution(path)
    assert r["num_frames"] == N and r["num_feet"] == n_ee
    np.testing.assert_allclose(r["base_lin"], s[:, base[:3]], rtol=1e-9)       # 10 significant digits
    np.testing.assert_allclose(r["foot_force"][2], s[:, frc[6:9]], rtol=1e-9)
    np.testing.assert_array_equal(r["foot_contact"][3], s[:, flag[3]].astype(np.int64))
    chd.io_formats.write_success_log(str(tmp_path / "success_log.txt"), True, False)
    assert open(str(tmp_path / "success_log.txt")).read() == "dynamics 1\ndurations 0\n"
