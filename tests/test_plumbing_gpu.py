"""BASELINE.json configs[0] ("single clip: contact detect + phys_optim", plumbing): the two drop-in scripts chained
through the reference's own files -- openpose_result/*.json -> foot_contacts.npy -> contact_info.txt (+ the three
other phys_optim inputs) -> sol_out_*.txt / success_log.txt.  First test: the motion side of the clip is synthetic
(chd.synth) and a 5-frame majority filter stands in for the label clean-up; second test: the step in between
(towr_utils.prepare_input, chd.prepare) turns a BVH clip + floor file + foot_contacts.npy into the four input files."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))


def test_single_clip_files_end_to_end(chd, tmp_path):
    from make_contact_golden import contact_weights, synth_keypoints
    F, fps = 101, 24.0                                   # dance2's shape (SURVEY 8(d))
    data, out = tmp_path / "data", tmp_path / "out"
    op = data / "clip" / "openpose_result"
    os.makedirs(op)
    kp = synth_keypoints(7, F)
    for i in range(F):
        people = [] if i == 40 else [{"pose_keypoints_2d": kp[i].reshape(-1).tolist()}]   # one frame without a detection
        with open(op / ("clip_%012d_keypoints.json" % i), "w") as f:
            json.dump({"version": 1.2, "people": people}, f)
    np.savez(tmp_path / "weights.npz", **contact_weights(0))
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "detect_contacts.py"), "--data", str(data), "--out", str(out),
                           "--weights-path", str(tmp_path / "weights.npz"), "--full-video", "--save-contacts", "--real-data",
                           "--copy-into-data"])
    labels = np.load(data / "clip" / "foot_contacts.npy")
    assert labels.shape == (F, 4) and labels.dtype == np.int64 and set(np.unique(labels)) <= {0, 1}
    np.testing.assert_array_equal(labels, np.load(out / "contact_results" / "clip" / "foot_contacts.npy"))

    # label clean-up stand-in: 5-frame majority vote on the toe columns (L toe = 1, R toe = 3), a stance at both ends
    toe = labels[:, [1, 3]].T.astype(np.int64)
    pad = np.pad(toe, ((0, 0), (2, 2)), mode="edge")
    toe = (sum(pad[:, k:k + F] for k in range(5)) >= 3).astype(np.int64)
    toe[:, :3], toe[:, -3:] = 1, 1
    p = chd.synth.make_problem(7, n_frames=F, n_ee=2, fps=fps, toe_flags=toe)
    ind, outd = tmp_path / "phys_optim_in_ybot", tmp_path / "phys_optim_out_ybot"
    os.makedirs(outd)
    chd.io_formats.write_phys_inputs(p, str(ind))
    # contact_info.txt carries exactly the phases of the detected labels (towr_utils.py:435-449)
    for e in range(2):
        np.testing.assert_allclose(p.ee_durations[e], chd.io_formats.find_contact_durations(list(toe[e]), 1.0 / fps))
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "phys_optim.py"), "--in_dir", str(ind), "--nframes", str(F),
                           "--out_dir", str(outd), "--n_ee", "2"])
    sols = {}
    for name in ("sol_out_no_dynamics.txt", "sol_out_dynamics.txt", "sol_out_durations.txt"):
        r = chd.io_formats.read_solution(str(outd / name))
        assert r["num_frames"] == F and r["num_feet"] == 2
        assert all(np.isfinite(np.asarray(v, float)).all() for v in r.values() if isinstance(v, np.ndarray))
        sols[name] = r
    log = open(outd / "success_log.txt").read().split()
    assert log[0] == "dynamics" and log[2] == "durations" and log[1] in "01" and log[3] in "01"
    # the written contact flags are the detected phases sampled at the frame times (boundary frames may go either way)
    flags = sols["sol_out_durations.txt"]["foot_contact"].T        # (F, 2)
    interior = np.ones(F, bool)
    for e in range(2):
        ch = np.flatnonzero(np.diff(toe[e]) != 0)
        interior[ch] = False
        interior[ch + 1] = False
    interior[-1] = False
    np.testing.assert_array_equal(flags[interior], toe.T[interior])


def test_bvh_clip_through_prepare_input(chd, tmp_path):
    """BVH clip -> chd.prepare.prepare_input (FK, COM, hip offsets, inertia, contact schedule) -> phys_optim_in_* ->
    scripts/phys_optim.py -> phys_optim_out_* -> chd.prepare.load_results (towr_utils.py:451-777, 51-122)."""
    P = chd.prepare
    F = 90
    bvh = str(tmp_path / "walk.bvh")
    P.write_test_bvh(bvh, F, seed=1)
    with open(tmp_path / "floor_out.txt", "w") as f:
        f.write("0.0 -1.0 0.0\n0.0 0.0 0.0\n")
    t = np.arange(F)
    period = 33                                           # frames per stride of the generated clip (0.9 Hz at 30 fps)
    fc = np.zeros((F, 4), np.int64)                       # L heel, L toe, R heel, R toe
    for col, shift in ((0, 0), (1, 2), (2, period // 2), (3, period // 2 + 2)):
        fc[:, col] = ((t + shift) % period) < 20
    fc[:2], fc[-3:] = fc[2], fc[-4]
    np.save(tmp_path / "foot_contacts.npy", fc)
    ind, outd = str(tmp_path / "phys_optim_in_biped"), str(tmp_path / "phys_optim_out_biped")
    os.makedirs(outd)
    p = P.prepare_input(bvh, str(tmp_path / "floor_out.txt"), str(tmp_path / "foot_contacts.npy"), ind, P.simple_biped_info())
    assert p.n_frames == F and p.n_ee == 4
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "phys_optim.py"), "--in_dir", ind, "--nframes", str(F),
                           "--out_dir", outd])
    r = P.load_results(outd)
    assert set(r) == {"no_dynamics", "dynamics", "durations", "success"}
    for key in ("no_dynamics", "dynamics", "durations"):
        assert r[key]["num_frames"] == F and r[key]["num_feet"] == 4
        assert all(np.isfinite(np.asarray(v, float)).all() for v in r[key].values() if isinstance(v, np.ndarray))
    # the kinematic stage tracks the prepared COM (z up, metres)
    assert np.abs(r["no_dynamics"]["base_lin"] - p.base_lin).mean() < 0.1


def test_run_phys_mocap_whole_chain(chd, tmp_path):
    """The reference's driver scripts/run_phys_mocap.py end to end on two synthetic video directories (configs[0] `single
    example_data clip (plumbing)`, SURVEY.md 8(d)): OpenPose JSON + MTC json + contact labels -> kinematic initialisation
    (torch on the GPU) -> phys_optim_in_* -> ONE batched staged solve (libchd) -> sol_out_* -> IK back onto the skeleton ->
    BVH files."""
    data = tmp_path / "data"
    gts = {}
    for name, F, seed in (("clipA", 40, 1), ("clipB", 48, 2)):
        gts[name] = (F, chd.synth.write_mocap_clip(str(data / name), F, seed=seed))
    skel = str(data / "clipA" / "skeleton.bvh")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "run_phys_mocap.py"), "--data", str(data), "--character", "combined",
                           "--skel_path", skel, "--fps", "30"])
    for name, (F, gt) in gts.items():
        vd = data / name
        for f in ("foot_contacts.npy", "floor_out.txt", "final_test.bvh", "combined_out.bvh"):
            assert (vd / "kinematic_results" / f).exists(), f
        for f in ("skel_info.txt", "motion_info.txt", "terrain_info.txt", "contact_info.txt"):
            assert (vd / "phys_optim_in_combined" / f).exists(), f
        out = vd / "phys_optim_out_combined"
        log = open(out / "success_log.txt").read().split()
        assert log[0] == "dynamics" and log[2] == "durations" and log[1] in "01" and log[3] in "01"
        for tag in ("no_dynamics", "dynamics", "durations"):
            r = chd.results.load_towr_results(str(out / ("sol_out_%s.txt" % tag)))
            assert r.num_feet == 4 and r.base_pos.shape == (F, 3) and np.isfinite(r.feet_pos).all()
            b = chd.prepare.load_bvh(str(out / ("%s_combined_%s.bvh" % (name, tag))))
            assert b.n_frames == F and len(b.names) == 28
            # the applied skeleton follows the optimised COM track: root within the body's extent of it (cm, BVH frame)
            R, T = chd.prepare.local_transforms(b)
            gp, _ = chd.prepare.forward_kinematics(b.parents, R, T)
            assert np.linalg.norm(gp[:, 0] - r.base_pos * 100.0, axis=1).max() < 40.0
            # the toes were pulled onto the optimised foot trajectories
            assert np.linalg.norm(gp[:, 5] - r.feet_pos[:, 0] * 100.0, axis=1).mean() < 3.0
        # kinematic stage of the physics solve stays near the kinematic initialisation (metres)
        r0 = chd.results.load_towr_results(str(out / "sol_out_no_dynamics.txt"))
        p = chd.io_formats.read_phys_inputs(str(vd / "phys_optim_in_combined"), F)
        com_bvh = -p.base_lin[:, [0, 2, 1]]
        assert np.abs(r0.base_pos - com_bvh).mean() < 0.05


def test_torch_batched_solvers_same_on_gpu_and_cpu(chd, tmp_path):
    """The kinematic optimiser with its IK initialisation (on cuda:0 through `chd_kin_solve` and `chd_ik_solve`): same
    numbers on cuda:0 and on the host."""
    import torch
    assert torch.cuda.is_available()
    vd = str(tmp_path / "w")
    chd.synth.write_mocap_clip(vd, 24, seed=5)
    outs = []
    for dev in (None, "cuda:0"):
        res = chd.kinopt.optimize_2d_3d(os.path.join(vd, "w.mp4"), os.path.join(vd, "skeleton.bvh"), str(tmp_path / ("k_%s" % dev)), 0, 24, device=dev)
        outs.append(res)
    c0, c1 = outs[0][-1]["stage2"]["cost"], outs[1][-1]["stage2"]["cost"]
    assert abs(c0 - c1) < 1e-3 * c0
    assert np.linalg.norm(outs[0][1] - outs[1][1], axis=-1).max() < 0.5        # cm; 100 LM evaluations amplify rounding differences
    np.testing.assert_allclose(outs[0][3], outs[1][3], atol=1e-3)              # floor normal


def test_run_phys_mocap_retargeted_character(chd, tmp_path):
    """Same chain with `--character ybot`: re-targeting onto a 67-joint skeleton, heel joints added for the physics inputs and
    the IK, removed again before the BVH is saved (run_phys_mocap.py:117-201, towr_utils.py:972-975)."""
    data = tmp_path / "data"
    F = 36
    chd.synth.write_mocap_clip(str(data / "clipC"), F, seed=4)
    skel = str(data / "clipC" / "skeleton.bvh")
    ybot = os.path.join(ROOT, "tests", "golden", "towr", "retarget", "ybot_skel.bvh")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "run_phys_mocap.py"), "--data", str(data), "--character", "ybot",
                           "--skel_path", skel, "--character_skel", ybot, "--fps", "30"])
    vd = data / "clipC"
    assert (vd / "kinematic_results" / "ybot_out.bvh").exists()
    assert chd.io_formats.read_phys_inputs(str(vd / "phys_optim_in_ybot"), F).n_ee == 4
    out = vd / "phys_optim_out_ybot"
    for tag in ("no_dynamics", "dynamics", "durations"):
        r = chd.results.load_towr_results(str(out / ("sol_out_%s.txt" % tag)))
        b = chd.prepare.load_bvh(str(out / ("clipC_ybot_%s.bvh" % tag)))
        assert b.n_frames == F and len(b.names) == 67                      # heels removed again
        gp, _ = chd.prepare.forward_kinematics(b.parents, *chd.prepare.local_transforms(b))
        assert np.linalg.norm(gp[:, 65] - r.feet_pos[:, 0] * 100.0, axis=1).mean() < 3.0      # left toe on its optimised track
