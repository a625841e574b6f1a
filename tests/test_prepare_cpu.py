"""CPU tests of the step before the hot path (SURVEY 8(f) rank 1): BVH -> forward kinematics -> COM / hip offsets /
inertia / root Euler angles / contact schedule -> the four phys_optim input files (towr_utils.py:451-777), and the
result parser (towr_utils.py:51-122).  The reference's own BVH / Animation library is not vendored and no motion data
ships with it, so the checks are independent recomputations on a generated biped clip."""
import os

import numpy as np
import pytest


@pytest.fixture(scope="module")
def clip(chd, tmp_path_factory):
    d = tmp_path_factory.mktemp("clip")
    F = 48
    bvh = str(d / "walk.bvh")
    chd.prepare.write_test_bvh(bvh, F, seed=3)
    with open(d / "floor_out.txt", "w") as f:
        f.write("0.01 -1.0 -0.02\n0.0 -1.5 10.0\n")             # normal / point in the BVH frame [cm], y down
    t = np.arange(F)
    fc = np.zeros((F, 4), np.int64)                              # L heel, L toe, R heel, R toe
    fc[:, 0] = (t % 32) < 18
    fc[:, 1] = ((t + 2) % 32) < 18
    fc[:, 2] = ((t + 16) % 32) < 18
    fc[:, 3] = ((t + 18) % 32) < 18
    np.save(d / "foot_contacts.npy", fc)
    return dict(dir=d, bvh=bvh, F=F, fc=fc)


def _fk_reference(b, f):
    """independent FK of one frame with scipy rotations (intrinsic rotations in channel order)"""
    from scipy.spatial.transform import Rotation as Rot
    J = len(b.names)
    gR, gP = [None] * J, [None] * J
    for j in range(J):
        o = b.chan_off[j]
        ch = b.channels[j]
        vals = b.motion[f, o:o + len(ch)]
        rot_ch = [c for c in ch if c.endswith("rotation")]
        ang = [v for c, v in zip(ch, vals) if c.endswith("rotation")]
        R = Rot.from_euler("".join(c[0] for c in rot_ch), ang, degrees=True).as_matrix() if rot_ch else np.eye(3)   # upper case = intrinsic
        T = b.offsets[j].copy()
        for c, v in zip(ch, vals):
            if c.endswith("position"):
                T["XYZ".index(c[0])] = v
        pj = b.parents[j]
        if pj < 0:
            gR[j], gP[j] = R, T
        else:
            gR[j], gP[j] = gR[pj] @ R, gP[pj] + gR[pj] @ T
    return np.array(gP), np.array(gR)


def test_bvh_reader_and_forward_kinematics(chd, clip):
    b = chd.prepare.load_bvh(clip["bvh"])
    assert b.n_frames == clip["F"] and len(b.names) == 16 and b.names[0] == "Hips" and abs(b.frame_time - 1 / 30) < 1e-6
    assert list(b.parents) == chd.prepare.SIMPLE_PARENTS
    np.testing.assert_allclose(b.offsets, chd.prepare.SIMPLE_OFFSETS)
    R, T = chd.prepare.local_transforms(b)
    pos, gR = chd.prepare.forward_kinematics(b.parents, R, T)
    for f in (0, 17, clip["F"] - 1):
        p_ref, r_ref = _fk_reference(b, f)
        np.testing.assert_allclose(pos[f], p_ref, atol=1e-9)
        np.testing.assert_allclose(gR[f], r_ref, atol=1e-12)
    import torch
    pos_t, _ = chd.prepare.forward_kinematics(b.parents, R, T, device=torch.device("cpu"))     # batched torch path
    np.testing.assert_allclose(pos_t, pos, atol=1e-10)


def test_prepare_input_quantities(chd, clip):
    P = chd.prepare
    info = P.simple_biped_info()
    b = P.load_bvh(clip["bvh"])
    p = P.build_problem(b, [0.01, -1.0, -0.02], [0.0, -1.5, 10.0], clip["fc"], info)
    F = clip["F"]
    assert p.n_frames == F and p.n_ee == 4 and p.body_mass == 73.0
    # COM: independent mass-weighted mean of segment centres, converted (x, y, z) -> (-x, -z, -y) cm -> m
    R, T = P.local_transforms(b)
    pos, gR = P.forward_kinematics(b.parents, R, T)
    com = np.zeros((F, 3))
    for k, joints in info.segment_to_joints.items():
        com += info.segment_mass_percent[k] * 0.01 * pos[:, joints].mean(axis=1)
    com_t = np.stack([-com[:, 0], -com[:, 2], -com[:, 1]], axis=1) * 0.01
    np.testing.assert_allclose(p.base_lin, com_t, atol=1e-12)
    assert 0.7 < p.base_lin[:, 2].mean() < 1.2                                  # z is up, metres
    # feet: toes from the FK, heels below the ankles at the toes' height
    toe_l = pos[:, 11]
    np.testing.assert_allclose(p.ee_pos[0], np.stack([-toe_l[:, 0], -toe_l[:, 2], -toe_l[:, 1]], axis=1) * 0.01, atol=1e-12)
    assert abs(p.heel_dist - np.mean(np.linalg.norm(p.ee_pos[0] - p.ee_pos[2], axis=1))) < 1e-12
    assert abs(p.max_leg_length - (42 + 42 + np.hypot(8, 14)) * 0.01) < 1e-12
    assert abs(p.max_heel_length - (42 + 42 + 8) * 0.01) < 1e-12
    # hip offsets: root rotation / translation zeroed, relative to the COM: left hip on +x of the BVH skeleton -> -x in towr
    assert (p.hip_left[:, 0] < 0).all() and (p.hip_right[:, 0] > 0).all()
    np.testing.assert_allclose(p.hip_left[:, 0] - p.hip_right[:, 0], -0.18, atol=1e-12)
    # inertia about the COM: symmetric positive definite, equal to the point-mass formula evaluated per frame
    for f in (0, F // 2):
        Ixx, Iyy, Izz, Ixy, Ixz, Iyz = p.inertia[f]
        I = np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]])
        assert (np.linalg.eigvalsh(I) > 0).all()
        R0, T0 = P.local_transforms(b, zero_root=True)
        pos0, _ = P.forward_kinematics(b.parents, R0, T0)
        cen = {k: pos0[f, j].mean(axis=0) for k, j in info.segment_to_joints.items()}
        c0 = sum(info.segment_mass_percent[k] * 0.01 * cen[k] for k in cen)
        I_ref = np.zeros((3, 3))
        for k in cen:
            r = P.to_towr(cen[k] - c0)
            I_ref += info.segment_mass_percent[k] * 0.01 * 73.0 * (np.eye(3) * (r @ r) - np.outer(r, r))
        np.testing.assert_allclose(I, I_ref, atol=1e-10)
    # root orientation: Rz Ry Rx of the written Euler angles reproduces C R C^T
    from scipy.spatial.transform import Rotation as Rot
    C = P.C_BVH_TO_TOWR
    assert abs(np.linalg.det(C) - 1.0) < 1e-15
    for f in (0, 11, F - 1):
        x, y, z = p.base_ang[f]
        Rz = Rot.from_euler("z", z).as_matrix() @ Rot.from_euler("y", y).as_matrix() @ Rot.from_euler("x", x).as_matrix()
        np.testing.assert_allclose(Rz, C @ gR[f, 0] @ C.T, atol=1e-12)
    assert np.abs(np.diff(p.base_ang, axis=0)).max() < np.pi                     # unwrapped
    # floor and contact schedule conventions
    np.testing.assert_allclose(p.floor_normal, [-0.01, 0.02, 1.0])               # z up after the coordinate change
    np.testing.assert_allclose(p.floor_point, [-0.0, -0.10, 0.015])
    fc = clip["fc"]
    assert p.ee_start_contact == [int(max(fc[0, 0], fc[0, 1])), int(max(fc[0, 2], fc[0, 3])), int(fc[0, 0]), int(fc[0, 2])]
    for e, col in zip(range(4), (1, 3, 0, 2)):                                   # toe durations from the toe column only (:719-737)
        np.testing.assert_allclose(p.ee_durations[e], chd.io_formats.find_contact_durations(list(fc[:, col]), 1 / 30.0))
        assert abs(sum(p.ee_durations[e]) - (F - 1) / 30.0) < 1e-9


def test_prepare_input_files_round_trip(chd, clip, tmp_path):
    P = chd.prepare
    out = str(tmp_path / "phys_optim_in_biped")
    p = P.prepare_input(clip["bvh"], str(clip["dir"] / "floor_out.txt"), str(clip["dir"] / "foot_contacts.npy"), out,
                        P.simple_biped_info(), start_idx=4, end_idx=44)
    assert p.n_frames == 40
    for name in ("skel_info.txt", "motion_info.txt", "terrain_info.txt", "contact_info.txt"):
        assert os.path.exists(os.path.join(out, name))
    q = chd.io_formats.read_phys_inputs(out, 40, n_ee=4)
    for k in ("hip_left", "hip_right", "inertia", "base_lin", "base_ang", "ee_pos", "floor_normal", "floor_point"):
        np.testing.assert_array_equal(getattr(q, k), getattr(p, k))            # str(float) round trips exactly
    assert q.ee_start_contact == p.ee_start_contact and q.max_leg_length == p.max_leg_length
    for a, b_ in zip(q.ee_durations, p.ee_durations):
        np.testing.assert_array_equal(a, b_)
    assert P.prepare_input("missing.bvh", "x", "y", out, P.simple_biped_info()) is None


def test_load_results_parses_solution_files(chd, tmp_path):
    rng = np.random.default_rng(0)
    N, n_ee = 12, 4
    s = rng.normal(size=(N, chd.phys.sample_stride(n_ee)))
    s[:, chd.phys.sample_columns(n_ee, n_ee)[3]] = rng.integers(0, 2, (N, n_ee))
    for name in ("sol_out_no_dynamics.txt", "sol_out_dynamics.txt", "sol_out_durations.txt"):
        chd.io_formats.write_solution(str(tmp_path / name), 1 / 30.0, s, n_ee)
    chd.io_formats.write_success_log(str(tmp_path / "success_log.txt"), True, False)
    r = chd.prepare.load_results(str(tmp_path))
    assert set(r) == {"no_dynamics", "dynamics", "durations", "success"} and r["success"] == {"dynamics": 1, "durations": 0}
    assert r["durations"]["num_frames"] == N and r["durations"]["num_feet"] == n_ee
