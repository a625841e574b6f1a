"""Seeded synthetic phys-optim inputs of the shapes BASELINE.json names (SURVEY.md section 8(d)).

The reference ships no pose fixtures, so benchmarks and parity tests are driven by planar-walk
sequences synthesised here: a COM that advances at constant speed with lateral sway, smooth small
root rotations, a gait clock that yields per-foot contact flags, fixed footprints during stance and
lifted cubic swings, plus millimetre jitter so that the physical constraints actually bite.  The
generator emits `PhysProblem`s (solver ee order: L toe, R toe[, L heel, R heel]) which
`io_formats.write_phys_inputs` can push through the reference's real 4-file boundary.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from .io_formats import PhysProblem, find_contact_durations


def _euler_R(e):
    x, y, z = e
    sx, cx, sy, cy, sz, cz = np.sin(x), np.cos(x), np.sin(y), np.cos(y), np.sin(z), np.cos(z)
    return np.array([[cy * cz, cz * sx * sy - cx * sz, sx * sz + cx * cz * sy],
                     [cy * sz, cx * cz + sx * sy * sz, cx * sy * sz - cz * sx],
                     [-sy, cy * sx, cx * cy]])


def _intervals(flags):
    """inclusive [a,b] runs of 1s"""
    out, F, i = [], len(flags), 0
    while i < F:
        if flags[i]:
            a = i
            while i + 1 < F and flags[i + 1]:
                i += 1
            out.append((a, i))
        i += 1
    return out


def _gait_flags(F, dt, rng, dense):
    """Per-foot toe contact flags (2,F)."""
    flags = np.zeros((2, F), dtype=np.int64)
    if not dense:
        T_step = rng.uniform(0.8, 1.2)
        duty = rng.uniform(0.55, 0.65)
        ph = rng.uniform(0.0, 1.0)
        t = np.arange(F) * dt
        for f in range(2):
            frac = np.mod(t / T_step + ph + 0.5 * f, 1.0)
            flags[f] = (frac < duty).astype(np.int64)
    else:
        # dense contact switching: alternating phases of 4..10 frames (SURVEY 8(d) long-horizon config)
        for f in range(2):
            i, state = 0, int(rng.integers(0, 2))
            while i < F:
                L = int(rng.integers(4, 11))
                flags[f, i:i + L] = state
                state = 1 - state
                i += L
    # keep at least two frames in the first and last phase so every duration is >= 1 frame after
    # find_contact_durations drops the final frame
    for f in range(2):
        flags[f, 1] = flags[f, 0]
        flags[f, -2] = flags[f, -1]
        flags[f, -3] = flags[f, -1]
    return flags


def make_problem(seed: int, n_frames: int = 120, n_ee: int = 2, fps: float = 30.0, dense: bool = False,
                 noise: float = 0.005, toe_flags=None) -> PhysProblem:
    """`toe_flags` (2 x F, 0/1; e.g. columns L toe / R toe of a `foot_contacts.npy`) replaces the gait clock: the
    synthetic feet then follow the given contact pattern (every foot needs at least one stance frame)."""
    rng = np.random.default_rng(seed)
    F, dt = n_frames, 1.0 / fps
    t = np.arange(F) * dt
    T = (F - 1) * dt
    # floor
    normal = np.array([rng.normal(0, 0.02), rng.normal(0, 0.02), 1.0])
    normal /= np.linalg.norm(normal)
    point = np.zeros(3)

    def height(x, y):
        return -(normal[0] * (x - point[0]) + normal[1] * (y - point[1])) / normal[2] + point[2]

    # COM: planar walk along +x
    v = rng.uniform(0.8, 1.6) if not dense else rng.uniform(0.3, 0.7)
    T_sway = rng.uniform(0.8, 1.2)
    A_y = rng.uniform(0.02, 0.05)
    z0 = 0.9 + rng.uniform(-0.05, 0.05)
    com = np.stack([v * t, A_y * np.sin(2 * np.pi * t / T_sway), z0 + 0.02 * np.sin(4 * np.pi * t / T_sway)], axis=1)
    com[:, 2] += height(com[:, 0], com[:, 1])
    # root Euler angles: small smooth sines
    amp = np.array([rng.uniform(0.02, 0.1), rng.uniform(0.02, 0.1), rng.uniform(0.05, 0.3)])
    ph = rng.uniform(0, 2 * np.pi, 3)
    per = np.array([T_sway, T_sway / 2, T_sway]) * rng.uniform(0.9, 1.1, 3)
    ang = amp[None, :] * np.sin(2 * np.pi * t[:, None] / per[None, :] + ph[None, :])

    gait = _gait_flags(F, dt, rng, dense)      # always drawn, so that the rest of the stream does not depend on the override
    toe_flags = gait if toe_flags is None else np.asarray(toe_flags, dtype=np.int64).reshape(2, F)
    d_foot = 0.17
    side = [0.09, -0.09]  # left +y, right -y
    dirx = np.array([1.0, 0.0, 0.0])
    up = np.array([0.0, 0.0, 1.0])
    apex = rng.uniform(0.08, 0.15)
    th0, th1 = rng.uniform(0.15, 0.3), rng.uniform(0.3, 0.5)

    toe = np.zeros((2, F, 3))
    heel = np.zeros((2, F, 3))
    heel_flags = np.zeros((2, F), dtype=np.int64)
    for f in range(2):
        runs = _intervals(toe_flags[f])
        # virtual stances before / after the clip so that leading / trailing swings are defined
        swing_len = (runs[1][0] - runs[0][1] - 1) if len(runs) > 1 else 10
        swing_len = max(swing_len, 4)
        allruns = list(runs)
        if runs[0][0] > 0:
            L0 = runs[0][1] - runs[0][0]
            allruns = [(runs[0][0] - swing_len - 1 - L0, runs[0][0] - swing_len - 1)] + allruns
        if runs[-1][1] < F - 1:
            L1 = runs[-1][1] - runs[-1][0]
            allruns = allruns + [(runs[-1][1] + swing_len + 1, runs[-1][1] + swing_len + 1 + L1)]
        G, ds, dl = [], [], []
        for (a, b) in allruns:
            mid = 0.5 * (a + b) * dt
            gx = v * mid
            gy = A_y * np.sin(2 * np.pi * mid / T_sway) + side[f]
            G.append(np.array([gx, gy, height(gx, gy)]))
            L = b - a + 1
            hi = max(1, min(4, (L - 2) // 2))
            lo = min(2, hi)
            ds.append(int(rng.integers(lo, hi + 1)))
            dl.append(int(rng.integers(lo, hi + 1)))
        K = len(allruns)

        def pitch_and_toe(i):
            """returns (toe position, pitch) at (possibly fractional) frame i"""
            for k in range(K):
                a, b = allruns[k]
                H = G[k] - d_foot * dirx
                H[2] = height(H[0], H[1])
                if a - ds[k] <= i < a:      # heel-only: pivot about the heel
                    phi = th0 * (a - i) / ds[k]
                    return H + d_foot * (np.cos(phi) * dirx + np.sin(phi) * up), phi
                if a <= i <= b - dl[k]:      # flat
                    return G[k].copy(), 0.0
                if b - dl[k] < i <= b:       # toe-only: pivot about the toe
                    phi = -th1 * (i - (b - dl[k])) / dl[k]
                    return G[k].copy(), phi
                if k + 1 < K:
                    a2 = allruns[k + 1][0] - ds[k + 1]
                    if b < i < a2:           # swing
                        s = (i - b) / float(a2 - b)
                        hs = 3 * s * s - 2 * s * s * s
                        H2 = G[k + 1] - d_foot * dirx
                        H2[2] = height(H2[0], H2[1])
                        p1 = H2 + d_foot * (np.cos(th0) * dirx + np.sin(th0) * up)
                        p = G[k] + hs * (p1 - G[k]) + apex * np.sin(np.pi * s) ** 2 * up
                        return p, -th1 + hs * (th0 + th1)
            # outside every window (cannot happen with the virtual stances) -> hold the nearest footprint
            return G[0].copy() if i < allruns[0][0] else G[-1].copy(), 0.0

        for i in range(F):
            p, phi = pitch_and_toe(i)
            toe[f, i] = p
            heel[f, i] = p - d_foot * (np.cos(phi) * dirx + np.sin(phi) * up)
            for k in range(K):
                a, b = allruns[k]
                if a - ds[k] <= i <= b - dl[k]:
                    heel_flags[f, i] = 1
        if n_ee == 2:
            # toes-only parameterisation: the toe is the only contact point, keep it on the floor all stance
            for i in range(F):
                if toe_flags[f, i]:
                    k = [kk for kk, (a, b) in enumerate(allruns) if a <= i <= b][0]
                    toe[f, i] = G[k]
        heel_flags[f, 1] = heel_flags[f, 0]
        heel_flags[f, -2] = heel_flags[f, -1]
        heel_flags[f, -3] = heel_flags[f, -1]

    # skeleton
    hip_l = np.array([0.0, 0.09, -0.10])[None, :] + rng.normal(0, 0.005, (F, 3))
    hip_r = np.array([0.0, -0.09, -0.10])[None, :] + rng.normal(0, 0.005, (F, 3))
    mass = 73.0
    scale = rng.uniform(0.8, 1.2)
    slow = np.sin(2 * np.pi * t / T + rng.uniform(0, 2 * np.pi))
    inertia = np.zeros((F, 6))
    inertia[:, 0] = 9.0 * scale * (1 + 0.05 * slow)
    inertia[:, 1] = 8.0 * scale * (1 - 0.05 * slow)
    inertia[:, 2] = 1.5 * scale * (1 + 0.03 * slow)
    inertia[:, 3] = 0.3 * rng.uniform(-1, 1) * slow
    inertia[:, 4] = 0.3 * rng.uniform(-1, 1) * np.cos(2 * np.pi * t / T)
    inertia[:, 5] = 0.3 * rng.uniform(-1, 1) * slow

    # leg length limits from the clean data so that the range-of-motion rows are active but satisfiable
    def max_reach(ee_pos, hip):
        m = 0.0
        for i in range(F):
            R = _euler_R(ang[i])
            m = max(m, np.linalg.norm(ee_pos[i] - (R @ hip[i] + com[i])))
        return m

    reach_toe = max(max_reach(toe[0], hip_l), max_reach(toe[1], hip_r))
    reach_heel = max(max_reach(heel[0], hip_l), max_reach(heel[1], hip_r))
    max_leg = reach_toe * rng.uniform(0.985, 1.03)
    max_heel = reach_heel * rng.uniform(0.985, 1.03)

    # measurement noise
    com_n = com + rng.normal(0, noise, com.shape)
    ang_n = ang + rng.normal(0, noise, ang.shape)
    toe_n = toe + rng.normal(0, noise, toe.shape)
    heel_n = heel + rng.normal(0, noise, heel.shape)

    if n_ee == 2:
        ee = np.stack([toe_n[0], toe_n[1]])
        flags = [toe_flags[0], toe_flags[1]]
    else:
        ee = np.stack([toe_n[0], toe_n[1], heel_n[0], heel_n[1]])
        flags = [toe_flags[0], toe_flags[1], heel_flags[0], heel_flags[1]]
    starts = [int(fl[0]) for fl in flags]
    durs = [np.array(find_contact_durations(list(fl), dt)) for fl in flags]
    return PhysProblem(dt=dt, hip_left=hip_l, hip_right=hip_r, max_leg_length=float(max_leg),
                       max_heel_length=float(max_heel), heel_dist=d_foot, body_mass=mass, inertia=inertia,
                       base_lin=com_n, base_ang=ang_n, ee_pos=ee, floor_normal=normal, floor_point=point,
                       ee_start_contact=starts, ee_durations=durs)


def make_batch(batch: int, n_frames: int = 120, n_ee: int = 2, seed0: int = 0, dense: bool = False,
               fps: float = 30.0) -> List[PhysProblem]:
    """Seeds seed0 .. seed0+batch-1, one per sequence (SURVEY 8(d))."""
    return [make_problem(seed0 + i, n_frames, n_ee, fps, dense) for i in range(batch)]


# ---------------------------------------------------------------------------------------------------------------------
# A synthetic video directory for the pipeline on either side of phys-optim (no capture data ships with the reference):
# OpenPose BODY_25 JSON files, a Monocular-Total-Capture `tracked_results.json`, contact labels, and the skeleton template.
# ---------------------------------------------------------------------------------------------------------------------
def _mocap_walk(n_frames: int, seed: int, fps: float):
    """The walk behind `write_mocap_clip`: (rng after its draws, IK-fitted SkelAnim, global joint positions (F, 28, 3), root
    (F, 3), foot contacts (F, 4) int64 [L heel, L toe, R heel, R toe], floor height) in the MTC camera frame, cm."""
    from . import prepare, results
    rng = np.random.default_rng(seed)
    F, J = n_frames, len(prepare.COMBINED_NAMES)
    t = np.arange(F) / fps
    T_step, speed, floor_y, z0 = rng.uniform(0.9, 1.0), rng.uniform(60.0, 75.0), 92.0, rng.uniform(380.0, 420.0)
    step = speed * T_step
    x0 = -60.0 + rng.uniform(-10, 10)

    def foot(offset, z_lat):
        ph = t / T_step + offset
        k, s = np.floor(ph), ph - np.floor(ph)
        stance = s < 0.6
        u = np.clip((s - 0.6) / 0.4, 0.0, 1.0)
        sm = u * u * (3.0 - 2.0 * u)
        x = x0 + (k + 0.3 + np.where(stance, 0.0, sm)) * step - offset * step      # lands ahead of the hips, leaves behind them
        y = floor_y - np.where(stance, 0.0, 9.0 * np.sin(np.pi * u))
        toe = np.stack([x, y, np.full(F, z0 + z_lat)], axis=1)
        return toe, toe - np.array([17.0, 0.0, 0.0]), stance

    l_toe, l_heel, l_st = foot(0.0, -9.5)
    r_toe, r_heel, r_st = foot(0.5, +9.5)
    root = np.stack([x0 + speed * t - 6.0, floor_y - 82.0 - 1.5 * np.sin(4 * np.pi * t / T_step), np.full(F, z0)], axis=1)
    off = np.asarray(prepare.COMBINED_OFFSETS, dtype=np.float64)
    R0 = np.tile(np.eye(3), (F, J, 1, 1))
    R0[:, 0] = results.rot_zyx(np.array([0.0, np.pi / 2, 0.0]))          # template faces +z, the walk goes along +x
    P0 = np.tile(off[None], (F, 1, 1))
    P0[:, 0] = root
    anim = results.SkelAnim(list(prepare.COMBINED_NAMES), np.array(prepare.COMBINED_PARENTS), off, R0, P0)
    targets = {4: l_heel, 5: l_toe, 10: r_heel, 11: r_toe, 16: root + np.array([4.0, -51.0, 0.0])}
    anim = results.ik_solve(anim, targets, iterations=80, damping=2.0, smoothness=0.0, translate=False)
    gp = anim.global_positions()                                                            # (F, 28, 3) absolute, skeleton order
    fc = np.stack([l_st, l_st, r_st, r_st], axis=1).astype(np.int64)                        # L heel, L toe, R heel, R toe
    return rng, anim, gp, root, fc, floor_y


def _project_keypoints(body, rng, noise_px: float, shift=(0.0, 0.0)):
    """BODY_25 joints (F, 25, 3) in the camera frame -> OpenPose keypoints (F, 25, 3) [x, y, confidence] at focal 2000 px,
    1920 x 1080, principal point moved by `shift` px."""
    F = body.shape[0]
    kp2d = body[:, :25, :2] / body[:, :25, 2:3] * 2000.0 + np.array([960.0 + shift[0], 540.0 + shift[1]]) + rng.normal(0, noise_px, (F, 25, 2))
    conf = rng.uniform(0.4, 1.0, (F, 25))
    return np.concatenate([kp2d, conf[..., None]], axis=2)


def _write_openpose_dir(path: str, name: str, kp):
    import json
    import os
    os.makedirs(path, exist_ok=True)
    for f in range(kp.shape[0]):
        doc = {"version": 1.3, "people": [{"person_id": [-1], "pose_keypoints_2d": [float(v) for v in kp[f].reshape(-1)]}]}
        with open(os.path.join(path, "%s_%012d_keypoints.json" % (name, f)), "w") as fh:
            json.dump(doc, fh)


def write_mocap_clip(video_dir: str, n_frames: int = 48, seed: int = 0, fps: float = 30.0, noise_px: float = 1.0, noise_cm: float = 0.5):
    """Walking clip in the MTC camera frame (x right, y down, z forward, cm; focal 2000 px, 1920 x 1080): feet planted during
    stance, joint angles from an IK fit of the `combined` template.  Writes `<video_dir>/openpose_result/*_keypoints.json`,
    `tracked_results.json`, `foot_contacts.npy`, `skeleton.bvh`; returns the ground truth (dict)."""
    import json
    import os
    from . import kinopt, prepare
    F, J = n_frames, len(prepare.COMBINED_NAMES)
    rng, anim, gp, root, fc, floor_y = _mocap_walk(n_frames, seed, fps)
    body = gp[:, kinopt.BACKWARD]                                                           # body-25 order (+3 spine)
    name = os.path.basename(os.path.normpath(video_dir))
    _write_openpose_dir(os.path.join(video_dir, "openpose_result"), name, _project_keypoints(body, rng, noise_px))
    # MTC results: BODY_25 joints relative to the root translation, 22 SMPL joints (root + spine positions, joint angles)
    Rl = anim.rotations
    ang = np.arccos(np.clip((np.trace(Rl, axis1=-2, axis2=-1) - 1.0) / 2.0, -1.0, 1.0))
    ax = np.stack([Rl[..., 2, 1] - Rl[..., 1, 2], Rl[..., 0, 2] - Rl[..., 2, 0], Rl[..., 1, 0] - Rl[..., 0, 1]], -1)
    aa = -(ax / (np.linalg.norm(ax, axis=-1, keepdims=True) + 1e-12)) * ang[..., None] + rng.normal(0, 0.02, (F, J, 3))
    rel = body[:, :25] - root[:, None] + rng.normal(0, noise_cm, (F, 25, 3))
    rel[:, kinopt.ROOT_IDX] = 0.0
    smpl_pos, smpl_rot = np.zeros((F, 22, 3)), np.zeros((F, 22, 3))
    for j, s in enumerate(kinopt.COMBINED_TO_SMPL):
        if s >= 0:
            smpl_pos[:, s] = gp[:, j] - root + rng.normal(0, noise_cm, (F, 3))
            smpl_rot[:, s] = aa[:, j]
    smpl_pos[:, 0] = 0.0
    xyz = lambda v: {"x": float(v[0]), "y": float(v[1]), "z": float(v[2])}
    frames = [{"trans": xyz(root[f]), "joints": [{"pos": xyz(rel[f, j])} for j in range(25)],
               "SMPLJoints": [{"pos": xyz(smpl_pos[f, s]), "rot": xyz(smpl_rot[f, s])} for s in range(22)], "bodyCoeffs": [], "faceCoeffs": []} for f in range(F)]
    with open(os.path.join(video_dir, "tracked_results.json"), "w") as fh:
        json.dump({"totalcapResults": frames}, fh)
    np.save(os.path.join(video_dir, "foot_contacts.npy"), fc)
    prepare.write_combined_template(os.path.join(video_dir, "skeleton.bvh"))
    return dict(root=root, joints=gp, contacts=fc, floor_y=floor_y, euler=None, fps=fps)


def write_contact_dataset(root: str, characters: int, motions: int, views: int, frames: int, seed: int = 0) -> List[str]:
    """A labelled tree in the layout of the reference's synthetic contact dataset (contact_data_utils.py:8-27), read by
    `chd.contact.read_synthetic_videos`:

        <root>/character<c>/motion<m>/foot_contacts.npy                 (frames, 4) int64, shared by the motion's views
        <root>/character<c>/motion<m>/view<k>/frame_<f>.png             empty placeholders: the reference counts frames here
        <root>/character<c>/motion<m>/keypoints_view<k>/*_keypoints.json

    Every motion is one `write_mocap_clip` walk (its own seed); every view projects it with its own principal point,
    pixel noise, confidences and a few low-confidence frames.  Keypoints are rounded to 1e-3 px (confidences to 1e-4), as
    OpenPose writes a handful of decimals; the files are then the same on any host.  Returns the motion directories."""
    import os
    from . import kinopt
    out = []
    for c in range(characters):
        for m in range(motions):
            mdir = os.path.join(root, "character%02d" % c, "motion%02d" % m)
            wseed = int(np.random.SeedSequence([seed, c, m]).generate_state(1)[0])
            _, _, gp, _, fc, _ = _mocap_walk(frames, wseed, 30.0)
            body = gp[:, kinopt.BACKWARD]
            os.makedirs(mdir, exist_ok=True)
            np.save(os.path.join(mdir, "foot_contacts.npy"), fc)
            for k in range(views):
                rng = np.random.default_rng([seed, c, m, k])
                kp = _project_keypoints(body, rng, 1.0, shift=tuple(rng.uniform(-200.0, 200.0, 2)))
                low = rng.uniform(size=kp.shape[:2]) < 0.03
                kp[:, :, 2] = np.where(low, kp[:, :, 2] * 0.25, kp[:, :, 2])
                kp[:, :, :2] = np.round(kp[:, :, :2], 3)
                kp[:, :, 2] = np.round(kp[:, :, 2], 4)
                vdir = os.path.join(mdir, "view%d" % k)
                os.makedirs(vdir, exist_ok=True)
                for f in range(frames):
                    open(os.path.join(vdir, "frame_%06d.png" % f), "wb").close()
                _write_openpose_dir(os.path.join(mdir, "keypoints_view%d" % k), "view%d" % k, kp)
            out.append(mdir)
    return out
