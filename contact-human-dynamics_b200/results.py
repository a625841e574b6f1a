"""The step behind the phys-optim hot path (SURVEY.md 8(f) rank 1): read a `sol_out_*.txt`, carry it back into the
skeleton's frame and units, and put the optimised root / foot trajectories back onto the original skeleton with a damped
least-squares full-body IK.

Reference: `src/utils/towr_utils.py:51-122` (load_results), `:779-857` (apply_results), the IK it calls
(`src/skeleton_fitting/ik/InverseKinematics.py:326-565`, JacobianInverseKinematicsCK with translate=True, 30 iterations,
damping 7, smoothness 0.001) and `BVH.save` (`src/skeleton_fitting/ik/BVH.py:174-291`).

Own formulation (rotation matrices, no quaternion library).  Every IK goes through `ik_solve_batch` (many clips of one
skeleton; a single clip is a batch of one): on a CUDA device one `chd_ik_solve` call (csrc/chd_ik.cu, one CTA per
frame, the Jacobian never formed), on the host `ik_solve` per clip.  `ik_solve` is the host reference, batched over the
frames with torch on the CPU:
* every IK iteration is one batched pass: forward kinematics, the 3T x 6J Jacobian of the T target joints with respect
  to every joint's Euler angles (R = Rz Ry Rx) and local translation, and the damped step.  The reference factors the
  6J x 6J matrix J^T J + lambda^2 I per frame with a dense LU (414 x 414 for the 69-joint character); because the damping
  is a multiple of the identity the same step is J^T (J J^T + lambda^2 I)^-1 e -- a 3T x 3T Cholesky (60 x 60), batched
  over all frames;
* the smoothing term couples a frame only to the previous iterate of its two neighbours, so the frames stay independent
  inside an iteration.

Pinned to the reference's own functions by tests/golden/make_towr_golden.py (tests/test_results_cpu.py).
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np

from .prepare import C_BVH_TO_TOWR, Bvh, CharacterInfo, euler_zyx_from_matrix, forward_kinematics, load_bvh, local_transforms, segment_centres


@dataclass
class TowrResults:
    """towr_utils.py:29-49.  Everything is in the skeleton's (BVH) frame: y / z swapped back and flipped, metres."""
    num_feet: int
    dt: float
    base_pos: np.ndarray      # (F, 3)
    base_rot: np.ndarray      # (F, 3) Euler angles x, y, z [rad] with R = Rz Ry Rx
    base_R: np.ndarray        # (F, 3, 3)
    feet_pos: np.ndarray      # (F, n_feet, 3)   order L toe, R toe, L heel, R heel
    feet_force: np.ndarray    # (F, n_feet, 3)
    feet_contact: np.ndarray  # (F, n_feet) int


def rot_zyx(e):
    """(..., 3) Euler angles x, y, z -> R = Rz(z) Ry(y) Rx(x)  (`Quaternions.from_euler(order='xyz', world=True)`)."""
    e = np.asarray(e, dtype=np.float64)
    cx, sx, cy, sy, cz, sz = np.cos(e[..., 0]), np.sin(e[..., 0]), np.cos(e[..., 1]), np.sin(e[..., 1]), np.cos(e[..., 2]), np.sin(e[..., 2])
    R = np.empty(e.shape[:-1] + (3, 3))
    R[..., 0, 0], R[..., 0, 1], R[..., 0, 2] = cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx
    R[..., 1, 0], R[..., 1, 1], R[..., 1, 2] = sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx
    R[..., 2, 0], R[..., 2, 1], R[..., 2, 2] = -sy, cy * sx, cy * cx
    return R


def load_towr_results(file_path: str, flip_coords: bool = True) -> Optional[TowrResults]:
    """towr_utils.load_results: label line / value line pairs (phys_optim.cpp:63-143); positions and forces get y / z swapped
    (and all axes flipped with `flip_coords`), the base orientation is conjugated with the same coordinate change."""
    if not os.path.exists(file_path):
        print("Could not find results file " + file_path)
        return None
    lines = [l.rstrip("\n") for l in open(file_path)]
    dt, N, n_feet = float(lines[1]), int(lines[3]), int(lines[5])
    idx = 7
    vec = lambda i: np.array(lines[i].split(" "), dtype=np.float64).reshape(N, 3)
    base_pos, base_ang = vec(idx), vec(idx + 2)
    idx += 4
    feet_pos = np.stack([vec(idx + 2 * k) for k in range(n_feet)], axis=1)
    idx += 2 * n_feet
    feet_force = np.stack([vec(idx + 2 * k) for k in range(n_feet)], axis=1)
    idx += 2 * n_feet
    feet_contact = np.stack([np.array(lines[idx + 2 * k].split(" "), dtype=np.int64) for k in range(n_feet)], axis=1)
    sgn = -1.0 if flip_coords else 1.0
    swap = lambda a: sgn * a[..., [0, 2, 1]]
    # orientation: the rotation axis is swapped / flipped like a vector, i.e. R' = C R C^T with the (proper, symmetric)
    # coordinate change C; without the flip the axis map is the improper y/z swap P: R' = (rotation about P a by the same angle)
    R = rot_zyx(np.radians(base_ang))
    if flip_coords:
        Rn = C_BVH_TO_TOWR @ R @ C_BVH_TO_TOWR.T
    else:
        P = np.array([[1.0, 0, 0], [0, 0, 1.0], [0, 1.0, 0]])
        Rn = np.swapaxes(P @ R @ P.T, -1, -2)      # a reflection conjugate reverses the sense of rotation
    return TowrResults(n_feet, dt, swap(base_pos), euler_zyx_from_matrix(Rn), Rn, swap(feet_pos), swap(feet_force), feet_contact)


@dataclass
class SkelAnim:
    """A skeleton animation in local form (what the reference's `Animation` holds)."""
    names: List[str]
    parents: np.ndarray       # (J,)
    offsets: np.ndarray       # (J, 3)
    rotations: np.ndarray     # (F, J, 3, 3) local rotation matrices
    positions: np.ndarray     # (F, J, 3) local translations

    def global_positions(self, device=None):
        return forward_kinematics(self.parents, self.rotations, self.positions, device)[0]


def anim_from_bvh(b: Bvh, start=None, end=None) -> SkelAnim:
    R, T = local_transforms(b)
    return SkelAnim(list(b.names), b.parents.copy(), b.offsets.copy(), R[start:end].copy(), T[start:end].copy())


def add_heel_to_anim(a: SkelAnim, toe_inds, ankle_inds) -> SkelAnim:
    """towr_utils.py:401-423: two dummy joints (left, right heel) below the ankles at the toes' vertical offset, appended last."""
    off = np.zeros((2, 3))
    off[:, 1] = a.offsets[list(toe_inds), 1]
    F = a.rotations.shape[0]
    return SkelAnim(a.names + ["LeftHeel", "RightHeel"], np.concatenate([a.parents, list(ankle_inds)]), np.concatenate([a.offsets, off]),
                    np.concatenate([a.rotations, np.tile(np.eye(3), (F, 2, 1, 1))], axis=1), np.concatenate([a.positions, np.tile(off[None], (F, 1, 1))], axis=1))


def remove_heel_from_anim(a: SkelAnim) -> SkelAnim:
    """towr_utils.py:425-433."""
    return SkelAnim(a.names[:-2], a.parents[:-2], a.offsets[:-2], a.rotations[:, :-2], a.positions[:, :-2])


def descendants_mask(parents) -> np.ndarray:
    """[k, t] = joint t is a strict descendant of joint k."""
    J = len(parents)
    m = np.zeros((J, J), dtype=bool)
    for t in range(J):
        k = int(parents[t])
        while k >= 0:
            m[k, t] = True
            k = int(parents[k])
    return m


def ik_solve(anim: SkelAnim, targets: Dict[int, np.ndarray], iterations: int = 30, damping: float = 7.0, smoothness: float = 0.001,
             history: Optional[list] = None, translate: bool = True) -> SkelAnim:
    """Damped least-squares full-body IK (JacobianInverseKinematicsCK, unit weights, no references / angle limits), all
    frames at once in torch on the CPU: the host reference `chd_ik_solve` is tested against.  `translate`: the joints'
    local translations are unknowns too.  `targets`: joint index -> (F, 3) world positions.  `history`, if given, gets
    the mean target distance before every iteration and after the last."""
    import torch
    f64 = dict(dtype=torch.float64)
    parents = [int(p) for p in anim.parents]
    J, F = len(parents), anim.rotations.shape[0]
    tj = list(targets.keys())
    T = len(tj)
    goal = torch.as_tensor(np.stack([np.asarray(targets[k], dtype=np.float64) for k in tj], axis=1), **f64)      # (F, T, 3)
    desc = descendants_mask(parents)
    dsc = torch.as_tensor(desc[:, tj].astype(np.float64), **f64)                                                # (J, T) rotation of k moves t
    tdsc = torch.as_tensor((desc | np.eye(J, dtype=bool))[:, tj].astype(np.float64), **f64)                     # translation of k moves t
    Rl = torch.as_tensor(anim.rotations, **f64)
    Pl = torch.as_tensor(anim.positions, **f64).clone()
    lam2 = (damping * (1.0 / (1.0 + 0.001))) ** 2
    eye3 = torch.eye(3, **f64)
    I3T = torch.eye(3 * T, **f64)

    def fk(Rl, Pl):
        gR, gP = [None] * J, [None] * J
        for j in range(J):
            p = parents[j]
            if p < 0:
                gR[j], gP[j] = Rl[:, j], Pl[:, j]
            else:
                gR[j] = gR[p] @ Rl[:, j]
                gP[j] = gP[p] + (gR[p] @ Pl[:, j].unsqueeze(-1)).squeeze(-1)
        return torch.stack(gR, 1), torch.stack(gP, 1)

    def euler_of(R):   # x, y, z with R = Rz Ry Rx
        return torch.stack([torch.atan2(R[..., 2, 1], R[..., 2, 2]), -torch.asin(R[..., 2, 0].clamp(-1.0, 1.0)), torch.atan2(R[..., 1, 0], R[..., 0, 0])], -1)

    def rot_of(e):
        cx, sx, cy, sy, cz, sz = torch.cos(e[..., 0]), torch.sin(e[..., 0]), torch.cos(e[..., 1]), torch.sin(e[..., 1]), torch.cos(e[..., 2]), torch.sin(e[..., 2])
        rows = [torch.stack([cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx], -1),
                torch.stack([sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx], -1), torch.stack([-sy, cy * sx, cy * cx], -1)]
        return torch.stack(rows, -2)

    par_idx = torch.as_tensor([max(p, 0) for p in parents])
    root_mask = torch.as_tensor([p < 0 for p in parents])
    for it in range(iterations):
        gR, gP = fk(Rl, Pl)
        e = euler_of(Rl)                                               # (F, J, 3)
        x = torch.cat([e.reshape(F, -1), Pl.reshape(F, -1)], dim=1) if translate else e.reshape(F, -1)   # (F, 6J) / (F, 3J)
        prs = gR[:, par_idx].clone()                                   # parent's global rotation, identity for the root
        prs[:, root_mask] = eye3
        cz, sz, cy, sy = torch.cos(e[..., 2]), torch.sin(e[..., 2]), torch.cos(e[..., 1]), torch.sin(e[..., 1])
        # rotation axes in the parent frame: x-axis after Rz Ry, y-axis after Rz, z-axis
        ax_x = torch.stack([cz * cy, sz * cy, -sy], -1)
        ax_y = torch.stack([-sz, cz, torch.zeros_like(cz)], -1)
        ax_z = torch.zeros_like(ax_x)
        ax_z[..., 2] = 1.0
        axes = torch.stack([ax_x, ax_y, ax_z], 2)                      # (F, J, 3 axes, 3)
        axes = torch.einsum("fjab,fjkb->fjka", prs, axes)              # world frame
        tp = gP[:, tj]                                                 # (F, T, 3)
        arm = tp[:, None, :, :] - gP[:, :, None, :]                    # (F, J, T, 3) target minus joint position
        jr = torch.cross(axes[:, :, :, None, :].expand(F, J, 3, T, 3), arm[:, :, None, :, :].expand(F, J, 3, T, 3), dim=-1) * dsc[None, :, None, :, None]
        if translate:
            jt = prs.transpose(-1, -2)[:, :, :, None, :].expand(F, J, 3, T, 3) * tdsc[None, :, None, :, None]   # column a of prs = prs e_a
            Jm = torch.cat([jr.reshape(F, 3 * J, 3 * T), jt.reshape(F, 3 * J, 3 * T)], dim=1).transpose(1, 2)     # (F, 3T, 6J)
        else:
            Jm = jr.reshape(F, 3 * J, 3 * T).transpose(1, 2)
        err = (goal - tp).reshape(F, 3 * T)
        if history is not None:
            history.append(float(torch.sqrt(((goal - tp) ** 2).sum(-1)).mean()))
        A = Jm @ Jm.transpose(1, 2) + lam2 * I3T
        y = torch.cholesky_solve(err.unsqueeze(-1), torch.linalg.cholesky(A))
        dx1 = (Jm.transpose(1, 2) @ y).squeeze(-1)
        xp = torch.cat([x[:1], x[:-1]], dim=0)
        xa = torch.cat([x[1:], x[-1:]], dim=0)
        x = x + dx1 + smoothness * (xp + xa - 2.0 * x)
        Rl = rot_of(x[:, :3 * J].reshape(F, J, 3))
        if translate:
            Pl = x[:, 3 * J:].reshape(F, J, 3)
    if history is not None:
        _, gP = fk(Rl, Pl)
        history.append(float(torch.sqrt(((goal - gP[:, tj]) ** 2).sum(-1)).mean()))
    return SkelAnim(anim.names, anim.parents, anim.offsets, Rl.numpy(), Pl.numpy())


IK_MAX_JOINTS = 128     # limits of the chd_ik_solve kernel (include/chd.h)
IK_MAX_TARGETS = 64


def _check_ik_batch(anims: Sequence[SkelAnim], targets: Sequence[Dict[int, np.ndarray]]) -> List[int]:
    """Raises ValueError unless the clips can go through one chd_ik_solve call; returns the target joints in order."""
    if len(anims) != len(targets):
        raise ValueError("ik_solve_batch: %d anims but %d target dicts" % (len(anims), len(targets)))
    parents = np.asarray(anims[0].parents)
    tj = [int(k) for k in targets[0].keys()]
    J, T = len(parents), len(tj)
    for a, tg in zip(anims, targets):
        if not np.array_equal(np.asarray(a.parents), parents):
            raise ValueError("ik_solve_batch: every anim must have the same parents")
        if set(int(k) for k in tg.keys()) != set(tj):
            raise ValueError("ik_solve_batch: every targets dict must have the same keys")
        F = a.rotations.shape[0]
        if a.rotations.shape != (F, J, 3, 3) or a.positions.shape != (F, J, 3) or any(np.shape(v) != (F, 3) for v in tg.values()):
            raise ValueError("ik_solve_batch: rotations (F, J, 3, 3), positions (F, J, 3) and targets (F, 3) must agree")
    if J < 1 or J > IK_MAX_JOINTS:
        raise ValueError("ik_solve_batch: %d joints, the kernel takes 1 .. %d" % (J, IK_MAX_JOINTS))
    if T < 1 or T > IK_MAX_TARGETS:
        raise ValueError("ik_solve_batch: %d targets, the kernel takes 1 .. %d" % (T, IK_MAX_TARGETS))
    if parents[0] != -1 or any(not (-1 <= parents[j] < j) for j in range(1, J)):
        raise ValueError("ik_solve_batch: parents must be ordered (parents[0] = -1, parents[j] < j)")
    if any(not (0 <= t < J) for t in tj):
        raise ValueError("ik_solve_batch: a target joint is out of range")
    return tj


def ik_solve_batch(anims: Sequence[SkelAnim], targets: Sequence[Dict[int, np.ndarray]], iterations: int = 30, damping: float = 7.0,
                   smoothness: float = 0.001, device=None, translate: bool = True) -> List[SkelAnim]:
    """`ik_solve` for many clips of one skeleton (same `parents`, same target joints): on a CUDA device one upload, one
    `chd_ik_solve` call (every frame of every clip, each clip smoothed on its own) and one download; on the host
    `ik_solve` per clip, bitwise.  Raises ValueError for clips that differ in skeleton or target joints and for more
    joints / targets than the kernel takes, before any device work."""
    anims, targets = list(anims), list(targets)
    if not anims and not targets:
        return []
    tj = _check_ik_batch(anims, targets)
    import torch
    dev = torch.device(device) if device is not None else torch.device("cpu")
    if dev.type != "cuda":
        return [ik_solve(a, tg, iterations=iterations, damping=damping, smoothness=smoothness, translate=translate)
                for a, tg in zip(anims, targets)]
    frames = [a.rotations.shape[0] for a in anims]
    J, T, Ft = len(anims[0].parents), len(tj), sum(frames)
    nR, nP = Ft * J * 9, Ft * J * 3
    host = np.concatenate([np.concatenate([a.rotations for a in anims]).reshape(-1), np.concatenate([a.positions for a in anims]).reshape(-1),
                           np.concatenate([np.stack([np.asarray(tg[k], dtype=np.float64) for k in tj], axis=1) for tg in targets]).reshape(-1)])
    buf = torch.as_tensor(host, dtype=torch.float64).to(dev)
    _ik_kernel(anims[0].parents, tj, frames, buf[:nR].view(Ft, J, 3, 3), buf[nR:nR + nP].view(Ft, J, 3), buf[nR + nP:].view(Ft, T, 3),
               iterations, damping, smoothness, translate)
    out = buf[:nR + nP].cpu().numpy()
    cut = np.cumsum(frames)[:-1]
    R, P = np.split(out[:nR].reshape(Ft, J, 3, 3), cut), np.split(out[nR:].reshape(Ft, J, 3), cut)
    return [SkelAnim(a.names, a.parents, a.offsets, r.copy(), p.copy()) for a, r, p in zip(anims, R, P)]


def _ik_kernel(parents, tj, frames, R, P, goal, iterations, damping, smoothness, translate):
    """One `chd_ik_solve` call on clips of `frames` frames stacked on the frame axis of the contiguous fp64 tensors on one
    CUDA device R (Ft, J, 3, 3) and P (Ft, J, 3), which it updates in place, and goal (Ft, T, 3); target joints `tj`.
    Allocates the kernel's work space on that device and runs on its current stream."""
    import torch
    from .phys import _ptr, load_lib
    L = load_lib()
    par, tjn = np.ascontiguousarray(parents, dtype=np.int32), np.ascontiguousarray(tj, dtype=np.int32)
    seg = np.zeros(len(frames) + 1, dtype=np.int32)
    seg[1:] = np.cumsum(frames)
    J, T, Ft = len(par), len(tjn), int(seg[-1])
    dev = R.device
    work = torch.empty(max(L.chd_ik_work_bytes(Ft, J, T) // 8, 1), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = L.chd_ik_solve(J, _ptr(par), T, _ptr(tjn), _ptr(seg), len(frames), Ft, R.data_ptr(), P.data_ptr(), goal.data_ptr(), int(iterations),
                            float(damping), float(smoothness), int(bool(translate)), work.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    if rc != 0:
        raise RuntimeError("chd_ik_solve failed with code %d" % rc)


def _apply_setup(res: TowrResults, anim_bvh: str, start_idx, end_idx, info: CharacterInfo, run_ik: bool, device):
    """apply_results up to the IK: (anim with the optimised root, anim_og, com, IK targets or None)."""
    b = load_bvh(anim_bvh)
    start_idx = 0 if start_idx is None else start_idx
    end_idx = b.n_frames if end_idx is None else end_idx
    anim = anim_from_bvh(b, start_idx, end_idx)
    n_feet = res.feet_pos.shape[1]
    if info.heel_inds is None and n_feet == 4:
        anim = add_heel_to_anim(anim, info.toes, info.ankles)
    init_pos = anim.global_positions(device)
    nj = len(b.names)
    cen, frac = segment_centres(init_pos[:, :max(nj, 1)], info)
    com = np.einsum("s,fsd->fd", frac, cen)
    upper = list(info.upper_body_joints)
    upper_off = init_pos[:, upper, :] - com[:, None, :]
    anim_og = SkelAnim(list(anim.names), anim.parents.copy(), anim.offsets.copy(), anim.rotations.copy(), anim.positions.copy())
    seq_len = end_idx - start_idx
    desired = upper_off + res.base_pos[:seq_len, None, :] * 100.0
    anim.rotations[:, 0] = rot_zyx(res.base_rot)[:seq_len]
    anim.positions[:, 0] = desired[:, 0]
    targets = None
    if run_ik:
        targets = {upper[i]: desired[:, i] for i in range(len(upper))}
        targets[info.toes[0]] = res.feet_pos[:seq_len, 0] * 100.0
        targets[info.toes[1]] = res.feet_pos[:seq_len, 1] * 100.0
        if n_feet == 4:
            lh, rh = info.heel_inds if info.heel_inds is not None else (anim.positions.shape[1] - 2, anim.positions.shape[1] - 1)
            targets[lh] = res.feet_pos[:seq_len, 2] * 100.0
            targets[rh] = res.feet_pos[:seq_len, 3] * 100.0
    return anim, anim_og, com, targets


def apply_results(res: TowrResults, anim_bvh: str, start_idx, end_idx, info: CharacterInfo, run_ik: bool = True, device=None,
                  iterations: int = 30):
    """towr_utils.apply_results: returns (anim, names, anim_og, com_og).  The root follows the optimised COM (keeping every
    upper-body joint's offset from the COM) and base orientation; with `run_ik` the upper-body joints, toes and (4-foot
    results) heels are IK targets.  A batch of one of `apply_results_batch`."""
    return apply_results_batch([(res, anim_bvh, start_idx, end_idx)], info, run_ik, device, iterations)[0]


def apply_results_batch(jobs, info: CharacterInfo, run_ik: bool = True, device=None, iterations: int = 30):
    """apply_results for every job (TowrResults, anim_bvh, start_idx, end_idx); returns one (anim, names, anim_og, com)
    per job.  Jobs with the same skeleton and target joints (e.g. all 2-foot or all 4-foot results of one character)
    share one `ik_solve_batch` call."""
    setups = [_apply_setup(res, anim_bvh, s, e, info, run_ik, device) for res, anim_bvh, s, e in jobs]
    anims = [s[0] for s in setups]
    if run_ik:
        groups: Dict[tuple, List[int]] = {}
        for i, (anim, _, _, targets) in enumerate(setups):
            groups.setdefault((tuple(int(p) for p in anim.parents), tuple(targets)), []).append(i)
        for idx in groups.values():
            solved = ik_solve_batch([anims[i] for i in idx], [setups[i][3] for i in idx], iterations=iterations, smoothness=0.001,
                                    damping=7.0, device=device)
            for i, a in zip(idx, solved):
                anims[i] = a
    return [(a, a.names, s[1], s[2]) for a, s in zip(anims, setups)]


def save_bvh(path: str, anim: SkelAnim, names: Optional[Sequence[str]] = None, frametime: float = 1.0 / 24.0):
    """BVH.save with its defaults (order 'zyx', root-only positions): channels Zrotation Yrotation Xrotation carrying the
    Euler angles of R = Rz Ry Rx in degrees, six decimals."""
    from .prepare import write_bvh
    names = list(names) if names is not None else ["joint_%d" % i for i in range(len(anim.parents))]
    e = np.degrees(euler_zyx_from_matrix(anim.rotations))             # (F, J, 3) = x, y, z
    F, J = e.shape[:2]
    rows = np.concatenate([anim.positions[:, 0], e[:, :, [2, 1, 0]].reshape(F, 3 * J)], axis=1)
    write_bvh(path, names, anim.parents, anim.offsets, rows, frametime, order="ZYX")


# ---------------------------------------------------------------------------------------------------------------------
# Re-targeting of the kinematic result (28-joint `combined` skeleton) to a character skeleton
# (src/skeleton_fitting/combined_to_mixamo.py:38-134), between kinematic_optimizer.py and towr_utils.py in the pipeline.
# ---------------------------------------------------------------------------------------------------------------------
COMBINED_FOOT_INDS = [4, 5, 6, 10, 11, 12]      # character_info_utils.py:196-199
COMBINED_ANKLE_INDS = [3, 9]


def _softmin(x, softness=0.5):
    """combined_to_mixamo.py:30-36 over axis 0: -(max(-x) + log(softness + exp(min(-x) - max(-x))))."""
    nx = -np.asarray(x, dtype=np.float64)
    return -(nx.max() + np.log(softness + np.exp(nx.min() - nx.max())))


def retarget(src_bvh: str, skel_bvh: str, info: CharacterInfo, out_bvh: Optional[str] = None, device=None, iterations: int = 200):
    """combined_to_mixamo.retarget: scales the source joint positions by the ratio of the hip heights (floor at 0 through a
    soft minimum of the foot heights), initialises the character's angles from the mapped source Euler angles, runs the
    damped least-squares IK (translating joints, 200 iterations, damping 7) towards the mapped joints, restores the bone
    offsets and corrects the root height by the median ankle difference.  Returns the SkelAnim (and saves it if asked).
    A batch of one of `retarget_batch`."""
    return retarget_batch([src_bvh], skel_bvh, info, [out_bvh], device, iterations)[0]


def retarget_batch(src_bvhs: Sequence[str], skel_bvh: str, info: CharacterInfo, out_bvhs: Optional[Sequence[Optional[str]]] = None,
                   device=None, iterations: int = 200) -> List[SkelAnim]:
    """retarget for every source clip onto one character skeleton, the IK of all clips in one `ik_solve_batch` call."""
    if out_bvhs is not None and len(out_bvhs) != len(src_bvhs):
        raise ValueError("retarget_batch: %d sources but %d outputs" % (len(src_bvhs), len(out_bvhs)))
    sk, skel_height = _retarget_skeleton(skel_bvh, info)
    setups = [_retarget_setup(s, sk, skel_height, info) for s in src_bvhs]
    anims = ik_solve_batch([s[0] for s in setups], [s[1] for s in setups], iterations=iterations, smoothness=0.0, damping=7.0,
                           translate=True, device=device)
    return [_retarget_finish(a, sk, s[2], s[3], info, out_bvhs[i] if out_bvhs is not None else None)
            for i, (a, s) in enumerate(zip(anims, setups))]


def _retarget_skeleton(skel_bvh: str, info: CharacterInfo):
    """The character skeleton and its height from the hips to the lowest foot joint, rotations zeroed."""
    sk = load_bvh(skel_bvh)
    J = len(sk.names)
    Rk, Tk = local_transforms(sk)
    skel_targets = forward_kinematics(sk.parents, np.tile(np.eye(3), (Tk.shape[0], J, 1, 1)), Tk)[0]      # rotations zeroed
    foot = [info.ankles[0], info.toes[0], info.ankles[1], info.toes[1]]
    fh = np.minimum(skel_targets[:, foot[:2], 1], skel_targets[:, foot[2:], 1]).min(axis=1)
    skel_targets[:, :, 1] -= _softmin(fh)
    skel_height = np.abs(np.amax(skel_targets[:, 0, 1]) - np.amin(skel_targets[:, foot, 1], axis=1)).max()
    return sk, skel_height


def _retarget_setup(src_bvh: str, sk: Bvh, skel_height, info: CharacterInfo):
    """retarget up to the IK: (initial anim, IK targets, scaled source joint positions, source floor height)."""
    J = len(sk.names)
    src = load_bvh(src_bvh)
    Rs, Ts = local_transforms(src)
    at = forward_kinematics(src.parents, Rs, Ts)[0]
    F = at.shape[0]
    at[:, :, 1] = -at[:, :, 1]                                                   # y points down in the source: flip to measure heights
    fl, fr = COMBINED_FOOT_INDS[:3], COMBINED_FOOT_INDS[3:]
    src_floor = _softmin(np.minimum(at[:, fl, 1], at[:, fr, 1]).min(axis=1))
    at[:, :, 1] -= src_floor
    anim_height = np.abs(np.amax(at[:, 0, 1]) - np.amin(at[:, COMBINED_FOOT_INDS, 1], axis=1)).max()
    at[:, :, 1] = -at[:, :, 1]
    ratio = skel_height / anim_height
    targets = at * ratio
    targets[:, :, [0, 2]] -= (targets[:, 0, [0, 2]] - at[:, 0, [0, 2]])[:, None, :]      # hip translation in x / z is not scaled
    mp = info.to_combined
    tm = {i: targets[:, mp[i]] for i in range(J) if mp[i] > -1 and i not in info.ik_blacklist}
    es = euler_zyx_from_matrix(Rs)
    ref = np.zeros((F, J, 3))
    for i in range(J):
        if mp[i] > -1:
            ref[:, i] = np.fmod(es[:, mp[i]] * 180 / 3.1415, 180) * 3.1415 / 180     # the reference's constants
    P0 = np.tile(sk.offsets[None], (F, 1, 1))
    P0[:, 0] = targets[:, 0]
    anim = SkelAnim(list(sk.names), sk.parents.copy(), sk.offsets.copy(), rot_zyx(ref), P0)
    return anim, tm, targets, src_floor


def _retarget_finish(anim: SkelAnim, sk: Bvh, targets, src_floor, info: CharacterInfo, out_bvh: Optional[str]) -> SkelAnim:
    """retarget after the IK: bone offsets restored, root height corrected, saved if asked."""
    anim.positions[:, 1:] = sk.offsets[None, 1:]
    ank = targets[:, COMBINED_ANKLE_INDS, 1] - anim.global_positions()[:, info.ankles, 1]
    anim.positions[:, 0, 1] += np.median(ank)
    anim.positions[:, 0, 1] -= src_floor
    if out_bvh:
        d = os.path.dirname(out_bvh)
        if d:
            os.makedirs(d, exist_ok=True)
        save_bvh(out_bvh, anim, anim.names)
    return anim
