"""File formats on either side of the phys-optim hot path (the reference's process/file boundary).

Inputs  (writer: reference src/utils/towr_utils.py:585-777, reader: towr_phys_optim/phys_optim.cpp:155-267):
    skel_info.txt, motion_info.txt, terrain_info.txt, contact_info.txt
Outputs (writer: phys_optim.cpp:63-153, readers: towr_utils.py:51-122 and src/viz/viz_blender.py:91-162):
    sol_out_no_dynamics.txt, sol_out_dynamics.txt, sol_out_durations.txt, success_log.txt

End-effector orders (SURVEY Appendix C.2):
    files   : L toe, L heel, R toe, R heel
    solver  : L toe, R toe, L heel, R heel          <- PhysProblem.ee_* arrays use this order
    foot_contacts.npy columns: L heel, L toe, R heel, R toe
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

FILE_TO_SOLVER_EE = [0, 2, 1, 3]  # solver ee i lives at file slot FILE_TO_SOLVER_EE[i]... (Ltoe,Rtoe,Lheel,Rheel) <- (0,2,1,3)


@dataclass
class PhysProblem:
    """Everything `phys_optim` reads for one sequence (phys_optim.cpp:380-417), solver ee order."""
    dt: float
    hip_left: np.ndarray          # (F,3) left-hip offset from COM, root frame
    hip_right: np.ndarray         # (F,3)
    max_leg_length: float
    max_heel_length: float
    heel_dist: float
    body_mass: float
    inertia: np.ndarray           # (F,6) Ixx Iyy Izz Ixy Ixz Iyz
    base_lin: np.ndarray          # (F,3) COM position targets
    base_ang: np.ndarray          # (F,3) root Euler xyz targets (rad)
    ee_pos: np.ndarray            # (n_ee,F,3) targets, solver order
    floor_normal: np.ndarray      # (3,)
    floor_point: np.ndarray       # (3,)
    ee_start_contact: List[int] = field(default_factory=list)      # per ee, solver order
    ee_durations: List[np.ndarray] = field(default_factory=list)   # per ee, solver order

    @property
    def n_frames(self) -> int:
        return int(self.base_lin.shape[0])

    @property
    def n_ee(self) -> int:
        return int(self.ee_pos.shape[0])

    @property
    def total_time(self) -> float:
        # phys_optim.cpp:420-423: taken from the left-toe durations only
        t = 0.0
        for d in self.ee_durations[0]:
            t += float(d)
        return t


def find_contact_durations(contacts: Sequence[int], dt: float) -> List[float]:
    """Restates towr_utils.py:435-449 (the last frame is ignored, so the sum is (F-1)*dt)."""
    prev_state = contacts[0]
    cur = 0.0
    out: List[float] = []
    for i in range(0, len(contacts) - 1):
        s = contacts[i]
        if s != prev_state:
            out.append(cur)
            cur = dt
        else:
            cur += dt
        prev_state = s
    out.append(cur)
    return out


def _fmt(v: float) -> str:
    return repr(float(v))  # Python str(float), as towr_utils.py writes it


def write_phys_inputs(p: PhysProblem, out_dir: str) -> None:
    """Writes the four input files exactly as towr_utils.prepare_input lays them out.  A 2-ee problem
    (toes only) writes its toe data into the heel slots as well so that the file stays readable by the
    reference's fixed 4-ee reader."""
    os.makedirs(out_dir, exist_ok=True)
    F = p.n_frames
    with open(os.path.join(out_dir, "skel_info.txt"), "w") as f:
        for arr in (p.hip_left, p.hip_right):
            for i in range(F):
                f.write(" ".join(_fmt(x) for x in arr[i]) + "\n")
        for v in (p.max_leg_length, p.max_heel_length, p.heel_dist, p.body_mass):
            f.write(_fmt(v) + "\n")
        for i in range(F):
            f.write(" ".join(_fmt(x) for x in p.inertia[i]) + "\n")
    slots = _file_slots(p)
    with open(os.path.join(out_dir, "motion_info.txt"), "w") as f:
        f.write(_fmt(p.dt) + "\n")
        for arr in (p.base_lin, p.base_ang, *[p.ee_pos[s] for s in slots]):
            f.write(" ".join(_fmt(x) for x in np.asarray(arr).reshape(-1)) + "\n")
    with open(os.path.join(out_dir, "terrain_info.txt"), "w") as f:
        f.write(" ".join(_fmt(x) for x in p.floor_normal) + "\n")
        f.write(" ".join(_fmt(x) for x in p.floor_point))
    with open(os.path.join(out_dir, "contact_info.txt"), "w") as f:
        for s in slots:
            f.write(str(int(p.ee_start_contact[s])) + "\n")
            f.write(str(len(p.ee_durations[s])) + "\n")
            f.write(" ".join(_fmt(x) for x in p.ee_durations[s]) + "\n")


def _file_slots(p: PhysProblem) -> List[int]:
    # file order L toe, L heel, R toe, R heel expressed as solver indices
    if p.n_ee == 4:
        return [0, 2, 1, 3]
    return [0, 0, 1, 1]


def read_phys_inputs(in_dir: str, nframes: int, n_ee: int = 4) -> PhysProblem:
    """Restates ReadSkeletonInfo / ReadMotionInfo / ReadTerrainInfo / ReadContactInfo
    (phys_optim.cpp:155-267): whitespace-separated `>>` parsing, exactly `nframes` rows."""
    F = nframes

    def toks(name):
        with open(os.path.join(in_dir, name)) as f:
            return f.read().split()

    t = toks("skel_info.txt")
    k = 0
    hip_left = np.array(t[k:k + 3 * F], dtype=np.float64).reshape(F, 3); k += 3 * F
    hip_right = np.array(t[k:k + 3 * F], dtype=np.float64).reshape(F, 3); k += 3 * F
    max_leg, max_heel, heel_dist, mass = (float(x) for x in t[k:k + 4]); k += 4
    inertia = np.array(t[k:k + 6 * F], dtype=np.float64).reshape(F, 6)

    t = toks("motion_info.txt")
    dt = float(t[0]); k = 1
    blocks = []
    for _ in range(6):
        blocks.append(np.array(t[k:k + 3 * F], dtype=np.float64).reshape(F, 3)); k += 3 * F
    base_lin, base_ang, ltoe, lheel, rtoe, rheel = blocks

    t = toks("terrain_info.txt")
    normal = np.array(t[0:3], dtype=np.float64)
    point = np.array(t[3:6], dtype=np.float64)

    t = toks("contact_info.txt")
    k = 0
    starts, durs = [], []
    for _ in range(4):
        # `f >> bool` accepts 0/1; towr_utils writes numpy ints
        starts.append(int(float(t[k]))); k += 1
        P = int(t[k]); k += 1
        durs.append(np.array(t[k:k + P], dtype=np.float64)); k += P
    # file order Ltoe, Lheel, Rtoe, Rheel -> solver order Ltoe, Rtoe, Lheel, Rheel (phys_optim.cpp:491-513)
    order = [0, 2, 1, 3]
    ee_pos = np.stack([ltoe, rtoe, lheel, rheel])[:n_ee]
    return PhysProblem(dt=dt, hip_left=hip_left, hip_right=hip_right, max_leg_length=max_leg,
                       max_heel_length=max_heel, heel_dist=heel_dist, body_mass=mass, inertia=inertia,
                       base_lin=base_lin, base_ang=base_ang, ee_pos=ee_pos, floor_normal=normal,
                       floor_point=point,
                       ee_start_contact=[starts[i] for i in order][:n_ee],
                       ee_durations=[durs[i] for i in order][:n_ee])


# ------------------------------------------------------------------ outputs -------------------------
def _g10(v: float) -> str:
    return "%.10g" % float(v)  # std::ofstream with precision(10), default floatfield (phys_optim.cpp:68)


def write_solution(path: str, dt: float, sample: np.ndarray, n_ee: int) -> None:
    """`sample` is (N, 6+7*n_ee): base_lin(3) base_ang_deg(3) ee_pos(3*n_ee) ee_force(3*n_ee)
    contact(n_ee) -- the layout SaveSolution walks (phys_optim.cpp:63-143).  Label line / value line
    pairs; values separated by single spaces, no trailing space."""
    from .phys import sample_columns        # here, not at the top: phys imports this module
    base, pos, frc, flag = sample_columns(n_ee, n_ee)
    N = sample.shape[0]
    with open(path, "w") as f:
        f.write("dt\n%s\n" % _g10(dt))
        f.write("num_frames\n%d\n" % N)
        f.write("num_feet\n%d\n" % n_ee)
        f.write("base_lin\n" + " ".join(_g10(x) for x in sample[:, base[:3]].reshape(-1)) + "\n")
        f.write("base_ang\n" + " ".join(_g10(x) for x in sample[:, base[3:]].reshape(-1)) + "\n")
        for i in range(n_ee):
            f.write("foot%d_pos\n" % i + " ".join(_g10(x) for x in sample[:, pos[3 * i:3 * i + 3]].reshape(-1)) + "\n")
        for i in range(n_ee):
            f.write("foot%d_force\n" % i + " ".join(_g10(x) for x in sample[:, frc[3 * i:3 * i + 3]].reshape(-1)) + "\n")
        for i in range(n_ee):
            f.write("foot%d_contact\n" % i + " ".join("%d" % int(round(x)) for x in sample[:, flag[i]]) + "\n")


def write_success_log(path: str, dynamics_succeed: bool, durations_succeed: bool) -> None:
    """phys_optim.cpp:145-153."""
    with open(path, "w") as f:
        f.write("dynamics %d\n" % int(bool(dynamics_succeed)))
        f.write("durations %d\n" % int(bool(durations_succeed)))


def read_solution(path: str) -> dict:
    """Line-index parser with the same arithmetic as towr_utils.load_results (towr_utils.py:51-99):
    value lines sit at odd indices; feet at 11+2i, forces at 11+2*nfeet+2i, contacts after that."""
    with open(path) as f:
        lines = f.read().split("\n")
    dt = float(lines[1])
    n = int(lines[3])
    nfeet = int(lines[5])
    out = {"dt": dt, "num_frames": n, "num_feet": nfeet}
    out["base_lin"] = np.array(lines[7].split(), dtype=np.float64).reshape(n, 3)
    out["base_ang_deg"] = np.array(lines[9].split(), dtype=np.float64).reshape(n, 3)
    out["foot_pos"] = np.stack([np.array(lines[11 + 2 * i].split(), dtype=np.float64).reshape(n, 3) for i in range(nfeet)])
    o = 11 + 2 * nfeet
    out["foot_force"] = np.stack([np.array(lines[o + 2 * i].split(), dtype=np.float64).reshape(n, 3) for i in range(nfeet)])
    o += 2 * nfeet
    out["foot_contact"] = np.stack([np.array(lines[o + 2 * i].split(), dtype=np.int64) for i in range(nfeet)])
    return out
