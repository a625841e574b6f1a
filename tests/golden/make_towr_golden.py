"""Golden vectors for the steps on either side of the phys-optim hot path, produced by the REFERENCE'S OWN code
(`src/utils/towr_utils.py`: prepare_input :451-777, load_results :51-122, apply_results :779-857, and the BVH / Animation
/ Quaternions / InverseKinematics library under `src/skeleton_fitting/ik`) imported from a checkout of the reference ($CHD_REFERENCE_DIR, default ../contact-human-dynamics).

The reference modules do not import on numpy 2 as they are: this script installs shims for `numpy.core.umath_tests`,
`np.float` / `np.int` and the plotting / image modules (none of which the three functions use) and then calls the
unmodified functions.  Run where that checkout exists (the committed outputs are all the tests need):

    python tests/golden/make_towr_golden.py

Writes tests/golden/towr/<case>/{anim.bvh, floor.txt, foot_contacts.npy, phys_in/*.txt, sol_out.txt, results.npz, applied.npz}.
Inputs are synthetic (no motion-capture data ships with the reference): walking-like clips of two skeletons with the
joint numbering of the reference's `combined` (28 joints, own heel joints) and `ybot` (67 joints, heels added) characters.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "towr")
REF = os.path.join(os.environ.get("CHD_REFERENCE_DIR", os.path.join(ROOT, "..", "contact-human-dynamics")), "src")


def import_reference():
    class _Any(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith("__"):
                raise AttributeError(k)
            return _Any(k)

        def __call__(self, *a, **k):
            return _Any("x")

    ut = types.ModuleType("numpy.core.umath_tests")
    ut.inner1d = lambda a, b: np.einsum("...i,...i->...", a, b)
    ut.matrix_multiply = np.matmul
    sys.modules["numpy.core.umath_tests"] = ut
    for m in ["matplotlib", "matplotlib.pyplot", "matplotlib.animation", "matplotlib.patheffects", "matplotlib.colors", "matplotlib.cm",
              "mpl_toolkits", "mpl_toolkits.mplot3d", "skimage", "skimage.io", "skimage.transform", "cv2"]:
        sys.modules[m] = _Any(m)
        sys.modules[m].__path__ = []
    np.float, np.int = float, int
    sys.dont_write_bytecode = True
    sys.path[:0] = [REF + "/skeleton_fitting/ik", REF + "/utils", REF, REF + "/optimize"]
    import towr_utils
    return towr_utils


# ---- synthetic skeletons with the reference characters' joint numbering (offsets in cm, y pointing down) ----
def combined_skeleton():
    names = ["Hips", "LHip", "LKnee", "LAnkle", "LHeel", "LBigToe", "LSmallToe", "RHip", "RKnee", "RAnkle", "RHeel", "RBigToe",
             "RSmallToe", "Spine", "Spine1", "Spine2", "Neck", "Nose", "LEye", "LEar", "REye", "REar", "LShoulder", "LElbow", "LWrist",
             "RShoulder", "RElbow", "RWrist"]
    parents = [-1, 0, 1, 2, 3, 3, 3, 0, 7, 8, 9, 9, 9, 0, 13, 14, 15, 16, 17, 18, 17, 20, 16, 22, 23, 16, 25, 26]
    off = [[0, 0, 0], [9.5, 3, 0.5], [0.4, 41, 0.8], [0.2, 40, -1.2], [0.3, 7.5, -5.5], [1.5, 8, 13.5], [-3.5, 8.2, 11],
           [-9.5, 3, 0.5], [-0.4, 41, 0.8], [-0.2, 40, -1.2], [-0.3, 7.5, -5.5], [-1.5, 8, 13.5], [3.5, 8.2, 11],
           [0, -11, -1], [0, -13, 0.5], [0, -13, 0.5], [0, -15, 1], [0, -12, 9], [3, -3, -2], [5, 1, -8], [-3, -3, -2], [-5, 1, -8],
           [17, 1, -1], [2, 27, 0], [1, 25, 2], [-17, 1, -1], [-2, 27, 0], [-1, 25, 2]]
    return names, parents, off, dict(l_hip=1, l_knee=2, r_hip=7, r_knee=8, spine=13, l_sh=22, r_sh=25)


def ybot_skeleton():
    names = ["Hips", "Spine", "Spine1", "Spine2", "Neck", "Head", "HeadTop_End", "LeftEye", "RightEye"]
    parents = [-1, 0, 1, 2, 3, 4, 5, 5, 5]
    off = [[0, 0, 0], [0, -10, -1], [0, -12, 0], [0, -13.5, 0], [0, -15, 0.5], [0, -10, 3], [0, -18, 0], [3, -8, 9], [-3, -8, 9]]

    def arm(side, sx):
        base = len(names)
        names.extend([side + n for n in ("Shoulder", "Arm", "ForeArm", "Hand")])
        parents.extend([3, base, base + 1, base + 2])
        off.extend([[sx * 6, -12, 0], [sx * 13, 0, 0], [sx * 1, 27, 0], [sx * 0.5, 27, 1]])
        hand = base + 3
        for fi, fn in enumerate(("Thumb", "Index", "Middle", "Ring", "Pinky")):
            for k in range(4):
                names.append("%sHand%s%d" % (side, fn, k + 1))
                parents.append(hand if k == 0 else len(names) - 2)
                off.append([sx * (fi - 2) * 2.0, 3.0 + (4 - k), 0.5] if k == 0 else [0, 3.0, 0])

    arm("Left", 1.0)
    arm("Right", -1.0)

    def leg(side, sx):
        base = len(names)
        names.extend([side + n for n in ("UpLeg", "Leg", "Foot", "ToeBase", "Toe_End")])
        parents.extend([0, base, base + 1, base + 2, base + 3])
        off.extend([[sx * 9.2, 5.5, 0.2], [sx * 0.3, 40.5, 0.4], [sx * 0.1, 42, -0.8], [0, 10.5, 12.5], [0, 0, 7]])

    leg("Right", -1.0)
    leg("Left", 1.0)
    assert len(names) == 67 and names[57] == "RightUpLeg" and names[62] == "LeftUpLeg" and names[10] == "LeftArm" and names[34] == "RightArm"
    return names, parents, off, dict(l_hip=62, l_knee=63, r_hip=57, r_knee=58, spine=1, l_sh=10, r_sh=34)


def make_motion(names, key, n_frames, fps, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n_frames) / fps
    J = len(names)
    rows = np.zeros((n_frames, 3 + 3 * J))
    rows[:, 0] = 3.0 * np.sin(2 * np.pi * 0.9 * t)
    rows[:, 1] = -95.0 - 1.5 * np.sin(2 * np.pi * 1.8 * t)
    rows[:, 2] = 100.0 * t
    col = lambda j: 3 + 3 * j                      # Z X Y rotation columns of joint j
    rows[:, col(0):col(0) + 3] = np.stack([5 * np.sin(2 * np.pi * 0.9 * t), 4 * np.sin(2 * np.pi * 1.8 * t + 0.3), 25 * np.sin(2 * np.pi * 0.3 * t) + 10], axis=1)
    swing = 27 * np.sin(2 * np.pi * 0.9 * t)
    rows[:, col(key["l_hip"]) + 1] = swing
    rows[:, col(key["r_hip"]) + 1] = -swing
    rows[:, col(key["l_knee"]) + 1] = 20 + 17 * np.cos(2 * np.pi * 0.9 * t)
    rows[:, col(key["r_knee"]) + 1] = 20 - 17 * np.cos(2 * np.pi * 0.9 * t)
    rows[:, col(key["spine"])] = 4 * np.sin(2 * np.pi * 0.9 * t + 1.0)
    rows[:, col(key["l_sh"]) + 1] = -20 * np.sin(2 * np.pi * 0.9 * t)
    rows[:, col(key["r_sh"]) + 1] = 20 * np.sin(2 * np.pi * 0.9 * t)
    smooth = np.cumsum(rng.normal(0, 0.25, rows[:, 6:].shape), axis=0)
    rows[:, 6:] += smooth - smooth.mean(axis=0)
    return rows


def gait_contacts(n_frames, fps, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n_frames) / fps
    ph = (t * 0.9 + rng.uniform(0, 1)) % 1.0
    l_toe, r_toe = ph < 0.6, ((ph + 0.5) % 1.0) < 0.6
    l_heel, r_heel = ((ph + 0.08) % 1.0) < 0.55, ((ph + 0.58) % 1.0) < 0.55
    return np.stack([l_heel, l_toe, r_heel, r_toe], axis=1).astype(np.int64)     # foot_contacts.npy column order


def main():
    tu = import_reference()
    import chd
    from chd import io_formats, prepare
    cases = [("combined", combined_skeleton, 44, 30.0, 3, 41, False, 1), ("ybot", ybot_skeleton, 40, 24.0, 2, 38, False, 2),
             ("ybot_noheel", ybot_skeleton, 36, 30.0, 0, 36, True, 3)]
    for case, skel, F, fps, s0, s1, comb, seed in cases:
        character = case.split("_")[0]
        d = os.path.join(OUT, case)
        os.makedirs(os.path.join(d, "phys_in"), exist_ok=True)
        names, parents, off, key = skel()
        rows = make_motion(names, key, F, fps, seed)
        bvh = os.path.join(d, "anim.bvh")
        prepare.write_bvh(bvh, names, parents, off, rows, 1.0 / fps, order="ZXY")
        floor = os.path.join(d, "floor.txt")
        n = np.array([0.02, -1.0, 0.015])
        open(floor, "w").write("%s %s %s\n1.5 1.2 -4.0\n" % tuple(str(float(v)) for v in n / np.linalg.norm(n)))
        fc = os.path.join(d, "foot_contacts.npy")
        np.save(fc, gait_contacts(F, fps, seed))
        # ---- reference prepare_input ----
        tu.prepare_input(bvh, floor, fc, os.path.join(d, "phys_in"), character, start_idx=s0, end_idx=s1, dt=1.0 / fps, combined_contacts=comb)
        # ---- a solution file in the phys_optim layout (synthetic values near the input motion), reference load_results ----
        p = io_formats.read_phys_inputs(os.path.join(d, "phys_in"), s1 - s0)
        rng = np.random.default_rng(100 + seed)
        N = s1 - s0
        n_ee = 2 if comb else 4
        sample = np.concatenate([p.base_lin + rng.normal(0, 0.01, (N, 3)), np.degrees(p.base_ang) + rng.normal(0, 1.0, (N, 3))] +
                                [p.ee_pos[k] + rng.normal(0, 0.01, (N, 3)) for k in range(n_ee)] + [rng.normal(0, 200, (N, 3)) for _ in range(n_ee)] +
                                [rng.integers(0, 2, (N, n_ee)).astype(np.float64)], axis=1)
        solf = os.path.join(d, "sol_out.txt")
        io_formats.write_solution(solf, p.dt, sample, n_ee)
        res = tu.load_results(solf, flip_coords=True)
        np.savez(os.path.join(d, "results.npz"), dt=res.dt, num_feet=res.num_feet, base_pos=res.base_pos, base_rot=res.base_rot, base_R=res.base_R,
                 feet_pos=res.feet_pos, feet_force=res.feet_force, feet_contact=res.feet_contact)
        # ---- reference apply_results (30 iterations of the damped least-squares IK) ----
        anim, _, anim_og, com_og = tu.apply_results(res, bvh, s0, s1, character, run_ik=True)
        anim0, _, _, _ = tu.apply_results(tu.load_results(solf, flip_coords=True), bvh, s0, s1, character, run_ik=False)
        import Animation
        np.savez(os.path.join(d, "applied.npz"), rot_q=anim.rotations.qs, pos=anim.positions, gpos=Animation.positions_global(anim),
                 rot_q_noik=anim0.rotations.qs, pos_noik=anim0.positions, com_og=com_og, parents=anim.parents, offsets=anim.offsets)
        print(case, "done", anim.rotations.qs.shape)


def retarget_golden():
    """combined_to_mixamo.retarget of the reference on the `combined` golden clip, towards the synthetic 67-joint skeleton (the
    reference hard-codes `<its dir>/<character>.bvh`: the loader is pointed at our skeleton file instead; h5py is stubbed)."""
    tu = import_reference()
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    sys.path.insert(0, REF + "/skeleton_fitting")
    from chd import prepare
    import combined_to_mixamo as ctm
    import Animation
    d = os.path.join(OUT, "retarget")
    os.makedirs(d, exist_ok=True)
    names, parents, off, key = ybot_skeleton()
    rest = np.zeros((1, 3 + 3 * len(names)))
    rest[0, 1] = -97.0
    skel = os.path.join(d, "ybot_skel.bvh")
    prepare.write_bvh(skel, names, parents, off, rest, 1.0 / 30.0, order="ZXY")
    orig = ctm.BVH.load
    ctm.BVH.load = lambda path, *a, **k: orig(skel if os.path.basename(path) == "ybot.bvh" else path, *a, **k)
    ctm.args = types.SimpleNamespace(character="ybot", src_bvh=os.path.join(OUT, "combined", "anim.bvh"))
    out = os.path.join(d, "ref_out.bvh")
    ctm.retarget(ctm.args.src_bvh, "ybot", out)
    ctm.BVH.load = orig
    anim, _, _ = orig(out)
    np.savez(os.path.join(d, "retarget.npz"), rot_q=anim.rotations.qs, pos=anim.positions, gpos=Animation.positions_global(anim))
    os.remove(out)
    print("retarget done", anim.rotations.qs.shape)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "retarget":
        retarget_golden()
    else:
        main()
