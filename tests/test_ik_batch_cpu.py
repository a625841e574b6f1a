"""The batched IK entry points on the host: `ik_solve_batch`, `apply_results_batch` and `retarget_batch` give bitwise
what `ik_solve` per clip gives (and the single-clip functions, a batch of one each, what the batch gives), and refuse
batches the `chd_ik_solve` kernel cannot take."""
import os

import numpy as np
import pytest

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "towr")
CASES = {"combined": (3, 41), "ybot": (2, 38), "ybot_noheel": (0, 36)}


def make_clip(chd, F, seed, targets=None):
    """F frames of the golden 28-joint clip (repeated when longer), the angles and translations disturbed, and targets at
    the undisturbed joint positions plus noise (cm)."""
    rs = chd.results
    a = rs.anim_from_bvh(chd.prepare.load_bvh(os.path.join(G, "combined", "anim.bvh")))
    idx = np.arange(F) % a.rotations.shape[0]
    rng = np.random.default_rng(seed)
    gp = rs.SkelAnim(a.names, a.parents, a.offsets, a.rotations[idx], a.positions[idx]).global_positions()
    e = chd.prepare.euler_zyx_from_matrix(a.rotations[idx]) + rng.normal(0, 0.1, (F, len(a.parents), 3))
    start = rs.SkelAnim(a.names, a.parents, a.offsets, rs.rot_zyx(e), a.positions[idx] + rng.normal(0, 0.5, (F, len(a.parents), 3)))
    tj = targets if targets is not None else list(range(0, len(a.parents), 2))
    return start, {j: gp[:, j] + rng.normal(0, 0.2, (F, 3)) for j in tj}


def assert_same(a, b):
    np.testing.assert_array_equal(a.rotations, b.rotations)
    np.testing.assert_array_equal(a.positions, b.positions)
    assert list(a.parents) == list(b.parents) and a.names == b.names


@pytest.mark.parametrize("smoothness", [0.0, 0.001])
@pytest.mark.parametrize("translate", [True, False])
def test_ik_solve_batch_host_is_ik_solve(chd, smoothness, translate):
    rs = chd.results
    clips = [make_clip(chd, F, seed) for seed, F in enumerate((1, 2, 3, 14))]
    got = rs.ik_solve_batch([c[0] for c in clips], [c[1] for c in clips], iterations=4, smoothness=smoothness, translate=translate)
    assert len(got) == len(clips)
    for (a, tg), g in zip(clips, got):
        assert_same(g, rs.ik_solve(a, tg, iterations=4, smoothness=smoothness, translate=translate))


def golden_jobs(chd):
    rs = chd.results
    jobs = []
    for case, (s0, s1) in CASES.items():
        d = os.path.join(G, case)
        jobs.append((case, rs.load_towr_results(d + "/sol_out.txt"), d + "/anim.bvh", s0, s1))
    # a 2-foot result: the toe columns of the 4-foot `combined` one
    r = rs.load_towr_results(os.path.join(G, "combined", "sol_out.txt"))
    r2 = rs.TowrResults(2, r.dt, r.base_pos, r.base_rot, r.base_R, r.feet_pos[:, :2], r.feet_force[:, :2], r.feet_contact[:, :2])
    jobs.append(("combined", r2, os.path.join(G, "combined", "anim.bvh"), *CASES["combined"]))
    return jobs


def host_apply(rs, job, info, iterations=3, run_ik=True):
    """apply_results composed from its steps on the host: the set-up, then `ik_solve`."""
    anim, anim_og, com, targets = rs._apply_setup(*job, info, run_ik, None)
    if run_ik:
        anim = rs.ik_solve(anim, targets, iterations=iterations, smoothness=0.001, damping=7.0)
    return anim, anim.names, anim_og, com


@pytest.mark.parametrize("case", list(CASES))
def test_apply_results_batch_host_is_apply_results(chd, case):
    rs = chd.results
    jobs = [j for j in golden_jobs(chd) if j[0] == case]
    info = chd.prepare.CHARACTERS[case.split("_")[0]]()
    got = rs.apply_results_batch([j[1:] for j in jobs], info, iterations=3)
    for j, g in zip(jobs, got):
        ref = host_apply(rs, j[1:], info)
        assert_same(g[0], ref[0])
        assert_same(g[2], ref[2])
        assert g[1] == ref[1]
        np.testing.assert_array_equal(g[3], ref[3])
        one = rs.apply_results(*j[1:], info, iterations=3)          # a batch of one
        assert_same(one[0], g[0])
        assert_same(one[2], g[2])
        assert one[1] == g[1]
        np.testing.assert_array_equal(one[3], g[3])


def test_apply_results_batch_mixes_2_and_4_feet(chd):
    rs = chd.results
    jobs = [j for j in golden_jobs(chd) if j[0] == "combined"]
    jobs = [jobs[0], jobs[1], jobs[0]]                  # 4 feet, 2 feet, 4 feet: two target sets in one call
    info = chd.prepare.combined_info()
    got = rs.apply_results_batch([j[1:] for j in jobs], info, iterations=3)
    for j, g in zip(jobs, got):
        assert_same(g[0], host_apply(rs, j[1:], info)[0])
    got0 = rs.apply_results_batch([j[1:] for j in jobs], info, run_ik=False)
    for j, g in zip(jobs, got0):
        assert_same(g[0], host_apply(rs, j[1:], info, run_ik=False)[0])


def test_retarget_batch_host_is_retarget(chd, tmp_path):
    rs = chd.results
    src, skel, info = os.path.join(G, "combined", "anim.bvh"), os.path.join(G, "retarget", "ybot_skel.bvh"), chd.prepare.ybot_info()
    outs = [str(tmp_path / "a.bvh"), None]
    got = rs.retarget_batch([src, src], skel, info, out_bvhs=outs, iterations=3)
    # retarget composed from its steps on the host: skeleton, set-up, `ik_solve`, finish
    sk, h = rs._retarget_skeleton(skel, info)
    anim, tm, targets, src_floor = rs._retarget_setup(src, sk, h, info)
    anim = rs.ik_solve(anim, tm, iterations=3, smoothness=0.0, damping=7.0, translate=True)
    ref = rs._retarget_finish(anim, sk, targets, src_floor, info, str(tmp_path / "r.bvh"))
    for g in got:
        assert_same(g, ref)
    assert open(outs[0]).read() == open(str(tmp_path / "r.bvh")).read()
    one = rs.retarget(src, skel, info, out_bvh=str(tmp_path / "one.bvh"), iterations=3)     # a batch of one
    assert_same(one, got[0])
    assert open(str(tmp_path / "one.bvh")).read() == open(outs[0]).read()


def test_ik_solve_batch_refuses(chd):
    rs = chd.results
    a, tg = make_clip(chd, 3, 0)
    b, tb = make_clip(chd, 3, 1)
    other = rs.SkelAnim(b.names, b.parents.copy(), b.offsets, b.rotations, b.positions)
    other.parents[5] = 1
    with pytest.raises(ValueError, match="parents"):
        rs.ik_solve_batch([a, other], [tg, tb])
    with pytest.raises(ValueError, match="keys"):
        rs.ik_solve_batch([a, b], [tg, {k: v for k, v in list(tb.items())[1:]}])
    unordered = rs.SkelAnim(a.names, a.parents.copy(), a.offsets, a.rotations, a.positions)
    unordered.parents[3] = 7
    with pytest.raises(ValueError, match="ordered"):
        rs.ik_solve_batch([unordered], [tg])
    # J = 129 and T = 65: a chain of joints
    J = 129
    chain = rs.SkelAnim(["j%d" % i for i in range(J)], np.arange(-1, J - 1), np.ones((J, 3)), np.tile(np.eye(3), (2, J, 1, 1)), np.ones((2, J, 3)))
    with pytest.raises(ValueError, match="joints"):
        rs.ik_solve_batch([chain], [{0: np.zeros((2, 3))}])
    chain = rs.SkelAnim(chain.names[:100], chain.parents[:100], chain.offsets[:100], chain.rotations[:, :100], chain.positions[:, :100])
    with pytest.raises(ValueError, match="targets"):
        rs.ik_solve_batch([chain], [{j: np.zeros((2, 3)) for j in range(65)}])
    with pytest.raises(ValueError):
        rs.ik_solve_batch([a], [tg, tb])
