"""`chd_ik_solve` (the batched full-body IK kernel) and the batch entry points on cuda:0, against the host IK
(`ik_solve`, fp64) and the reference goldens."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.test_ik_batch_cpu import CASES, G, golden_jobs, make_clip
from tests.test_results_cpu import qmat

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROT_TOL, POS_TOL = 1e-9, 1e-7      # rotation-matrix entries, cm


def ik_pair(chd, anim, targets, **kw):
    rs = chd.results
    ref = rs.ik_solve(anim, targets, **kw)
    got = rs.ik_solve_batch([anim], [targets], device=DEV, **kw)[0]
    dr, dp = np.abs(got.rotations - ref.rotations).max(), np.abs(got.positions - ref.positions).max()
    print("max |dR| %.3e  max |dP| %.3e cm" % (dr, dp))
    return dr, dp


def test_kernel_matches_host_apply(chd):
    """`apply_results` on the 69-joint `ybot` golden (heels added, 61 targets): 30 iterations, smoothness 1e-3."""
    rs = chd.results
    s0, s1 = CASES["ybot"]
    d = os.path.join(G, "ybot")
    anim, _, _, tg = rs._apply_setup(rs.load_towr_results(d + "/sol_out.txt"), d + "/anim.bvh", s0, s1, chd.prepare.ybot_info(), True, None)
    assert len(anim.parents) == 69 and len(tg) == 61
    dr, dp = ik_pair(chd, anim, tg, iterations=30, smoothness=0.001, damping=7.0, translate=True)
    assert dr <= ROT_TOL and dp <= POS_TOL


def test_kernel_matches_host_retarget(chd):
    """`retarget` onto the 67-joint golden skeleton: 200 iterations, no smoothing, translating joints."""
    rs = chd.results
    sk, h = rs._retarget_skeleton(os.path.join(G, "retarget", "ybot_skel.bvh"), chd.prepare.ybot_info())
    anim, tm, _, _ = rs._retarget_setup(os.path.join(G, "combined", "anim.bvh"), sk, h, chd.prepare.ybot_info())
    dr, dp = ik_pair(chd, anim, tm, iterations=200, smoothness=0.0, damping=7.0, translate=True)
    assert dr <= ROT_TOL and dp <= POS_TOL


def test_kernel_matches_host_rotations_only(chd):
    """Like the kinematic initialisation's IK: 28-joint `combined`, rotations only, 200 iterations."""
    anim, tg = make_clip(chd, 40, 3, targets=[j for j in range(28) if j not in chd.kinopt.SPINE_IDX])
    dr, dp = ik_pair(chd, anim, tg, iterations=200, smoothness=0.0, damping=7.0, translate=False)
    assert dr <= ROT_TOL and dp == 0.0


@pytest.mark.parametrize("case", list(CASES))
def test_apply_results_batch_matches_reference(chd, case):
    rs = chd.results
    s0, s1 = CASES[case]
    d = os.path.join(G, case)
    a = np.load(d + "/applied.npz")
    info = chd.prepare.CHARACTERS[case.split("_")[0]]()
    jobs = [j[1:] for j in golden_jobs(chd) if j[0] == case]
    out = rs.apply_results_batch(jobs, info, device=DEV)
    an = out[0][0]
    np.testing.assert_allclose(an.rotations, qmat(a["rot_q"]), atol=5e-8)
    np.testing.assert_allclose(an.positions, a["pos"], atol=5e-8)
    np.testing.assert_allclose(an.global_positions(), a["gpos"], atol=1e-6)
    r = jobs[0][0]
    toe_err = np.linalg.norm(an.global_positions()[:, info.toes[0]] - r.feet_pos[:s1 - s0, 0] * 100.0, axis=1).mean()
    toe_err0 = np.linalg.norm(out[0][2].global_positions()[:, info.toes[0]] - r.feet_pos[:s1 - s0, 0] * 100.0, axis=1).mean()
    assert toe_err < 0.25 * toe_err0
    # every job (for `combined` also the 2-foot one, solved in its own group): the single-clip call on the device is the
    # batch element bitwise, and the host IK within tolerance
    for j, o in zip(jobs, out):
        one = rs.apply_results(*j, info, device=DEV)[0]
        np.testing.assert_array_equal(one.rotations, o[0].rotations)
        np.testing.assert_array_equal(one.positions, o[0].positions)
        ref = rs.apply_results(*j, info)[0]
        assert np.abs(o[0].rotations - ref.rotations).max() <= ROT_TOL
        assert np.abs(o[0].positions - ref.positions).max() <= POS_TOL


def test_retarget_batch_matches_reference(chd):
    rs = chd.results
    g = np.load(os.path.join(G, "retarget", "retarget.npz"))
    src, skel, info = os.path.join(G, "combined", "anim.bvh"), os.path.join(G, "retarget", "ybot_skel.bvh"), chd.prepare.ybot_info()
    one = rs.retarget(src, skel, info, device=DEV)
    host = rs.retarget(src, skel, info)
    assert np.abs(one.rotations - host.rotations).max() <= ROT_TOL
    assert np.abs(one.positions - host.positions).max() <= POS_TOL
    for a in rs.retarget_batch([src, src], skel, info, device=DEV):
        np.testing.assert_allclose(a.rotations, qmat(g["rot_q"]), atol=5e-7)
        np.testing.assert_allclose(a.positions, g["pos"], atol=2e-6)
        np.testing.assert_allclose(a.global_positions(), g["gpos"], atol=2e-5)
        np.testing.assert_allclose(a.positions[:, 1:], np.tile(a.offsets[None, 1:], (a.positions.shape[0], 1, 1)), atol=0)
        np.testing.assert_array_equal(a.rotations, one.rotations)          # the single-clip call is a batch of one
        np.testing.assert_array_equal(a.positions, one.positions)


def test_batch_invariance(chd):
    """Each clip's result is bitwise the same alone and in the batch, and over two runs."""
    rs = chd.results
    clips = [make_clip(chd, F, 10 + i) for i, F in enumerate((1, 2, 3, 14, 120, 600))]
    kw = dict(iterations=30, smoothness=0.001, damping=7.0, translate=True, device=DEV)
    batch = rs.ik_solve_batch([c[0] for c in clips], [c[1] for c in clips], **kw)
    again = rs.ik_solve_batch([c[0] for c in clips], [c[1] for c in clips], **kw)
    for (a, tg), b1, b2 in zip(clips, batch, again):
        alone = rs.ik_solve_batch([a], [tg], **kw)[0]
        for x in (b1, b2):
            np.testing.assert_array_equal(x.rotations, alone.rotations)
            np.testing.assert_array_equal(x.positions, alone.positions)
    # and the clips did move towards their targets
    a, tg = clips[4]
    tj = list(tg)
    goal = np.stack([tg[j] for j in tj], 1)
    assert np.linalg.norm(batch[4].global_positions()[:, tj] - goal, axis=-1).mean() < 0.5 * np.linalg.norm(a.global_positions()[:, tj] - goal, axis=-1).mean()


def test_entry_point_refuses_without_launching(chd):
    import torch
    L = chd.phys.load_lib()
    J, T, F = 28, 10, 6
    a, tg = make_clip(chd, F, 0, targets=list(range(T)))
    R = torch.as_tensor(a.rotations, device=DEV).contiguous()
    P = torch.as_tensor(a.positions, device=DEV).contiguous()
    goal = torch.as_tensor(np.stack([tg[j] for j in range(T)], 1), device=DEV).contiguous()
    work = torch.zeros(L.chd_ik_work_bytes(F, J, 64) // 8, dtype=torch.float64, device=DEV)
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ptr = lambda v: v.ctypes.data_as(C.c_void_p)
    parents, seg = i32(a.parents), i32([0, 2, F])
    stream = torch.cuda.current_stream().cuda_stream

    def call(par, tgt, sg, K, Tn):
        return L.chd_ik_solve(J, ptr(par), Tn, ptr(tgt), ptr(sg), K, F, R.data_ptr(), P.data_ptr(), goal.data_ptr(), 5, 7.0, 0.001, 1,
                              work.data_ptr(), stream)

    bad_parents = parents.copy()
    bad_parents[3] = 7
    assert call(parents, i32(range(65)), seg, 2, 65) == -1                 # T = 65
    assert call(bad_parents, i32(range(T)), seg, 2, T) == -1               # unordered parents
    assert call(parents, i32(range(T)), i32([0, 2, F - 1]), 2, T) == -1   # seg does not end at F_total
    torch.cuda.synchronize()
    np.testing.assert_array_equal(R.cpu().numpy(), a.rotations)
    np.testing.assert_array_equal(P.cpu().numpy(), a.positions)
    assert float(work.abs().sum()) == 0.0
    assert call(parents, i32(range(T)), seg, 2, T) == 0
    torch.cuda.synchronize()
    assert not np.array_equal(R.cpu().numpy(), a.rotations)
