"""Batched kinematic initialisation (`optimize_trajectory_batch`, `optimize_2d_3d_batch`) on the CPU: every clip of a batch
reproduces its own single-clip run, and no residual row couples two clips."""
import os

import numpy as np
import pytest

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kinopt")
ARGS = ("poses2D", "conf", "poses3D", "root_pos", "ang", "parents", "offsets", "ppx", "ppy", "focal", "vel")


def golden_clip(chd):
    inp, run = np.load(os.path.join(G, "inputs.npz")), np.load(os.path.join(G, "run.npz"))
    b = chd.prepare.load_bvh(os.path.join(G, "skeleton.bvh"))
    return dict(poses2D=inp["poses2D"], conf=inp["conf"], poses3D=inp["poses3D"], root_pos=inp["root_pos"], ang=inp["joint_angles"],
                parents=b.parents, offsets=b.offsets, ppx=inp["pp"][0], ppy=inp["pp"][1], focal=inp["focal"], vel=inp["vel"],
                normal=run["plane_normal"], point=run["plane_point"])


def synth_clip(chd, d, F, seed):
    ko = chd.kinopt
    chd.synth.write_mocap_clip(d, F, seed=seed)
    kp = chd.contact.load_keypoint_dir(os.path.join(d, "openpose_result"))
    p3, rp, ang = ko.combined_inputs(ko.load_totalcap_results(os.path.join(d, "tracked_results.json")))
    b = chd.prepare.load_bvh(os.path.join(d, "skeleton.bvh"))
    return dict(poses2D=np.concatenate([kp[:, :, :2], np.zeros((F, 3, 2))], 1), conf=np.concatenate([kp[:, :, 2], np.zeros((F, 3))], 1),
                poses3D=p3, root_pos=rp, ang=ang, parents=b.parents, offsets=b.offsets, ppx=960.0, ppy=540.0, focal=np.array(ko.MTC_FOCAL),
                vel=ko.contacts_to_constraints(np.load(os.path.join(d, "foot_contacts.npy"))), normal=None, point=None)


def run_single(chd, c, **kw):
    return chd.kinopt.optimize_trajectory(*[c[a] for a in ARGS], plane_normal=c["normal"], plane_point=c["point"], **kw)


def run_batch(chd, clips, **kw):
    return chd.kinopt.optimize_trajectory_batch(*[[c[a] for c in clips] for a in ARGS], plane_normal=[c["normal"] for c in clips],
                                                plane_point=[c["point"] for c in clips], **kw)


@pytest.fixture(scope="module")
def clips(chd, tmp_path_factory):
    d = tmp_path_factory.mktemp("kinb")
    return [golden_clip(chd)] + [synth_clip(chd, str(d / ("c%d" % F)), F, seed) for F, seed in ((13, 11), (24, 12), (40, 13))]


def assert_same_result(one, bat):
    a1, n1, p1, pn1, pp1, v1, i1 = one
    a2, n2, p2, pn2, pp2, v2, i2 = bat
    for st in ("stage1", "stage2"):
        assert i1[st]["nfev"] == i2[st]["nfev"], st
        assert abs(i1[st]["cost"] - i2[st]["cost"]) <= 1e-9 * i1[st]["cost"], st
    np.testing.assert_allclose(n2, n1, rtol=0, atol=1e-5)
    np.testing.assert_allclose(pn2, pn1, rtol=0, atol=1e-9)
    np.testing.assert_allclose(pp2, pp1, rtol=0, atol=1e-6)
    np.testing.assert_array_equal(v2, v1)


def test_batch_matches_each_clip(chd, clips):
    kw = dict(ik_iterations=60, max_nfev=25)
    singles = [run_single(chd, c, **kw) for c in clips]
    batch = run_batch(chd, clips, **kw)
    assert len(batch) == len(clips)
    for one, bat in zip(singles, batch):
        assert_same_result(one, bat)
    assert all(r[6]["stage2"]["nfev"] > 1 for r in batch)


def test_batch_of_one_is_the_single_clip_call(chd, clips):
    kw = dict(ik_iterations=60, max_nfev=25)
    assert_same_result(run_single(chd, clips[2], **kw), run_batch(chd, clips[2:3], **kw)[0])


def test_no_row_couples_two_clips(chd, clips):
    """The batch Jacobian is block diagonal over the clips and holds exactly the rows of every clip's own Jacobian."""
    import torch
    ko = chd.kinopt
    probs, xs = [], []
    rng = np.random.default_rng(0)
    for c in clips[1:]:
        j2n, pw, dw = ko.make_weights(c["poses2D"], c["conf"], (c["ppx"], c["ppy"]), c["focal"])
        F = c["poses3D"].shape[0]
        n = rng.normal(size=3)
        probs.append(ko.Problem(c["parents"], c["offsets"] * rng.uniform(0.9, 1.1), c["poses3D"], c["root_pos"], j2n, pw, dw, c["vel"],
                                n / np.linalg.norm(n), rng.normal(size=3)))
        x = np.zeros((F, ko.NV))
        x[:, :3] = c["root_pos"]
        xs.append(x + rng.normal(0, 0.1, x.shape))
    probs = [probs[0], probs[1]]
    probs[0].poses3D, probs[0].root_trans, probs[0].joints2d = probs[0].poses3D[:5], probs[0].root_trans[:5], probs[0].joints2d[:5]
    probs[0].proj_w, probs[0].data_w, probs[0].contacts = probs[0].proj_w[:5], probs[0].data_w[:5], probs[0].contacts[:5]
    probs[1].poses3D, probs[1].root_trans, probs[1].joints2d = probs[1].poses3D[:4], probs[1].root_trans[:4], probs[1].joints2d[:4]
    probs[1].proj_w, probs[1].data_w, probs[1].contacts = probs[1].proj_w[:4], probs[1].data_w[:4], probs[1].contacts[:4]
    xs = [xs[0][:5], xs[1][:4]]
    w = ko.StageWeights(floor=10.0)
    bm = ko._Model(probs, None)
    Jb = bm.dense_jacobian(torch.as_tensor(np.concatenate(xs)), w).numpy()
    Js = [ko._Model(p).dense_jacobian(torch.as_tensor(x), w).numpy() for p, x in zip(probs, xs)]
    assert Jb.shape == (sum(J.shape[0] for J in Js), sum(J.shape[1] for J in Js))
    c0 = Js[0].shape[1]
    in0, in1 = np.abs(Jb[:, :c0]).sum(1) > 0, np.abs(Jb[:, c0:]).sum(1) > 0
    assert not (in0 & in1).any()                                          # no row touches both clips
    for k, J in enumerate(Js):
        blk = Jb[in0][:, :c0] if k == 0 else Jb[in1][:, c0:]
        own = J[np.abs(J).sum(1) > 0]
        # same set of rows (the batch orders them group by group over the concatenated frames)
        key = lambda M: M[np.lexsort(M.T[::-1])]
        assert blk.shape == own.shape
        np.testing.assert_allclose(key(blk), key(own), rtol=1e-12, atol=1e-12)
    # and the normal equations carry no coupling block between the clips
    cost, H, g = bm.normal_equations(torch.as_tensor(np.concatenate(xs)), w)
    assert float(H[1][4].abs().max()) == 0.0 and float(H[2][3].abs().max()) == 0.0 and float(H[2][4].abs().max()) == 0.0
    for k, (p, x) in enumerate(zip(probs, xs)):
        c1 = ko._Model(p).cost(torch.as_tensor(x), w)
        assert abs(cost[k] - c1) <= 1e-12 * c1


def test_optimize_2d_3d_batch_writes_per_video_files(chd, tmp_path):
    ko = chd.kinopt
    jobs = []
    for F, seed in ((12, 21), (17, 22)):
        vd = str(tmp_path / ("v%d" % F))
        chd.synth.write_mocap_clip(vd, F, seed=seed)
        jobs.append((os.path.join(vd, "w.mp4"), os.path.join(vd, "skeleton.bvh"), str(tmp_path / ("kb%d" % F)), 0, F, False))
    out = ko.optimize_2d_3d_batch(jobs)
    assert len(out) == 2
    for (inp, sk, op, lo, hi, gt), res in zip(jobs, out):
        ref = str(tmp_path / ("ks_" + os.path.basename(op)))
        ko.optimize_2d_3d(inp, sk, ref, lo, hi, gt)
        np.testing.assert_array_equal(np.load(os.path.join(op, "foot_contacts.npy")), np.load(os.path.join(ref, "foot_contacts.npy")))
        fa = np.array(open(os.path.join(op, "floor_out.txt")).read().split(), dtype=np.float64)
        fb = np.array(open(os.path.join(ref, "floor_out.txt")).read().split(), dtype=np.float64)
        np.testing.assert_allclose(fa, fb, rtol=0, atol=1e-9)
        ba, bb = chd.prepare.load_bvh(os.path.join(op, "final_test.bvh")), chd.prepare.load_bvh(os.path.join(ref, "final_test.bvh"))
        assert ba.names == bb.names
        la, lb = open(os.path.join(op, "final_test.bvh")).read().split(), open(os.path.join(ref, "final_test.bvh")).read().split()
        assert len(la) == len(lb)
        num = [(a, b) for a, b in zip(la, lb) if a != b]
        assert all(abs(float(a) - float(b)) <= 2e-6 for a, b in num)       # six decimals: at most a last-digit flip
