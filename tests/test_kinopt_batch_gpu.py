"""`chd_kin_solve` (the block-banded Cholesky kernel of the batched kinematic initialisation) and
`optimize_2d_3d_batch` on cuda:0."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LENS = (1, 2, 3, 14, 120, 600)
LAMS = (1e-3, 3e-2, 1e-1, 1e-3, 5e-3, 2e-4)


@pytest.fixture(scope="module")
def systems(chd, tmp_path_factory):
    """Normal equations of synthetic clips of every length in LENS (frames of one 600-frame walk), on the host."""
    import torch
    ko = chd.kinopt
    vd = str(tmp_path_factory.mktemp("kin") / "walk")
    chd.synth.write_mocap_clip(vd, 600, seed=7)
    kp = chd.contact.load_keypoint_dir(os.path.join(vd, "openpose_result"))
    p3, rp, ang = ko.combined_inputs(ko.load_totalcap_results(os.path.join(vd, "tracked_results.json")))
    b = chd.prepare.load_bvh(os.path.join(vd, "skeleton.bvh"))
    vel = ko.contacts_to_constraints(np.load(os.path.join(vd, "foot_contacts.npy")))
    rng = np.random.default_rng(1)
    out = []
    for i, F in enumerate(LENS):
        a = (37 * i) % (600 - F + 1)
        sl = slice(a, a + F)
        j2n, pw, dw = ko.make_weights(np.concatenate([kp[sl, :, :2], np.zeros((F, 3, 2))], 1), np.concatenate([kp[sl, :, 2], np.zeros((F, 3))], 1),
                                      (960.0, 540.0), np.array(ko.MTC_FOCAL))
        off = ko.update_skeleton(b.parents, b.offsets, p3[sl][:, ko.FORWARD] + rp[sl][:, None])
        p = ko.Problem(b.parents, off, p3[sl], rp[sl], j2n, pw, dw, vel[sl], np.array([0.0, -1.0, 0.0]), np.array([0.0, 92.0, 0.0]))
        x = np.zeros((F, ko.NV))
        x[:, :3] = rp[sl]
        x[:, 3:] = rng.normal(0, 0.2, (F, ko.NV - 3))
        cost, H, g = ko._Model(p).normal_equations(torch.as_tensor(x), ko.StageWeights(floor=10.0))
        out.append((H, g))
    return out


def launch(chd, systems, lams, sel=None):
    """Concatenates the systems, runs one chd_kin_solve launch; returns (s per clip, status) on the host."""
    import torch
    L = chd.phys.load_lib()
    dev = torch.device("cuda:0")
    lens = [H[0].shape[0] for H, _ in systems]
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    Ft = int(seg[-1])
    D = torch.cat([H[0] for H, _ in systems]).to(dev).contiguous()
    B1, B2 = torch.zeros(max(Ft - 1, 0), 87, 87, dtype=torch.float64), torch.zeros(max(Ft - 2, 0), 87, 87, dtype=torch.float64)
    for k, (H, _) in enumerate(systems):
        a, n = int(seg[k]), lens[k]
        B1[a:a + max(n - 1, 0)] = H[1]
        B2[a:a + max(n - 2, 0)] = H[2]
    B1, B2 = B1.to(dev), B2.to(dev)
    g = torch.cat([gg for _, gg in systems]).to(dev).contiguous()
    s = torch.full((Ft, 87), float("nan"), dtype=torch.float64, device=dev)
    st = torch.full((len(systems),), -7, dtype=torch.int32, device=dev)
    work = torch.empty(L.chd_kin_work_bytes(Ft) // 8, dtype=torch.float64, device=dev)
    segd = torch.as_tensor(seg, device=dev)
    lamd = torch.as_tensor(np.asarray(lams, np.float64), device=dev)
    seld = torch.as_tensor(np.asarray(sel, np.int32), device=dev) if sel is not None else None
    p = lambda a: a.data_ptr() if a is not None and a.numel() else None
    rc = L.chd_kin_solve(p(D), p(B1), p(B2), p(g), p(segd), p(lamd), p(seld), len(sel) if sel is not None else 0, len(systems), Ft,
                         p(work), p(s), p(st), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    s = s.cpu()
    return [s[seg[k]:seg[k + 1]].clone() for k in range(len(systems))], st.cpu().numpy()


def damped(H, lam):
    import torch
    D = H[0]
    return D + lam * torch.diag_embed(torch.diagonal(D, dim1=1, dim2=2).clamp_min(1e-12))


def band_matvec(H, Dd, s):
    r = (Dd @ s[:, :, None])[..., 0]
    if s.shape[0] > 1:
        r[1:] += (H[1] @ s[:-1, :, None])[..., 0]
        r[:-1] += (H[1].transpose(1, 2) @ s[1:, :, None])[..., 0]
    if s.shape[0] > 2:
        r[2:] += (H[2] @ s[:-2, :, None])[..., 0]
        r[:-2] += (H[2].transpose(1, 2) @ s[2:, :, None])[..., 0]
    return r


def test_kin_solve_mixed_batch_matches_references(chd, systems):
    import torch
    ko = chd.kinopt
    sols, st = launch(chd, systems, LAMS)
    assert (st == 0).all(), st
    for (H, g), lam, s in zip(systems, LAMS, sols):
        F = g.shape[0]
        ref = ko._banded_cholesky_solve(torch, H, g, lam)
        np.testing.assert_allclose(s.numpy(), ref.numpy(), rtol=1e-8, atol=1e-10)
        Dd = damped(H, lam)
        if F <= 120:
            A = np.zeros((F * 87, F * 87))
            for f in range(F):
                A[f * 87:(f + 1) * 87, f * 87:(f + 1) * 87] = Dd[f].numpy()
                if f + 1 < F:
                    A[(f + 1) * 87:(f + 2) * 87, f * 87:(f + 1) * 87] = H[1][f].numpy()
                    A[f * 87:(f + 1) * 87, (f + 1) * 87:(f + 2) * 87] = H[1][f].numpy().T
                if f + 2 < F:
                    A[(f + 2) * 87:(f + 3) * 87, f * 87:(f + 1) * 87] = H[2][f].numpy()
                    A[f * 87:(f + 1) * 87, (f + 2) * 87:(f + 3) * 87] = H[2][f].numpy().T
            np.testing.assert_allclose(s.numpy().reshape(-1), np.linalg.solve(A, g.numpy().reshape(-1)), rtol=1e-6, atol=1e-9)
        # normwise backward error, ||A|| bounded by the Frobenius norm of the band
        r = band_matvec(H, Dd, s) - g
        nA = float(torch.sqrt((Dd ** 2).sum() + 2 * (H[1] ** 2).sum() + 2 * (H[2] ** 2).sum()))
        eta = float(r.norm()) / (nA * float(s.norm()) + float(g.norm()))
        assert eta <= 1e-11, (F, eta)


def test_kin_solve_bitwise_alone_in_batch_and_between_launches(chd, systems):
    import torch
    sols, _ = launch(chd, systems, LAMS)
    again, _ = launch(chd, systems, LAMS)
    for a, b in zip(sols, again):
        assert torch.equal(a, b)
    for k in (0, 3, 4):
        alone, st = launch(chd, [systems[k]], [LAMS[k]])
        assert st[0] == 0 and torch.equal(alone[0], sols[k])
    # a selection of clips: the others are not touched
    part, st = launch(chd, systems, LAMS, sel=[4, 1])
    assert list(st) == [-7, 0, -7, -7, 0, -7]
    assert torch.equal(part[4], sols[4]) and torch.equal(part[1], sols[1]) and bool(torch.isnan(part[0]).all())


def test_kin_solve_reports_the_indefinite_block(chd, systems):
    import torch
    sols, _ = launch(chd, systems, LAMS)
    bad = list(systems)
    H, g = systems[3]
    f = 9
    D = H[0].clone()
    D[f] = -D[f]
    bad[3] = ((D, H[1], H[2]), g)
    got, st = launch(chd, bad, LAMS)
    assert st[3] == f + 1
    assert all(st[k] == 0 for k in range(len(bad)) if k != 3)
    for k in range(len(bad)):
        if k != 3:
            assert torch.equal(got[k], sols[k])


def test_optimize_2d_3d_batch_on_gpu_matches_cpu(chd, tmp_path):
    import torch
    assert torch.cuda.is_available()
    ko = chd.kinopt
    jobs = []
    for F, seed in ((24, 31), (40, 32), (290, 33)):
        vd = str(tmp_path / ("v%d" % F))
        chd.synth.write_mocap_clip(vd, F, seed=seed)
        jobs.append((os.path.join(vd, "w.mp4"), os.path.join(vd, "skeleton.bvh"), str(tmp_path / ("g%d" % F)), 0, F, False))
    gpu = ko.optimize_2d_3d_batch(jobs, device="cuda:0")
    for job, rg in zip(jobs, gpu):
        rc = ko.optimize_2d_3d(job[0], job[1], job[2] + "_cpu", job[3], job[4], job[5])
        c0, c1 = rc[-1]["stage2"]["cost"], rg[-1]["stage2"]["cost"]
        assert abs(c0 - c1) < 1e-3 * c0
        assert np.linalg.norm(rc[1] - rg[1], axis=-1).max() < 0.5
        np.testing.assert_allclose(rc[3], rg[3], atol=1e-3)
        for name in ("foot_contacts.npy", "floor_out.txt", "final_test.bvh"):
            assert os.path.isfile(os.path.join(job[2], name))
