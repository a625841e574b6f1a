"""Property tests (hypothesis) of the host-side pieces around the hot path: file round trips, rotation conventions, the
block-banded solver, the Huber estimator's optimality conditions."""
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st


@settings(max_examples=25, deadline=None, derandomize=True)
@given(seed=st.integers(0, 10_000), n_ee=st.sampled_from([2, 4]), N=st.integers(3, 40))
def test_solution_file_round_trip_through_load_results(chd, tmp_path_factory, seed, n_ee, N):
    """write_solution (phys_optim.cpp:63-143 layout, 10 significant digits) -> load_towr_results: positions come back with
    y / z swapped and flipped, forces likewise, contacts exact, rotation = C R C^T."""
    rng = np.random.default_rng(seed)
    sample = np.concatenate([rng.normal(0, 1, (N, 3)), rng.uniform(-170, 170, (N, 3)), rng.normal(0, 1, (N, 3 * n_ee)), rng.normal(0, 300, (N, 3 * n_ee)),
                             rng.integers(0, 2, (N, n_ee)).astype(float)], axis=1)
    sample[:, 4] = rng.uniform(-85, 85, N)                       # pitch away from the Euler singularity
    path = str(tmp_path_factory.mktemp("sol") / "sol.txt")
    chd.io_formats.write_solution(path, 1.0 / 30.0, sample, n_ee)
    r = chd.results.load_towr_results(path)
    assert r.num_feet == n_ee and r.base_pos.shape == (N, 3)
    base, pos, frc, flag = chd.phys.sample_columns(n_ee, n_ee)
    np.testing.assert_allclose(r.base_pos, -sample[:, base[[0, 2, 1]]], rtol=1e-9, atol=1e-12)
    for e in range(n_ee):
        np.testing.assert_allclose(r.feet_pos[:, e], -sample[:, pos[3 * e:3 * e + 3]][:, [0, 2, 1]], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(r.feet_force[:, e], -sample[:, frc[3 * e:3 * e + 3]][:, [0, 2, 1]], rtol=1e-9, atol=1e-9)
    np.testing.assert_array_equal(r.feet_contact, sample[:, flag].astype(int))
    C = chd.prepare.C_BVH_TO_TOWR
    R = chd.results.rot_zyx(np.radians(np.array([[float("%.10g" % v) for v in row] for row in sample[:, base[3:]]])))
    np.testing.assert_allclose(r.base_R, C @ R @ C.T, atol=1e-12)
    np.testing.assert_allclose(chd.results.rot_zyx(r.base_rot), r.base_R, atol=1e-9)      # base_rot are the Euler angles of base_R


@settings(max_examples=20, deadline=None, derandomize=True)
@given(seed=st.integers(0, 10_000), F=st.integers(1, 6))
def test_bvh_save_load_round_trip(chd, tmp_path_factory, seed, F):
    """save_bvh (Z Y X channels carrying the Euler angles of Rz Ry Rx) -> load_bvh -> local_transforms: same skeleton, same
    rotations to the printed precision; forward kinematics agree."""
    rng = np.random.default_rng(seed)
    P, O = chd.prepare.COMBINED_PARENTS, np.asarray(chd.prepare.COMBINED_OFFSETS, float)
    J = len(P)
    e = rng.uniform(-1.2, 1.2, (F, J, 3))
    pos = np.tile(O[None], (F, 1, 1))
    pos[:, 0] = rng.normal(0, 50, (F, 3))
    a = chd.results.SkelAnim(list(chd.prepare.COMBINED_NAMES), np.array(P), O, chd.results.rot_zyx(e), pos)
    path = str(tmp_path_factory.mktemp("bvh") / "a.bvh")
    chd.results.save_bvh(path, a, a.names, 1.0 / 30.0)
    b = chd.prepare.load_bvh(path)
    R, T = chd.prepare.local_transforms(b)
    np.testing.assert_allclose(R, a.rotations, atol=5e-8)
    np.testing.assert_allclose(T, a.positions, atol=1e-6)
    np.testing.assert_allclose(chd.prepare.forward_kinematics(b.parents, R, T)[0], a.global_positions(), atol=1e-4)
    np.testing.assert_allclose(chd.prepare.euler_zyx_from_matrix(a.rotations), e, atol=1e-9)


@settings(max_examples=15, deadline=None, derandomize=True)
@given(seed=st.integers(0, 10_000), F=st.integers(1, 7), n=st.integers(1, 5))
def test_block_pentadiagonal_solver(chd, seed, F, n):
    import torch
    g = torch.Generator().manual_seed(seed)
    N = F * n
    A = torch.zeros(N, N, dtype=torch.float64)
    for f in range(F):
        for k in range(3):
            if f + k < F:
                A[(f + k) * n:(f + k + 1) * n, f * n:(f + 1) * n] = torch.randn(n, n, generator=g, dtype=torch.float64) * 0.3
    A = A + A.T + torch.eye(N, dtype=torch.float64) * (4.0 + 2.0 * n)
    D = torch.stack([A[f * n:(f + 1) * n, f * n:(f + 1) * n] for f in range(F)])
    B1 = torch.stack([A[(f + 1) * n:(f + 2) * n, f * n:(f + 1) * n] for f in range(F - 1)]) if F > 1 else torch.zeros(0, n, n, dtype=torch.float64)
    B2 = torch.stack([A[(f + 2) * n:(f + 3) * n, f * n:(f + 1) * n] for f in range(F - 2)]) if F > 2 else torch.zeros(0, n, n, dtype=torch.float64)
    rhs = torch.randn(F, n, generator=g, dtype=torch.float64)
    lam = 0.01
    ref = torch.linalg.solve(A + lam * torch.diag(torch.diagonal(A)), rhs.reshape(-1))
    s = chd.kinopt._banded_cholesky_solve(torch, (D, B1, B2), rhs, lam).reshape(-1)
    np.testing.assert_allclose(s.numpy(), ref.numpy(), rtol=1e-9, atol=1e-11)


@settings(max_examples=15, deadline=None, derandomize=True)
@given(seed=st.integers(0, 10_000), eps=st.sampled_from([1.35, 1.5, 2.2]))
def test_huber_fit_first_order_conditions(chd, seed, eps):
    """At the returned point the gradient of the concomitant-scale Huber objective vanishes (to the L-BFGS tolerance) and
    outliers are exactly the residuals beyond eps * scale."""
    rng = np.random.default_rng(seed)
    n = 60
    X = rng.uniform(-50, 50, (n, 2))
    y = X @ rng.normal(0, 0.1, 2) + rng.normal(0, 1.0) * 10 + rng.normal(0, 0.5, n)
    y[:6] += rng.uniform(5, 20, 6)
    w, c, s, out = chd.kinopt.huber_fit(X, y, eps)
    res = y - X @ w - c
    np.testing.assert_array_equal(out, np.abs(res) > eps * s)
    gin = ~out
    gw = -2.0 * eps * (X[out].T @ np.sign(res[out])) - 2.0 / s * (X[gin].T @ res[gin]) + 2e-4 * w
    gc = -2.0 * eps * np.sign(res[out]).sum() - 2.0 / s * res[gin].sum()
    gs = n - out.sum() * eps ** 2 - (res[gin] ** 2).sum() / s ** 2
    scale = 2.0 / s * (np.abs(X) * np.abs(res)[:, None]).sum()        # natural size of the terms that cancel in gw
    assert np.abs(gw).max() < 1e-3 * scale and abs(gc) < 1e-3 * scale / 25.0 and abs(gs) < 1e-2


@settings(max_examples=10, deadline=None, derandomize=True)
@given(seed=st.integers(0, 1000))
def test_ik_reaches_reachable_targets(chd, seed):
    """Targets generated by the skeleton itself are reachable: the damped IK drives the error to (near) zero from a perturbed pose."""
    rng = np.random.default_rng(seed)
    P, O = np.array(chd.prepare.COMBINED_PARENTS), np.asarray(chd.prepare.COMBINED_OFFSETS, float)
    F, J = 3, len(P)
    e = rng.uniform(-0.5, 0.5, (F, J, 3))
    pos = np.tile(O[None], (F, 1, 1))
    truth = chd.results.SkelAnim(["j"] * J, P, O, chd.results.rot_zyx(e), pos)
    gp = truth.global_positions()
    start = chd.results.SkelAnim(["j"] * J, P, O, chd.results.rot_zyx(e + rng.normal(0, 0.15, e.shape)), pos.copy())
    hist = []
    chd.results.ik_solve(start, {j: gp[:, j] for j in range(1, J)}, iterations=60, damping=1.0, smoothness=0.0, translate=False, history=hist)
    assert hist[-1] < 0.05 * hist[0] + 1e-6
