"""Kinematic initialisation (SURVEY.md 8(a) rows E1-E3, 8(f) rank 2): refine a monocular 3D pose track on the `combined`
skeleton so that it re-projects onto the 2D detections, stays smooth, keeps contact feet still and on a fitted floor.

Reference: `src/optimize/optimize_trajectory.py` -- residual vector `fun_anim_for_projection` (:324-483), Jacobian
`jac_anim_for_projection_sparse` / `jac_root_all_for_projection` (:51-322), skeleton fit `update_skeleton` (:485-520), driver
`optimize_trajectory` (:522-834: IK initialisation, two `scipy.least_squares(max_nfev=50, tr_solver='lsmr')` stages,
Huber floor fit + contact pruning in between).

What is different here, deliberately (GPU-first):
* The reference materialises a dense (terms x 84 F) Jacobian in Python loops (4 GB at 120 frames), multiplies it frame by
  frame with the IK Jacobian and hands a `lil_matrix` to LSMR.  Every residual is *linear* in the joint positions of at most
  three consecutive frames (only the projection term is not, and it touches one frame), so J = A * blockdiag(dP_f/dx_f) + E
  with tiny per-frame blocks: the Gauss-Newton matrix J^T J is block-pentadiagonal with 87 x 87 blocks and is assembled
  and factorised directly (batched matmuls over the frames + one block-banded Cholesky sweep), on the GPU when a device is
  given.  Levenberg-Marquardt with gain-ratio control replaces the trust-region/LSMR loop; same evaluation budget (50).
* The reference's analytic Jacobian of the projection term is not the derivative of its residual: the root-translation
  columns are written at the columns of body-25 joint 0 (the nose) instead of the root's (`varIndex + 0` without
  `root_idx * 3`, optimize_trajectory.py:106-137), so d(projection)/d(root translation) is missing for every joint but the
  root and the nose picks up a spurious term.  The residual here is the reference's, term for term (tested against the
  reference's own function); the Jacobian is the exact derivative (tested by finite differences, and equal to the
  reference's in every other block).
Units: cm, camera frame (x right, y down, z forward), angles in radians, Euler x, y, z with R = Rz Ry Rx per joint.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from .results import SkelAnim, descendants_mask, ik_solve, rot_zyx

# ---- the `combined` skeleton <-> BODY_25(+3 spine) correspondence and per-joint weights (SkeletonDefinitions.py:62-140) ----
ROOT_IDX = 8                                    # MidHip in body-25 order
FEET_IDX = [4, 5, 6, 10, 11, 12]                # skeleton joints: heels and toes
SPINE_IDX = [13, 14, 15]
# skeleton joint -> body-25 index
FORWARD = [8, 12, 13, 14, 21, 19, 20, 9, 10, 11, 24, 22, 23, 25, 26, 27, 1, 0, 16, 18, 15, 17, 5, 6, 7, 2, 3, 4]
BACKWARD = [int(i) for i in np.argsort(FORWARD)]   # body-25 index -> skeleton joint
PROJ_WEIGHTS = np.array([0.1, 0.1, 0.3, 0.1, 0.1, 0.3, 0.1, 0.1, 0.1, 1.0, 0.1, 0.1, 1.0] + [0.1] * 12 + [0.0] * 3)
DATA_WEIGHTS = np.array([2.5] + [1.0] * 14 + [2.5] * 4 + [1.0] * 6 + [0.0] * 3)
SMOOTH_WEIGHTS = np.array([2.5, 2.5, 2.5, 1.5, 1.0, 2.5, 1.5, 1.0, 1.0, 2.5, 1.5, 1.0, 2.5, 1.5] + [1.0] * 11 + [1.5] * 3)
SMOOTH_VEL = np.array([1.0, 1.0, 2.0])          # per axis, optimize_trajectory.py:42-44
SMOOTH_EULER = 10.0                             # :45-47
NJ = 28
NV = 3 * (NJ + 1)                               # unknowns per frame: root translation + 28 Euler triples


@dataclass
class StageWeights:
    proj: float = 1000.0
    smooth_vel: float = 0.1
    smooth_acc: float = 0.5
    data: float = 0.3
    vel: float = 10.0
    floor: float = 0.0


@dataclass
class Problem:
    """Everything the residual needs besides x (all numpy, body-25 joint order where per joint)."""
    parents: np.ndarray          # (28,) skeleton
    offsets: np.ndarray          # (28, 3) fitted skeleton, root offset 0
    poses3D: np.ndarray          # (F, 28, 3) root-relative data
    root_trans: np.ndarray       # (F, 3)
    joints2d: np.ndarray         # (F, 28, 2) normalised image coordinates
    proj_w: np.ndarray           # (F, 28)
    data_w: np.ndarray           # (F, 28)
    contacts: np.ndarray         # (F, 28) 0/1
    floor_normal: np.ndarray
    floor_point: np.ndarray


def update_skeleton(parents, offsets, targets):
    """optimize_trajectory.py:485-520: bone lengths = per-bone median over the frames of the target joint distances; the three
    spine bones each get a third of the root -> Spine2 distance; directions stay those of the template; root offset 0."""
    parents = np.asarray(parents)
    J = len(parents)
    bones = np.zeros(J)
    for j in range(1, J):
        if j in SPINE_IDX:
            bones[j] = np.median(np.linalg.norm(targets[:, SPINE_IDX[2]] - targets[:, 0], axis=1) / 3.0)
        else:
            bones[j] = np.median(np.linalg.norm(targets[:, j] - targets[:, parents[j]], axis=1))
    out = np.asarray(offsets, dtype=np.float64).copy()
    out[1:] = out[1:] / np.linalg.norm(out[1:], axis=1, keepdims=True) * bones[1:, None]
    out[0] = 0.0
    return out


def make_weights(poses2D, conf, cam_center, focal):
    """optimize_trajectory.py:553-573: normalised 2D coordinates, projection and data weights (spine joints 25-27 have no 2D)."""
    j2n = np.asarray(poses2D, dtype=np.float64).copy()
    j2n[:, :25] = (j2n[:, :25] - np.asarray(cam_center)) / np.asarray(focal)
    pw = conf * PROJ_WEIGHTS
    pw[:, 25:] = 0.0
    dw = (1.0 + conf) * DATA_WEIGHTS
    dw[:, 25:] = (1.0 + 0.4) * DATA_WEIGHTS[25:]
    return j2n, pw, dw


class _Model:
    """Residuals and the block structure of their Jacobian, batched over the frames (torch, fp64)."""

    def __init__(self, p: Problem, device=None):
        import torch
        self.t = torch
        self.dev = torch.device(device) if device is not None else torch.device("cpu")
        f64 = dict(dtype=torch.float64, device=self.dev)
        self.f64 = f64
        self.p = p
        self.F = p.poses3D.shape[0]
        self.parents = [int(v) for v in p.parents]
        self.off = torch.as_tensor(p.offsets, **f64)
        self.back = torch.as_tensor(BACKWARD, device=self.dev)
        self.desc = torch.as_tensor(descendants_mask(self.parents).astype(np.float64), **f64)   # [m, k]: k strict descendant of m
        self.par_idx = torch.as_tensor([max(q, 0) for q in self.parents], device=self.dev)
        self.root_mask = torch.as_tensor([q < 0 for q in self.parents], device=self.dev)
        as_t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), **f64)
        self.poses3D, self.root_trans, self.j2n = as_t(p.poses3D), as_t(p.root_trans), as_t(p.joints2d)
        self.pw, self.dw, self.con = as_t(p.proj_w), as_t(p.data_w), as_t(p.contacts)
        self.n, self.pt = as_t(p.floor_normal), as_t(p.floor_point)
        self.sw = as_t(SMOOTH_WEIGHTS)[:, None] * as_t(SMOOTH_VEL)[None, :]            # (28, 3)
        self.is_root = torch.zeros(NJ, **f64)
        self.is_root[ROOT_IDX] = 1.0

    # ---- forward kinematics: y (F, 28, 3) in body-25 order (root entry = root translation, others root-relative) ----
    def points(self, x, jac=False):
        t = self.t
        F = x.shape[0]
        e = x[:, 3:].reshape(F, NJ, 3)
        cx, sx, cy, sy, cz, sz = t.cos(e[..., 0]), t.sin(e[..., 0]), t.cos(e[..., 1]), t.sin(e[..., 1]), t.cos(e[..., 2]), t.sin(e[..., 2])
        Rl = t.stack([t.stack([cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx], -1),
                      t.stack([sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx], -1), t.stack([-sy, cy * sx, cy * cx], -1)], -2)
        gR, gP = [None] * NJ, [None] * NJ
        for j in range(NJ):
            q = self.parents[j]
            if q < 0:
                gR[j], gP[j] = Rl[:, j], t.zeros(F, 3, **self.f64)
            else:
                gR[j] = gR[q] @ Rl[:, j]
                gP[j] = gP[q] + gR[q] @ self.off[j]
        gR, gP = t.stack(gR, 1), t.stack(gP, 1)                                       # skeleton order, root at the origin
        y = gP[:, self.back].clone()
        y[:, ROOT_IDX] = x[:, :3]
        if not jac:
            return y, None
        # dP: (F, 28 points [body order], 3, 87): d y / d x_f
        prs = gR[:, self.par_idx].clone()
        prs[:, self.root_mask] = t.eye(3, **self.f64)
        ax = t.stack([t.stack([cz * cy, sz * cy, -sy], -1), t.stack([-sz, cz, t.zeros_like(cz)], -1),
                      t.stack([t.zeros_like(cz), t.zeros_like(cz), t.ones_like(cz)], -1)], 2)   # (F, J, axis, 3) in the parent frame
        ax = t.einsum("fjab,fjkb->fjka", prs, ax)
        arm = gP[:, None, :, :] - gP[:, :, None, :]                                    # (F, m, k, 3): point k minus joint m
        d = t.cross(ax[:, :, :, None, :].expand(F, NJ, 3, NJ, 3), arm[:, :, None, :, :].expand(F, NJ, 3, NJ, 3), dim=-1)
        d = d * self.desc[None, :, None, :, None]                                      # (F, m, axis, k, 3)
        dP = t.zeros(F, NJ, 3, NV, **self.f64)
        dP[:, :, :, 3:] = d.permute(0, 3, 4, 1, 2).reshape(F, NJ, 3, 3 * NJ)[:, self.back]
        dP[:, ROOT_IDX] = 0.0
        dP[:, ROOT_IDX, 0, 0] = dP[:, ROOT_IDX, 1, 1] = dP[:, ROOT_IDX, 2, 2] = 1.0
        return y, dP

    # ---- residual groups; each returns (r, [(frame offset d, dr/dy_{f+d} as (F', rows, 84))]) ----
    def residuals(self, x, w: StageWeights, jac=False):
        """List of (base frames F', r (F', rows), blocks {d: G (F', rows, 87)} = dr/dx_{f+d})."""
        t = self.t
        F = self.F
        y, dP = self.points(x, jac)
        out = []
        eye3 = t.eye(3, **self.f64)
        nr = 1.0 - self.is_root                                                       # 0 for the root entry
        # absolute position of every point: root + relative (the root entry itself is the root)
        root = y[:, ROOT_IDX]
        ab = y + root[:, None, :] * nr[None, :, None]
        dab = None
        if jac:
            dab = dP + dP[:, ROOT_IDX][:, None] * nr[None, :, None, None]             # d(abs point)/dx_f
        # 1. projection (own frame)
        on = (self.pw > 0).to(t.float64)
        wp = w.proj * self.pw * on
        z = t.where(ab[..., 2] == 0, t.ones_like(ab[..., 2]), ab[..., 2])
        pr = t.stack([ab[..., 0] / z, ab[..., 1] / z], -1)
        r = (wp[..., None] * (pr - self.j2n)).reshape(F, -1)
        G = None
        if jac:
            dpr = t.stack([(dab[:, :, 0] * z[..., None] - ab[..., 0, None] * dab[:, :, 2]) / (z * z)[..., None],
                           (dab[:, :, 1] * z[..., None] - ab[..., 1, None] * dab[:, :, 2]) / (z * z)[..., None]], 2)   # (F, 28, 2, 87)
            G = {0: (wp[..., None, None] * dpr).reshape(F, -1, NV)}
        out.append((0, r, G))
        # 2. velocity smoothness of the points (frames f, f+1)
        ws = w.smooth_vel * self.sw
        if F > 1:
            r = (ws[None] * (y[:-1] - y[1:])).reshape(F - 1, -1)
            G = None
            if jac:
                g0 = (ws[None, :, :, None] * dP[:-1]).reshape(F - 1, -1, NV)
                g1 = (-ws[None, :, :, None] * dP[1:]).reshape(F - 1, -1, NV)
                G = {0: g0, 1: g1}
            out.append((0, r, G))
        # 3. acceleration smoothness (frames f, f+1, f+2)
        if F > 2:
            r = (w.smooth_acc * (y[2:] - 2.0 * y[1:-1] + y[:-2])).reshape(F - 2, -1)
            G = None
            if jac:
                G = {0: (w.smooth_acc * dP[:-2]).reshape(F - 2, -1, NV), 1: (-2.0 * w.smooth_acc * dP[1:-1]).reshape(F - 2, -1, NV),
                     2: (w.smooth_acc * dP[2:]).reshape(F - 2, -1, NV)}
            out.append((0, r, G))
        # 4. data
        tgt = self.poses3D * nr[None, :, None] + self.root_trans[:, None, :] * self.is_root[None, :, None]
        wd = w.data * self.dw
        r = (wd[..., None] * (y - tgt)).reshape(F, -1)
        G = {0: (wd[..., None, None] * dP).reshape(F, -1, NV)} if jac else None
        out.append((0, r, G))
        # 5. contact velocity (frames f, f+1), labels of frame f
        if F > 1:
            c = w.vel * self.con[:-1]
            r = (c[..., None] * (ab[:-1] - ab[1:])).reshape(F - 1, -1)
            G = None
            if jac:
                G = {0: (c[..., None, None] * dab[:-1]).reshape(F - 1, -1, NV), 1: (-c[..., None, None] * dab[1:]).reshape(F - 1, -1, NV)}
            out.append((0, r, G))
        # 6. floor
        cf = w.floor * self.con
        r = cf * ((ab - self.pt) @ self.n)
        G = {0: cf[..., None] * t.einsum("c,fjcv->fjv", self.n, dab)} if jac else None
        out.append((0, r, G))
        # 7. smoothness of the unknowns themselves (root translation and Euler angles)
        if F > 1:
            we = w.smooth_vel * SMOOTH_EULER
            r = we * (x[:-1] - x[1:])
            G = None
            if jac:
                I = (we * t.eye(NV, **self.f64)).expand(F - 1, NV, NV)
                G = {0: I, 1: -I}
            out.append((0, r, G))
        return out

    def residual_vector(self, x, w):
        """The reference's f, same ordering (group by group, frame by frame)."""
        return self.t.cat([r.reshape(-1) for _, r, _ in self.residuals(x, w, jac=False)])

    def cost(self, x, w):
        return 0.5 * float(sum((r * r).sum() for _, r, _ in self.residuals(x, w, jac=False)))

    def dense_jacobian(self, x, w):
        """(terms, 87 F) -- tests only (small F)."""
        t = self.t
        rows = []
        for _, r, G in self.residuals(x, w, jac=True):
            Fp, nr_ = r.shape[0], r.reshape(r.shape[0], -1).shape[1]
            blk = t.zeros(Fp, nr_, self.F * NV, **self.f64)
            for d, g in G.items():
                for f in range(Fp):
                    blk[f, :, (f + d) * NV:(f + d + 1) * NV] = g[f]
            rows.append(blk.reshape(-1, self.F * NV))
        return t.cat(rows, 0)

    # ---- Gauss-Newton system: block-pentadiagonal H (diag, +1, +2 block bands) and gradient ----
    def normal_equations(self, x, w):
        t = self.t
        F = self.F
        H = [t.zeros(F, NV, NV, **self.f64), t.zeros(max(F - 1, 0), NV, NV, **self.f64), t.zeros(max(F - 2, 0), NV, NV, **self.f64)]
        g = t.zeros(F, NV, **self.f64)
        cost = 0.0
        for _, r, G in self.residuals(x, w, jac=True):
            Fp = r.shape[0]
            rr = r.reshape(Fp, -1)
            cost += 0.5 * float((rr * rr).sum())
            for d, gd in G.items():
                g[d:d + Fp] += t.einsum("frv,fr->fv", gd, rr)
                for e_, ge in G.items():
                    if e_ < d:
                        continue
                    H[e_ - d][d:d + Fp] += gd.transpose(1, 2) @ ge if e_ == d else ge.transpose(1, 2) @ gd   # block (f+e, f+d), lower band
        return cost, H, g


DENSE_MAX_UNKNOWNS = 24000      # 4.6 GB of fp64 at the limit (275 frames)


def _banded_cholesky_solve(t, H, g, lam, dense=None):
    """Solves (H + lam * diag(H)) s = g for the symmetric block-pentadiagonal H = (diag blocks, first and second lower block
    bands: H[1][f] = block (f+1, f), H[2][f] = block (f+2, f)).  One sweep of block Cholesky, F steps of 87 x 87 work."""
    D, B1, B2 = H
    F, n = D.shape[0], D.shape[1]
    Dd = D + lam * t.diag_embed(t.diagonal(D, dim1=1, dim2=2).clamp_min(1e-12))
    if dense is None:
        # on the GPU the sweep below is F dependent steps of a few tiny kernels each (launch bound); one dense fp64
        # Cholesky of the (87 F)^2 matrix is far faster there as long as it fits comfortably
        dense = D.is_cuda and F * n <= DENSE_MAX_UNKNOWNS
    if dense:
        A = t.zeros(F * n, F * n, dtype=D.dtype, device=D.device)
        A4 = A.view(F, n, F, n)
        i0 = t.arange(F, device=D.device)
        A4[i0, :, i0, :] = Dd
        if F > 1:
            A4[i0[1:], :, i0[:-1], :] = B1
        if F > 2:
            A4[i0[2:], :, i0[:-2], :] = B2
        L = t.linalg.cholesky(A)                       # reads the lower triangle only
        return t.cholesky_solve(g.reshape(-1, 1), L).reshape(F, n)
    L0, L1, L2 = [None] * F, [None] * F, [None] * F                               # L1[f] = L(f+1, f), L2[f] = L(f+2, f)
    for f in range(F):
        A = Dd[f].clone()
        if f >= 1:
            A -= L1[f - 1] @ L1[f - 1].T
        if f >= 2:
            A -= L2[f - 2] @ L2[f - 2].T
        L0[f] = t.linalg.cholesky(A)
        if f + 1 < F:
            A1 = B1[f].clone()
            if f >= 1:
                A1 -= L2[f - 1] @ L1[f - 1].T
            L1[f] = t.linalg.solve_triangular(L0[f], A1.T, upper=False).T
        if f + 2 < F:
            L2[f] = t.linalg.solve_triangular(L0[f], B2[f].T, upper=False).T
    # forward
    yv = [None] * F
    for f in range(F):
        b = g[f].clone()
        if f >= 1:
            b -= L1[f - 1] @ yv[f - 1]
        if f >= 2:
            b -= L2[f - 2] @ yv[f - 2]
        yv[f] = t.linalg.solve_triangular(L0[f], b[:, None], upper=False)[:, 0]
    # backward
    s = [None] * F
    for f in range(F - 1, -1, -1):
        b = yv[f].clone()
        if f + 1 < F:
            b -= L1[f].T @ s[f + 1]
        if f + 2 < F:
            b -= L2[f].T @ s[f + 2]
        s[f] = t.linalg.solve_triangular(L0[f].T, b[:, None], upper=True)[:, 0]
    return t.stack(s, 0)


def levenberg_marquardt(model: _Model, x0, w: StageWeights, max_nfev: int = 50, rtol: float = 1e-10, verbose: bool = False):
    """Minimises 0.5 |f(x)|^2 from x0 (F, 87).  Returns (x, cost, evaluations)."""
    t = model.t
    x = t.as_tensor(np.asarray(x0, dtype=np.float64).reshape(model.F, NV), **model.f64).clone()
    cost, H, g = model.normal_equations(x, w)
    nfev, lam = 1, 1e-3
    while nfev < max_nfev:
        try:
            step = -_banded_cholesky_solve(t, H, g, lam)
        except Exception:                 # not positive definite at this damping
            lam *= 10.0
            if lam > 1e12:
                break
            continue
        xn = x + step
        cn = model.cost(xn, w)
        nfev += 1
        # predicted decrease of the damped Gauss-Newton model: 0.5 step^T (lam D step - g)
        dg = t.stack([t.diagonal(H[0][f]) for f in range(model.F)], 0).clamp_min(1e-12)
        pred = 0.5 * float((step * (lam * dg * step - g)).sum())
        rho = (cost - cn) / pred if pred > 0 else -1.0
        if verbose:
            print("  nfev %3d  cost %.6e -> %.6e  lam %.1e  rho %.2f" % (nfev, cost, cn, lam, rho))
        if cn < cost:
            small = (cost - cn) <= rtol * cost
            x = xn
            cost, H, g = model.normal_equations(x, w)
            lam = max(lam * max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3), 1e-9) if rho > 0 else lam
            if small:
                break
        else:
            lam *= 4.0
            if lam > 1e12:
                break
    return x, cost, nfev


def huber_fit(X, y, epsilon: float, alpha: float = 1e-4, max_iter: int = 100, tol: float = 1e-5):
    """Linear fit with the Huber loss and a concomitant scale (the estimator `sklearn.linear_model.HuberRegressor`
    implements; optimize_trajectory.py:719-750 uses it with epsilon 1.5 / 2.2):
        min_{w, c, s > 0}  n s + sum_i H_eps((y_i - X_i w - c) / s) s + alpha |w|^2,
    L-BFGS-B from (0, 0, 1).  Returns (coef, intercept, scale, outlier mask)."""
    from scipy import optimize
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    n, k = X.shape

    def fun(p):
        wv, c, s = p[:k], p[k], p[k + 1]
        res = y - X @ wv - c
        a = np.abs(res)
        out = a > epsilon * s
        n_out = int(out.sum())
        loss = n * s + 2.0 * epsilon * a[out].sum() - s * n_out * epsilon ** 2 + (res[~out] ** 2).sum() / s + alpha * wv @ wv
        grad = np.zeros(k + 2)
        sg = np.sign(res[out])
        grad[:k] = -2.0 * epsilon * (X[out].T @ sg) - 2.0 / s * (X[~out].T @ res[~out]) + 2.0 * alpha * wv
        grad[k] = -2.0 * epsilon * sg.sum() - 2.0 / s * res[~out].sum()
        grad[k + 1] = n - n_out * epsilon ** 2 - (res[~out] ** 2).sum() / s ** 2
        return loss, grad

    p0 = np.zeros(k + 2)
    p0[k + 1] = 1.0
    bounds = [(-np.inf, np.inf)] * (k + 1) + [(np.finfo(np.float64).eps * 10, np.inf)]
    sol = optimize.minimize(fun, p0, method="L-BFGS-B", jac=True, bounds=bounds, options={"maxiter": max_iter, "gtol": tol})
    wv, c, s = sol.x[:k], sol.x[k], sol.x[k + 1]
    return wv, c, s, np.abs(y - X @ wv - c) > epsilon * s


def fit_floor(feet_pos, epsilon: float = 1.5):
    """optimize_trajectory.py:717-736: Huber fit of the height y over (x, z) of the contact points -> plane normal / point."""
    wv, c, s, out = huber_fit(feet_pos[:, [0, 2]], feet_pos[:, 1], epsilon)
    h = lambda xz: wv[0] * xz[0] + wv[1] * xz[1] + c
    v = np.array([[0.0, h((0.0, 0.0)), 0.0], [0.0, h((0.0, 100.0)), 100.0], [100.0, h((100.0, 0.0)), 0.0]])
    n = np.cross(v[2] - v[0], v[1] - v[2])
    return n / np.linalg.norm(n), v[0], out


def optimize_trajectory(poses2D, joint_conf_2d, poses3D, root_pos, joint_angles, parents, offsets, ppx, ppy, cam_focal, vel_constraints,
                        plane_normal=None, plane_point=None, device=None, ik_iterations: int = 200, max_nfev: int = 50, verbose: bool = False):
    """Driver with the reference's argument meaning (optimize_trajectory.py:522-834); the skeleton is given as (parents,
    offsets) of the 28-joint `combined` template.  Returns (anim, newPose3D, projPose2D, plane_normal, plane_point,
    vel_constraints, info)."""
    poses2D, poses3D, root_pos = np.asarray(poses2D, np.float64), np.asarray(poses3D, np.float64), np.asarray(root_pos, np.float64)
    vel = np.asarray(vel_constraints, dtype=np.float64).copy()
    F, J = poses3D.shape[:2]
    if poses2D.shape[1] != J:
        print("2D and 3D data must have the same number of joints!")
        return None
    given_floor = plane_normal is not None and plane_point is not None
    targets = poses3D[:, FORWARD] + root_pos[:, None, :]
    off = update_skeleton(parents, offsets, targets)
    j2n, pw, dw = make_weights(poses2D, np.asarray(joint_conf_2d, np.float64), (ppx, ppy), cam_focal)
    # IK initialisation from the given joint angles (axis-angle; the reference negates the axis), no IK on the spine
    aa = -np.asarray(joint_angles, np.float64)
    ang = np.linalg.norm(aa, axis=2)
    axis = aa / (ang + 1e-10)[..., None]
    K = np.zeros(aa.shape[:2] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 0], K[..., 1, 2], K[..., 2, 0], K[..., 2, 1] = -axis[..., 2], axis[..., 1], axis[..., 2], -axis[..., 0], -axis[..., 1], axis[..., 0]
    R0 = np.eye(3) + np.sin(ang)[..., None, None] * K + (1.0 - np.cos(ang))[..., None, None] * (K @ K)
    P0 = np.tile(off[None], (F, 1, 1))
    P0[:, 0] = root_pos
    names = ["joint_%d" % i for i in range(J)]
    anim = SkelAnim(names, np.asarray(parents), off, R0, P0)
    tm = {j: targets[:, j] for j in range(J) if j not in SPINE_IDX}
    anim = ik_solve(anim, tm, iterations=ik_iterations, smoothness=0.0, damping=7.0, translate=False, device=device)
    from .prepare import euler_zyx_from_matrix
    x = np.concatenate([anim.positions[:, 0], euler_zyx_from_matrix(anim.rotations).reshape(F, -1)], axis=1)
    zero = np.zeros(3)
    prob = Problem(np.asarray(parents), off, poses3D, root_pos, j2n, pw, dw, vel, zero if not given_floor else np.asarray(plane_normal, np.float64),
                   zero if not given_floor else np.asarray(plane_point, np.float64))
    info = {}
    # stage 1: no floor term
    m = _Model(prob, device)
    xs, c1, n1 = levenberg_marquardt(m, x, StageWeights(floor=0.0), max_nfev, verbose=verbose)
    info["stage1"] = dict(cost=c1, nfev=n1)
    x = xs.cpu().numpy()
    # floor fit on the contact feet, contact pruning
    gp = _global_positions(parents, off, x)
    feet_lab = np.array([FORWARD[k] for k in FEET_IDX])
    sel = vel[:, feet_lab] == 1
    feet_pos = gp[:, FEET_IDX][sel]
    if not given_floor:
        plane_normal, plane_point, _ = fit_floor(feet_pos, 1.5)
        _, _, _, outl = huber_fit(feet_pos[:, [0, 2]], feet_pos[:, 1], 2.2)
        fv = vel[:, feet_lab]
        fv[sel] = np.where(outl, 0.0, 1.0)          # row-major order of the selection = the reference's frame / foot loop
        vel[:, feet_lab] = fv
    # stage 2: feet on the floor
    prob.contacts, prob.floor_normal, prob.floor_point = vel, np.asarray(plane_normal, np.float64), np.asarray(plane_point, np.float64)
    m = _Model(prob, device)
    xs, c2, n2 = levenberg_marquardt(m, x, StageWeights(floor=10.0), max_nfev, verbose=verbose)
    info["stage2"] = dict(cost=c2, nfev=n2)
    x = xs.cpu().numpy()
    info["x"] = x
    gp = _global_positions(parents, off, x)
    new3d = gp[:, BACKWARD]
    proj = np.stack([cam_focal[0] * new3d[..., 0] / new3d[..., 2] + ppx, cam_focal[1] * new3d[..., 1] / new3d[..., 2] + ppy], -1)
    Pl = np.tile(off[None], (F, 1, 1))
    Pl[:, 0] = x[:, :3]
    anim = SkelAnim(names, np.asarray(parents), off, rot_zyx(x[:, 3:].reshape(F, J, 3)), Pl)
    return anim, new3d, proj, np.asarray(plane_normal), np.asarray(plane_point), vel, info


def _global_positions(parents, off, x):
    from .prepare import forward_kinematics
    F = x.shape[0]
    T = np.tile(np.asarray(off)[None], (F, 1, 1))
    T[:, 0] = x[:, :3]
    return forward_kinematics(np.asarray(parents), rot_zyx(x[:, 3:].reshape(F, NJ, 3)), T)[0]


# ---------------------------------------------------------------------------------------------------------------------
# File-level driver (src/optimize/kinematic_optimizer.py:30-224 optimize_2d_3d) and the Monocular-Total-Capture reader
# ---------------------------------------------------------------------------------------------------------------------
SMPL_SPINE_JOINTS = [3, 6, 9]                   # totalcap_utils.py:18
# combined skeleton joint -> SMPL joint (-1: none), character_info_utils.py:222-251
COMBINED_TO_SMPL = [0, 1, 4, 7, -1, -1, 10, 2, 5, 8, -1, -1, 11, 3, 6, 9, 12, 15, -1, -1, -1, -1, 16, 18, 20, 17, 19, 21]
MTC_FOCAL = (2000.0, 2000.0)                    # kinematic_optimizer.py:22-28
MTC_SIZE = (1920, 1080)


def load_totalcap_results(path: str) -> dict:
    """totalcap_utils.py:33-79: `tracked_results.json` of Monocular Total Capture -> root translation (F,3), BODY_25 joints
    (F,25,3), SMPL joints (F,Js,3) and SMPL joint angles (F,Js,3 axis-angle)."""
    import json
    with open(path) as f:
        frames = json.load(f)["totalcapResults"]
    xyz = lambda d: [d["x"], d["y"], d["z"]]
    return dict(root_trans=np.array([xyz(fr["trans"]) for fr in frames], dtype=np.float64),
                joint3d=np.array([[xyz(j["pos"]) for j in fr["joints"]] for fr in frames], dtype=np.float64),
                smpl_joint3d=np.array([[xyz(j["pos"]) for j in fr["SMPLJoints"]] for fr in frames], dtype=np.float64),
                smpl_joint_angles=np.array([[xyz(j["rot"]) for j in fr["SMPLJoints"]] for fr in frames], dtype=np.float64))


def combined_inputs(tc: dict):
    """kinematic_optimizer.py:64-73: root-relative BODY_25 joints + the three SMPL spine joints, root translation moved into
    `root_pos`, initial joint angles of the combined skeleton from the SMPL angles."""
    root = tc["root_trans"] + tc["joint3d"][:, ROOT_IDX]
    body = tc["joint3d"] - tc["joint3d"][:, ROOT_IDX:ROOT_IDX + 1]
    smpl = tc["smpl_joint3d"] - tc["smpl_joint3d"][:, 0:1]
    poses3D = np.concatenate([body, smpl[:, SMPL_SPINE_JOINTS]], axis=1)
    ang = np.zeros((root.shape[0], NJ, 3))
    for j, s in enumerate(COMBINED_TO_SMPL):
        if s >= 0:
            ang[:, j] = tc["smpl_joint_angles"][:, s]
    return poses3D, root, ang


def contacts_to_constraints(foot_contacts):
    """(F,4) labels [L heel, L toe, R heel, R toe] -> (F,28) per-joint labels in body-25 order (kinematic_optimizer.py:106-116)."""
    fc = np.asarray(foot_contacts)
    vel = np.zeros((fc.shape[0], NJ))
    vel[:, 19] = vel[:, 20] = fc[:, 1]
    vel[:, 21] = fc[:, 0]
    vel[:, 22] = vel[:, 23] = fc[:, 3]
    vel[:, 24] = fc[:, 2]
    return vel


def constraints_to_contacts(vel):
    """Refined per-joint labels -> (F,4) int [L heel, L toe, R heel, R toe] (kinematic_optimizer.py:183-204)."""
    v = np.asarray(vel)
    return np.stack([v[:, 21], np.logical_or(v[:, 19], v[:, 20]), v[:, 24], np.logical_or(v[:, 22], v[:, 23])], axis=1).astype(int)


def optimize_2d_3d(input_path: str, skel_path: str, output_path: str, min_idx: int = 0, max_idx: int = 100, use_gt_floor: bool = False,
                   device=None, frametime: float = 1.0 / 24.0):
    """kinematic_optimizer.optimize_2d_3d: reads `<dir>/openpose_result/*.json`, `<dir>/tracked_results.json`,
    `<dir>/foot_contacts.npy` next to `input_path`; writes `foot_contacts.npy` (refined, int), `floor_out.txt` and
    `final_test.bvh` into `output_path`."""
    import os
    from . import contact
    from .prepare import load_bvh
    from .results import save_bvh
    os.makedirs(output_path, exist_ok=True)
    d = os.path.dirname(input_path)
    op_dir, tc_path, fc_path = os.path.join(d, "openpose_result"), os.path.join(d, "tracked_results.json"), os.path.join(d, "foot_contacts.npy")
    if not os.path.isdir(op_dir):
        print("Could not find openpose results in " + op_dir + "!")
        return None
    if not os.path.isfile(tc_path):
        print("Could not find total capture results!")
        return None
    if not os.path.isfile(fc_path):
        print("Could not find foot contact labels!")
        return None
    kp = contact.load_keypoint_dir(op_dir)
    poses3D, root_pos, ang = combined_inputs(load_totalcap_results(tc_path))
    sl = slice(min_idx, max_idx)
    n = len(range(*sl.indices(kp.shape[0])))
    poses2D = np.concatenate([kp[sl, :, :2], np.zeros((n, 3, 2))], axis=1)
    conf = np.concatenate([kp[sl, :, 2], np.zeros((n, 3))], axis=1)
    fc = np.load(fc_path)
    vel = contacts_to_constraints(fc[sl])
    normal = point = None
    if use_gt_floor:
        with open(os.path.join(d, "floor_gt.txt")) as f:
            normal = np.array([float(v) for v in f.readline().split()])
            point = np.array([float(v) for v in f.readline().split()]) * 100.0
    b = load_bvh(skel_path)
    res = optimize_trajectory(poses2D, conf, poses3D[sl], root_pos[sl], ang[sl], b.parents, b.offsets, MTC_SIZE[0] / 2, MTC_SIZE[1] / 2,
                              np.array(MTC_FOCAL), vel, plane_normal=normal, plane_point=point, device=device)
    anim, new3d, proj, pn, pp, newvel, info = res
    anim.names = list(b.names)
    np.save(os.path.join(output_path, "foot_contacts"), constraints_to_contacts(newvel))
    with open(os.path.join(output_path, "floor_out.txt"), "w") as f:
        f.write("%s %s %s\n%s %s %s" % tuple(str(float(v)) for v in list(pn) + list(pp)))
    save_bvh(os.path.join(output_path, "final_test.bvh"), anim, b.names, frametime)
    print("Finished kinematic optimization!")
    return res
