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

from .results import SkelAnim, descendants_mask, ik_solve_batch, rot_zyx

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
    """Residuals and the block structure of their Jacobian over the concatenated frames of K >= 1 clips of the same
    skeleton, batched over the frames (torch, fp64).  Offsets and floor are per clip, and the rows that would couple the
    last frames of one clip with the next clip (velocity, acceleration, contact velocity, Euler smoothness) are dropped,
    so H has no block coupling two clips.  `probs`: a list of `Problem`s, or one `Problem` for a single clip.  Cost and
    normal equations return per-clip costs (numpy, K)."""

    def __init__(self, probs, device=None):
        import torch
        if isinstance(probs, Problem):
            probs = [probs]
        if not probs:
            raise ValueError("no clips")
        parents = np.asarray(probs[0].parents)
        if any(not np.array_equal(np.asarray(p.parents), parents) for p in probs):
            raise ValueError("all clips of a batch must use the same skeleton hierarchy")
        self.lens = np.array([p.poses3D.shape[0] for p in probs], dtype=np.int64)
        if (self.lens < 1).any():
            raise ValueError("every clip needs at least one frame")
        self.K = len(probs)
        self.seg = np.concatenate([[0], np.cumsum(self.lens)]).astype(np.int64)
        self.spans = [(int(a), int(b)) for a, b in zip(self.seg[:-1], self.seg[1:])]
        self.t = torch
        self.dev = torch.device(device) if device is not None else torch.device("cpu")
        f64 = dict(dtype=torch.float64, device=self.dev)
        self.f64 = f64
        self.F = F = int(self.seg[-1])
        self.parents = [int(v) for v in parents]
        self.back = torch.as_tensor(BACKWARD, device=self.dev)
        self.desc = torch.as_tensor(descendants_mask(self.parents).astype(np.float64), **f64)   # [m, k]: k strict descendant of m
        self.par_idx = torch.as_tensor([max(q, 0) for q in self.parents], device=self.dev)
        self.root_mask = torch.as_tensor([q < 0 for q in self.parents], device=self.dev)
        as_t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), **f64)
        cat = lambda a: as_t(np.concatenate([np.asarray(getattr(p, a), np.float64) for p in probs], 0))
        self.poses3D, self.root_trans, self.j2n = cat("poses3D"), cat("root_trans"), cat("joints2d")
        self.pw, self.dw, self.con = cat("proj_w"), cat("data_w"), cat("contacts")
        self.sw = as_t(SMOOTH_WEIGHTS)[:, None] * as_t(SMOOTH_VEL)[None, :]            # (28, 3)
        self.is_root = torch.zeros(NJ, **f64)
        self.is_root[ROOT_IDX] = 1.0
        # each clip's skeleton offsets and floor, and per frame (the clip of every frame)
        per_clip = lambda a: as_t(np.stack([np.asarray(getattr(p, a), np.float64) for p in probs]))
        self.off_k, self.n_k, self.pt_k = per_clip("offsets"), per_clip("floor_normal"), per_clip("floor_point")
        self.clip = torch.as_tensor(np.repeat(np.arange(self.K), self.lens), device=self.dev)
        self.off, self.n, self.pt = self.off_k[self.clip], self.n_k[self.clip], self.pt_k[self.clip]
        # rows of a group that couples frames f .. f+k: those whose last frame lies in the clip of f
        end = np.repeat(self.seg[1:], self.lens)
        self.keep = {k: torch.as_tensor(np.nonzero(np.arange(max(F - k, 0)) + k < end[:max(F - k, 0)])[0], device=self.dev)
                     for k in (1, 2)}
        self.all = torch.arange(F, device=self.dev)
        # On the CPU the products with a clip's offsets and floor are taken clip by clip, as matrix-vector products: a
        # per-frame batched product rounds differently in the last bit, and Levenberg-Marquardt amplifies that along
        # weakly determined directions.  So a clip's result on the CPU does not depend on the other clips of its batch.
        # On a GPU one batched product serves all clips.
        self.by_clip = self.dev.type == "cpu"

    def _bone(self, gRq, j):
        """Offset of joint j rotated by its parent's global rotation."""
        if self.by_clip:
            return self.t.cat([gRq[a:b] @ self.off_k[k, j] for k, (a, b) in enumerate(self.spans)], 0)
        return (gRq @ self.off[:, j, :, None])[..., 0]

    def _rows(self, span, r, G):
        """A residual group whose row of base frame f couples frames f .. f+span -> (base frames, r, G) without the rows
        that would couple two clips."""
        idx = self.keep[span]
        return idx, r[idx], ({d: g[idx] for d, g in G.items()} if G is not None else None)

    def _floor(self, cf, ab, dab, jac):
        t = self.t
        if self.by_clip:
            r = t.cat([cf[a:b] * ((ab[a:b] - self.pt_k[k]) @ self.n_k[k]) for k, (a, b) in enumerate(self.spans)], 0)
            G = {0: t.cat([cf[a:b, :, None] * t.einsum("c,fjcv->fjv", self.n_k[k], dab[a:b]) for k, (a, b) in enumerate(self.spans)], 0)} if jac else None
            return r, G
        r = cf * t.einsum("fjc,fc->fj", ab - self.pt[:, None, :], self.n)
        G = {0: cf[..., None] * t.einsum("fc,fjcv->fjv", self.n, dab)} if jac else None
        return r, G

    def _base(self, base, Fp):
        return self.all[:Fp] if isinstance(base, int) else base

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
                gP[j] = gP[q] + self._bone(gR[q], j)
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
        """List of (base frames, r (F', rows), blocks {d: G (F', rows, 87)} = dr/dx_{f+d}); base frames 0: 0 .. F'-1."""
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
            out.append(self._rows(1, r, G))
        # 3. acceleration smoothness (frames f, f+1, f+2)
        if F > 2:
            r = (w.smooth_acc * (y[2:] - 2.0 * y[1:-1] + y[:-2])).reshape(F - 2, -1)
            G = None
            if jac:
                G = {0: (w.smooth_acc * dP[:-2]).reshape(F - 2, -1, NV), 1: (-2.0 * w.smooth_acc * dP[1:-1]).reshape(F - 2, -1, NV),
                     2: (w.smooth_acc * dP[2:]).reshape(F - 2, -1, NV)}
            out.append(self._rows(2, r, G))
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
            out.append(self._rows(1, r, G))
        # 6. floor
        r, G = self._floor(w.floor * self.con, ab, dab, jac)
        out.append((0, r, G))
        # 7. smoothness of the unknowns themselves (root translation and Euler angles)
        if F > 1:
            we = w.smooth_vel * SMOOTH_EULER
            r = we * (x[:-1] - x[1:])
            G = None
            if jac:
                I = (we * t.eye(NV, **self.f64)).expand(F - 1, NV, NV)
                G = {0: I, 1: -I}
            out.append(self._rows(1, r, G))
        return out

    def residual_vector(self, x, w):
        """The reference's f, same ordering (group by group, frame by frame)."""
        return self.t.cat([r.reshape(-1) for _, r, _ in self.residuals(x, w, jac=False)])

    def per_clip(self, v):
        """Segment sums of a per-frame numpy vector."""
        return np.add.reduceat(np.asarray(v, dtype=np.float64), self.seg[:-1])

    def _costs(self, groups, each):
        """0.5 * sum of squares per clip of the residual groups [(base, r)]; `each`: halve every group's sum (as the
        normal equations accumulate it) instead of the total (as `cost`).  By clip: one reduction per clip and group.
        Otherwise per frame on the device (a row counts for its first frame), then per clip on the host."""
        if self.by_clip:
            c = np.zeros(self.K)
            for base, r in groups:
                rr = r.reshape(r.shape[0], -1)
                cuts = self.seg if isinstance(base, int) else np.searchsorted(base.cpu().numpy(), self.seg)
                for k in range(self.K):
                    v = rr[cuts[k]:cuts[k + 1]]
                    if v.shape[0]:
                        c[k] += 0.5 * float((v * v).sum()) if each else float((v * v).sum())
            return c if each else 0.5 * c
        return 0.5 * self.per_clip(self.frame_costs(groups).cpu().numpy())

    def frame_costs(self, groups):
        cf = self.t.zeros(self.F, **self.f64)
        for base, r in groups:
            rr = r.reshape(r.shape[0], -1)
            cf.index_add_(0, self._base(base, rr.shape[0]), (rr * rr).sum(1))
        return cf

    def cost(self, x, w):
        return self._costs([(b, r) for b, r, _ in self.residuals(x, w, jac=False)], each=False)

    def trial(self, xn, w, step, lam, H, g, status):
        """(cost at xn, predicted decrease 0.5 step^T (lam diag(H) step - g), solve status) per clip, numpy; one device to
        host copy."""
        t = self.t
        dg = t.diagonal(H[0], dim1=1, dim2=2).clamp_min(1e-12)
        if self.by_clip:
            pred = np.array([0.5 * float((step[a:b] * (float(lam[k]) * dg[a:b] * step[a:b] - g[a:b])).sum()) for k, (a, b) in enumerate(self.spans)])
            return self.cost(xn, w), pred, status.cpu().numpy()
        lamf = t.as_tensor(np.repeat(lam, self.lens), **self.f64)
        pf = (step * (lamf[:, None] * dg * step - g)).sum(1)
        cf = self.frame_costs([(b, r) for b, r, _ in self.residuals(xn, w, jac=False)])
        host = t.cat([cf, pf, status.to(t.float64)]).cpu().numpy()
        F = self.F
        return 0.5 * self.per_clip(host[:F]), 0.5 * self.per_clip(host[F:2 * F]), host[2 * F:]

    def dense_jacobian(self, x, w):
        """(terms, 87 F) -- tests only (small F)."""
        t = self.t
        rows = []
        for base, r, G in self.residuals(x, w, jac=True):
            Fp, nr_ = r.shape[0], r.reshape(r.shape[0], -1).shape[1]
            bf = self._base(base, Fp).tolist()
            blk = t.zeros(Fp, nr_, self.F * NV, **self.f64)
            for d, g in G.items():
                for i, f in enumerate(bf):
                    blk[i, :, (f + d) * NV:(f + d + 1) * NV] = g[i]
            rows.append(blk.reshape(-1, self.F * NV))
        return t.cat(rows, 0)

    # ---- Gauss-Newton system: block-pentadiagonal H (diag, +1, +2 block bands) and gradient ----
    def normal_equations(self, x, w):
        t = self.t
        F = self.F
        H = [t.zeros(F, NV, NV, **self.f64), t.zeros(max(F - 1, 0), NV, NV, **self.f64), t.zeros(max(F - 2, 0), NV, NV, **self.f64)]
        g = t.zeros(F, NV, **self.f64)
        groups = []
        for base, r, G in self.residuals(x, w, jac=True):
            Fp = r.shape[0]
            rr = r.reshape(Fp, -1)
            bf = self._base(base, Fp)
            groups.append((base, r))
            for d, gd in G.items():
                g.index_add_(0, bf + d, t.einsum("frv,fr->fv", gd, rr))
                for e_, ge in G.items():
                    if e_ < d:
                        continue
                    H[e_ - d].index_add_(0, bf + d, gd.transpose(1, 2) @ ge if e_ == d else ge.transpose(1, 2) @ gd)   # block (f+e, f+d), lower band
        return self._costs(groups, each=True), H, g


def _banded_cholesky_solve(t, H, g, lam):
    """Solves (H + lam * diag(H)) s = g for the symmetric block-pentadiagonal H = (diag blocks, first and second lower block
    bands: H[1][f] = block (f+1, f), H[2][f] = block (f+2, f)).  One sweep of block Cholesky, F steps of 87 x 87 work."""
    D, B1, B2 = H
    F = D.shape[0]
    Dd = D + lam * t.diag_embed(t.diagonal(D, dim1=1, dim2=2).clamp_min(1e-12))
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


class _KinSolver:
    """The damped block-banded solves of all live clips of a `_Model` in one step: one `chd_kin_solve` launch on a
    CUDA device (libchd is required there), `_banded_cholesky_solve` per clip segment on the CPU."""

    def __init__(self, model: _Model):
        t = model.t
        self.m = model
        self.cuda = model.dev.type == "cuda"
        self.s = t.zeros(model.F, NV, **model.f64)
        self.status = t.zeros(model.K, dtype=t.int32, device=model.dev)
        if self.cuda:
            from .phys import load_lib
            self.L = load_lib()
            nb = self.L.chd_kin_work_bytes(int(model.F))
            self.work = t.empty(max(nb // 8, 1), **model.f64)
            self.seg = t.as_tensor(model.seg, dtype=t.int32, device=model.dev)

    def __call__(self, H, g, lam, live):
        """Solves (H + lam_k diag H) s = g for the clips `live`.  Returns (s, status) on the model's device; status is 0
        for a solved clip, nonzero for a failed factorisation or a clip not in `live`, and s is only defined where 0."""
        t, m = self.m.t, self.m
        self.status.fill_(-2)
        if not self.cuda:
            st = np.full(m.K, -2, dtype=np.int32)
            for k in live:
                a, b = int(m.seg[k]), int(m.seg[k + 1])
                try:
                    self.s[a:b] = _banded_cholesky_solve(t, (H[0][a:b], H[1][a:b - 1], H[2][a:b - 2]), g[a:b], float(lam[k]))
                    st[k] = 0
                except Exception:         # not positive definite at this damping
                    st[k] = 1
            self.status.copy_(t.as_tensor(st))
            return self.s, self.status
        ptr = lambda a: a.data_ptr() if a.numel() else None
        lam_d = t.as_tensor(np.asarray(lam, np.float64), **m.f64)
        sel = t.as_tensor(np.asarray(live, np.int32), device=m.dev)
        D, B1, B2, gc = (a.contiguous() for a in (H[0], H[1], H[2], g))
        with t.cuda.device(m.dev):
            rc = self.L.chd_kin_solve(ptr(D), ptr(B1), ptr(B2), ptr(gc), self.seg.data_ptr(), lam_d.data_ptr(), sel.data_ptr(),
                                      len(live), m.K, m.F, self.work.data_ptr(), self.s.data_ptr(), self.status.data_ptr(),
                                      t.cuda.current_stream(m.dev).cuda_stream)
        if rc != 0:
            raise RuntimeError("chd_kin_solve failed with code %d" % rc)
        return self.s, self.status


def levenberg_marquardt(model: _Model, x0s, w: StageWeights, max_nfev: int = 50, rtol: float = 1e-10, verbose: bool = False):
    """Minimises 0.5 |f_k(x_k)|^2 for every clip k of `model` from x0s (one (F_k, 87) array per clip).  Each clip keeps its
    own state (damping, cost, evaluation count); a round solves all live clips in one step and synchronises the host once
    for the accept decisions.  Returns (xs, costs, nfevs), lists."""
    t = model.t
    K, seg = model.K, model.seg
    x = t.as_tensor(np.concatenate([np.asarray(a, np.float64).reshape(-1, NV) for a in x0s], 0), **model.f64).clone()
    if x.shape[0] != model.F:
        raise ValueError("x0s do not match the model's frames")
    solve = _KinSolver(model)
    cost, H, g = model.normal_equations(x, w)
    nfev = np.ones(K, dtype=np.int64)
    lam = np.full(K, 1e-3)
    done = nfev >= max_nfev
    rnd = 0
    while not done.all():
        live = np.nonzero(~done)[0]
        s, status = solve(H, g, lam, live)
        okf = (status == 0)[model.clip]                                           # frames of the clips that got a step
        step = -t.where(okf[:, None], s, t.zeros_like(s))
        xn = x + step
        cn, pred, st = model.trial(xn, w, step, lam, H, g, status)
        acc = np.zeros(K, dtype=bool)
        for k in live:
            if st[k] != 0:                # not positive definite at this damping
                lam[k] *= 10.0
                done[k] = lam[k] > 1e12
                continue
            nfev[k] += 1
            rho = (cost[k] - cn[k]) / pred[k] if pred[k] > 0 else -1.0
            if cn[k] < cost[k]:
                acc[k] = True
                done[k] = (cost[k] - cn[k]) <= rtol * cost[k]
                lam[k] = max(lam[k] * max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3), 1e-9) if rho > 0 else lam[k]
            else:
                lam[k] *= 4.0
                done[k] = lam[k] > 1e12
            done[k] = done[k] or nfev[k] >= max_nfev
        if verbose:
            rnd += 1
            print("  round %3d  live %d  accepted %d  cost %.6e" % (rnd, len(live), int(acc.sum()), float(np.sum(cost))))
        if acc.any():
            x = t.where(t.as_tensor(acc, device=model.dev)[model.clip][:, None], xn, x)
            cnew, H, g = model.normal_equations(x, w)
            cost = np.where(acc, cnew, cost)
    xs = [x[seg[k]:seg[k + 1]] for k in range(K)]
    return xs, [float(c) for c in cost], [int(n) for n in nfev]


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
    """One clip with the reference's signature (optimize_trajectory.py:522-834), run as a batch of one by
    `optimize_trajectory_batch`.  Returns (anim, newPose3D, projPose2D, plane_normal, plane_point, vel_constraints, info),
    or None after the reference's message when the 2D and 3D data have different numbers of joints."""
    if np.shape(poses2D)[1] != np.shape(poses3D)[1]:
        print("2D and 3D data must have the same number of joints!")
        return None
    return optimize_trajectory_batch([poses2D], [joint_conf_2d], [poses3D], [root_pos], [joint_angles], [parents], [offsets], [ppx], [ppy],
                                     [cam_focal], [vel_constraints], plane_normal=[plane_normal], plane_point=[plane_point], device=device,
                                     ik_iterations=ik_iterations, max_nfev=max_nfev, verbose=verbose)[0]


def _global_positions(parents, off, x):
    from .prepare import forward_kinematics
    F = x.shape[0]
    T = np.tile(np.asarray(off)[None], (F, 1, 1))
    T[:, 0] = x[:, :3]
    return forward_kinematics(np.asarray(parents), rot_zyx(x[:, 3:].reshape(F, NJ, 3)), T)[0]


def optimize_trajectory_batch(poses2D, joint_conf_2d, poses3D, root_pos, joint_angles, parents, offsets, ppx, ppy, cam_focal, vel_constraints,
                              plane_normal=None, plane_point=None, device=None, ik_iterations: int = 200, max_nfev: int = 50, verbose: bool = False):
    """Driver with the reference's argument meaning (optimize_trajectory.py:522-834) for K clips at once; the skeleton is
    given as (parents, offsets) of the 28-joint `combined` template.  Every per-clip argument is a list with one entry per
    clip (plane_normal / plane_point: None, or a list whose None entries mean "fit the floor" for that clip).  The IK
    initialisation is one call over all frames, each Levenberg-Marquardt stage runs all clips together; the skeleton fit,
    the floor fit and the contact pruning stay per clip.  Returns one (anim, newPose3D, projPose2D, plane_normal,
    plane_point, vel_constraints, info) per clip."""
    from .prepare import euler_zyx_from_matrix
    K = len(poses3D)
    pn_in = plane_normal if plane_normal is not None else [None] * K
    pp_in = plane_point if plane_point is not None else [None] * K
    clips = []
    for k in range(K):
        p2, p3, rp = np.asarray(poses2D[k], np.float64), np.asarray(poses3D[k], np.float64), np.asarray(root_pos[k], np.float64)
        F, J = p3.shape[:2]
        if p2.shape[1] != J:
            raise ValueError("clip %d: 2D and 3D data must have the same number of joints" % k)
        targets = p3[:, FORWARD] + rp[:, None, :]
        off = update_skeleton(parents[k], offsets[k], targets)
        j2n, pw, dw = make_weights(p2, np.asarray(joint_conf_2d[k], np.float64), (ppx[k], ppy[k]), cam_focal[k])
        given = pn_in[k] is not None and pp_in[k] is not None
        clips.append(dict(F=F, p3=p3, rp=rp, targets=targets, off=off, j2n=j2n, pw=pw, dw=dw, given=given,
                          vel=np.asarray(vel_constraints[k], dtype=np.float64).copy(), parents=np.asarray(parents[k]),
                          pn=np.asarray(pn_in[k], np.float64) if given else None, pp=np.asarray(pp_in[k], np.float64) if given else None))
    J = clips[0]["p3"].shape[1]
    # IK initialisation from the given joint angles (axis-angle; the reference negates the axis), no IK on the spine; every
    # frame of every clip in one call (smoothness 0: the frames are independent)
    R0, P0 = [], []
    for k, c in enumerate(clips):
        aa = -np.asarray(joint_angles[k], np.float64)
        ang = np.linalg.norm(aa, axis=2)
        axis = aa / (ang + 1e-10)[..., None]
        Km = np.zeros(aa.shape[:2] + (3, 3))
        Km[..., 0, 1], Km[..., 0, 2], Km[..., 1, 0], Km[..., 1, 2], Km[..., 2, 0], Km[..., 2, 1] = -axis[..., 2], axis[..., 1], axis[..., 2], -axis[..., 0], -axis[..., 1], axis[..., 0]
        R0.append(np.eye(3) + np.sin(ang)[..., None, None] * Km + (1.0 - np.cos(ang))[..., None, None] * (Km @ Km))
        P = np.tile(c["off"][None], (c["F"], 1, 1))
        P[:, 0] = c["rp"]
        P0.append(P)
    names = ["joint_%d" % i for i in range(J)]
    anim = SkelAnim(names, clips[0]["parents"], clips[0]["off"], np.concatenate(R0), np.concatenate(P0))
    tm = {j: np.concatenate([c["targets"][:, j] for c in clips]) for j in range(J) if j not in SPINE_IDX}
    anim = ik_solve_batch([anim], [tm], iterations=ik_iterations, smoothness=0.0, damping=7.0, translate=False, device=device)[0]
    xall = np.concatenate([anim.positions[:, 0], euler_zyx_from_matrix(anim.rotations).reshape(anim.rotations.shape[0], -1)], axis=1)
    seg = np.concatenate([[0], np.cumsum([c["F"] for c in clips])])
    xs = [xall[seg[k]:seg[k + 1]] for k in range(K)]
    zero = np.zeros(3)
    probs = [Problem(c["parents"], c["off"], c["p3"], c["rp"], c["j2n"], c["pw"], c["dw"], c["vel"], c["pn"] if c["given"] else zero,
                     c["pp"] if c["given"] else zero) for c in clips]
    # stage 1: no floor term
    out1, c1, n1 = levenberg_marquardt(_Model(probs, device), xs, StageWeights(floor=0.0), max_nfev, verbose=verbose)
    xs = [v.cpu().numpy() for v in out1]
    # floor fit on the contact feet, contact pruning (per clip)
    feet_lab = np.array([FORWARD[k] for k in FEET_IDX])
    for k, c in enumerate(clips):
        vel = c["vel"]
        gp = _global_positions(c["parents"], c["off"], xs[k])
        sel = vel[:, feet_lab] == 1
        feet_pos = gp[:, FEET_IDX][sel]
        if not c["given"]:
            c["pn"], c["pp"], _ = fit_floor(feet_pos, 1.5)
            _, _, _, outl = huber_fit(feet_pos[:, [0, 2]], feet_pos[:, 1], 2.2)
            fv = vel[:, feet_lab]
            fv[sel] = np.where(outl, 0.0, 1.0)          # row-major order of the selection = the reference's frame / foot loop
            vel[:, feet_lab] = fv
        probs[k].contacts, probs[k].floor_normal, probs[k].floor_point = vel, np.asarray(c["pn"], np.float64), np.asarray(c["pp"], np.float64)
    # stage 2: feet on the floor
    out2, c2, n2 = levenberg_marquardt(_Model(probs, device), xs, StageWeights(floor=10.0), max_nfev, verbose=verbose)
    res = []
    for k, c in enumerate(clips):
        x = out2[k].cpu().numpy()
        F, off = c["F"], c["off"]
        info = dict(stage1=dict(cost=c1[k], nfev=n1[k]), stage2=dict(cost=c2[k], nfev=n2[k]), x=x)
        gp = _global_positions(c["parents"], off, x)
        new3d = gp[:, BACKWARD]
        fo = cam_focal[k]
        proj = np.stack([fo[0] * new3d[..., 0] / new3d[..., 2] + ppx[k], fo[1] * new3d[..., 1] / new3d[..., 2] + ppy[k]], -1)
        Pl = np.tile(off[None], (F, 1, 1))
        Pl[:, 0] = x[:, :3]
        a = SkelAnim(names, c["parents"], off, rot_zyx(x[:, 3:].reshape(F, J, 3)), Pl)
        res.append((a, new3d, proj, np.asarray(c["pn"]), np.asarray(c["pp"]), c["vel"], info))
    return res


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
    `final_test.bvh` into `output_path`.  Returns `optimize_trajectory`'s tuple, or None after a message naming the missing
    input; a batch of one of `optimize_2d_3d_batch`."""
    return optimize_2d_3d_batch([(input_path, skel_path, output_path, min_idx, max_idx, use_gt_floor)], device, frametime)[0]


def optimize_2d_3d_batch(jobs, device=None, frametime: float = 1.0 / 24.0):
    """`optimize_2d_3d` for several videos with one `optimize_trajectory_batch` call.  `jobs`: list of (input_path,
    skel_path, output_path, min_idx, max_idx, use_gt_floor); every video gets the three files `optimize_2d_3d` writes.
    Returns one result per job (None for a video whose inputs are missing, after a message naming the missing input)."""
    import os
    from . import contact
    from .prepare import load_bvh
    from .results import save_bvh
    loaded = []
    for input_path, skel_path, output_path, min_idx, max_idx, use_gt_floor in jobs:
        os.makedirs(output_path, exist_ok=True)
        d = os.path.dirname(input_path)
        op_dir, tc_path, fc_path = os.path.join(d, "openpose_result"), os.path.join(d, "tracked_results.json"), os.path.join(d, "foot_contacts.npy")
        missing = [m for ok, m in ((os.path.isdir(op_dir), "Could not find openpose results in " + op_dir + "!"),
                                   (os.path.isfile(tc_path), "Could not find total capture results!"),
                                   (os.path.isfile(fc_path), "Could not find foot contact labels!")) if not ok]
        if missing:
            print(missing[0])
            loaded.append(None)
            continue
        kp = contact.load_keypoint_dir(op_dir)
        poses3D, root_pos, ang = combined_inputs(load_totalcap_results(tc_path))
        sl = slice(min_idx, max_idx)
        n = len(range(*sl.indices(kp.shape[0])))
        normal = point = None
        if use_gt_floor:
            with open(os.path.join(d, "floor_gt.txt")) as f:
                normal = np.array([float(v) for v in f.readline().split()])
                point = np.array([float(v) for v in f.readline().split()]) * 100.0
        loaded.append(dict(out=output_path, bvh=load_bvh(skel_path), normal=normal, point=point,
                           poses2D=np.concatenate([kp[sl, :, :2], np.zeros((n, 3, 2))], axis=1),
                           conf=np.concatenate([kp[sl, :, 2], np.zeros((n, 3))], axis=1), poses3D=poses3D[sl], root_pos=root_pos[sl],
                           ang=ang[sl], vel=contacts_to_constraints(np.load(fc_path)[sl])))
    vids = [v for v in loaded if v is not None]
    results = []
    if vids:
        col = lambda key: [v[key] for v in vids]
        K = len(vids)
        results = optimize_trajectory_batch(col("poses2D"), col("conf"), col("poses3D"), col("root_pos"), col("ang"), [v["bvh"].parents for v in vids],
                                            [v["bvh"].offsets for v in vids], [MTC_SIZE[0] / 2] * K, [MTC_SIZE[1] / 2] * K, [np.array(MTC_FOCAL)] * K,
                                            col("vel"), plane_normal=col("normal"), plane_point=col("point"), device=device)
    it = iter(results)
    out = []
    for v in loaded:
        if v is None:
            out.append(None)
            continue
        res = next(it)
        anim, new3d, proj, pn, pp, newvel, info = res
        anim.names = list(v["bvh"].names)
        np.save(os.path.join(v["out"], "foot_contacts"), constraints_to_contacts(newvel))
        with open(os.path.join(v["out"], "floor_out.txt"), "w") as f:
            f.write("%s %s %s\n%s %s %s" % tuple(str(float(q)) for q in list(pn) + list(pp)))
        save_bvh(os.path.join(v["out"], "final_test.bvh"), anim, v["bvh"].names, frametime)
        out.append(res)
    if vids:
        print("Finished kinematic optimization!")
    return out
