"""Shared helpers of the parity tests: mapping between the product's master row order and the
oracle's ifopt row order (which follows phys_optim.cpp's per-stage AddConstraintSet order), the checks that compare
a GPU solve with the oracle's or with another form of the same solve, and stand-ins for the queue's results and ABI."""
import ctypes as C

import numpy as np

import chd

ORACLE_PREFIX = {"acc": "splineacc", "terrain": "terrain-", "rom": "leg-length", "dyn": "dynamic", "force": "force-",
                 "heel": "ee-dist", "height": "height-", "tottime": "contactduration-"}


def oracle_type_blocks(o):
    """{type name: (start, stop)} of the oracle's rows for its current stage."""
    out, off = {}, 0
    for name, rows in o.constraint_sets():
        for k, pre in ORACLE_PREFIX.items():
            if name.startswith(pre):
                a, b = out.get(k, (off, off))
                out[k] = (a, off + rows)
        off += rows
    return out


def master_to_oracle_perm(master_slices, o):
    """index array idx such that g_master[idx_master] aligns with g_oracle[idx_oracle] for the types the
    oracle stage has; returns (idx_master, idx_oracle)."""
    blocks = oracle_type_blocks(o)
    im, io = [], []
    for name, a, b in master_slices:
        if name in blocks:
            oa, ob = blocks[name]
            assert ob - oa == b - a, (name, oa, ob, a, b)
            im.append(np.arange(a, b))
            io.append(np.arange(oa, ob))
    return np.concatenate(im), np.concatenate(io)


def to_tau(M, blocks):
    """Columns (last axis) with respect to phase durations d -> columns with respect to switch times tau (d = D tau):
    col(tau_k) = col(d_k) - col(d_{k+1}) inside every PhaseDurations block (offset, count)."""
    M = np.array(M, dtype=float, copy=True)
    for off, cnt in blocks:
        for k in range(cnt - 1):
            M[..., off + k] -= M[..., off + k + 1]
    return M


def duration_blocks(p, n):
    """(offset, count) of the PhaseDurations sets of problem p inside an x of length n (they are stacked last)."""
    cnts = [len(d) - 1 for d in p.ee_durations]
    off = n - sum(cnts)
    out = []
    for c in cnts:
        out.append((off, c))
        off += c
    return out


def assert_ipopt_termination(chd, b, i, p, stage):
    """IPOPT's termination test (phys_optim.cpp:578) at the final point of `stage` of sequence i of the solved batch b
    (problem p), with the residuals recomputed in numpy from the ORACLE's NLP callbacks (values, Jacobian, gradient:
    finite-difference verified in test_oracle_cpu.py); none of the solver's own error measures is used.  Scaled
    stationarity / feasibility / complementarity <= tol = 1e-3, unscaled constraint violation <= constr_viol_tol = 1e-4.
    Stage 3 adds the bounds d >= 0 of the phase durations (the product's `durpos` rows) and measures stationarity with
    respect to the switch times, the variables the solver drives it to zero in."""
    from oracle.phys import OracleProblem
    x, du, lay = b.get_x()[i], b.duals(), b.layout()
    o = OracleProblem(p)
    o.set_stage(stage)
    n = o.n
    o.set_x(x[:n])
    sl = chd.phys.master_row_slices(b, i, lay)
    im, io = master_to_oracle_perm(sl, o)
    assert len(io) == o.m
    c, J, g = o.cons(), o.jac().tocsr(), o.grad()
    cl, cu = o.con_bounds()
    sc, sf = du["row_scale"][i], du["obj_scale"][i]
    y, zL, zU, s = du["y"][i], du["zL"][i], du["zU"][i], du["s"][i]
    viol = max(np.maximum(cl - c, c - cu).max(), 0.0)           # primal feasibility (unscaled)
    lam = np.zeros(o.m)
    lam[io] = (sc * y)[im]
    r = sf * g + J.T @ lam                                      # stationarity of the scaled problem  sf grad f + J^T (sc y)
    cm = np.zeros(len(y))                                       # constraint values in master row order
    cm[im] = c[io]
    rows = im
    if stage == "3":
        nd = sum(len(d) - 1 for d in p.ee_durations)
        dur = x[n - nd:n]
        rows_dp = np.concatenate([np.arange(a, e) for nm, a, e in sl if nm == "durpos"])
        viol = max(viol, (-dur).max())
        r[n - nd:n] += (sc * y)[rows_dp]
        r = to_tau(r, duration_blocks(p, n))
        cm[rows_dp] = dur
        rows = np.concatenate([im, rows_dp])
    assert viol <= 1e-4, viol
    free = lay["var_kkt"][i, :n] >= 0
    lo, hi = lay["row_lo"][i, rows], lay["row_hi"][i, rows]
    ineq = lo != hi
    nbnd = int((lo[ineq] > -1e19).sum() + (hi[ineq] < 1e19).sum())
    s_d = max(100.0, (np.abs(y[rows]).sum() + (zL[rows][ineq] + zU[rows][ineq]).sum()) / (len(rows) + nbnd)) / 100.0
    assert np.abs(r[free]).max() / s_d <= 1e-3, (np.abs(r[free]).max(), s_d)
    # slack consistency and complementarity of the inequality rows
    ri = rows[ineq]
    assert np.abs(sc[ri] * cm[ri] - s[ri]).max() <= 1e-3
    lo_s, hi_s = lo[ineq] * sc[ri], hi[ineq] * sc[ri]
    relax = lambda v: 1e-8 * np.maximum(1.0, np.abs(v))
    hasl, hasu = lo[ineq] > -1e19, hi[ineq] < 1e19
    comp = np.concatenate([((s[ri] - (lo_s - relax(lo_s))) * zL[ri])[hasl], (((hi_s + relax(hi_s)) - s[ri]) * zU[ri])[hasu]])
    s_c = max(100.0, (zL[ri][hasl].sum() + zU[ri][hasu].sum()) / max(len(comp), 1)) / 100.0
    assert (comp >= 0).all() and comp.max() / s_c <= 1e-3, (comp.max(), s_c)
    assert np.abs(-y[ri] - zL[ri] + zU[ri]).max() / s_d <= 1e-3


def assert_samples_close(got, exp, n_ee, pos_atol=1e-5, frc_atol=1e-3):
    """Two solutions sampled as SaveSolution rows for n_ee end-effectors: base and foot positions (m, degrees) within
    pos_atol, foot forces within frc_atol (N), contact flags bit-exact; a tolerance of None skips its check.  Returns
    the max |diff| of the positions and of the forces."""
    base, pos, frc, flag = chd.phys.sample_columns(n_ee, n_ee)
    assert got.shape == exp.shape, (got.shape, exp.shape)
    pc = np.concatenate([base, pos])
    dp, df = np.abs(got[:, pc] - exp[:, pc]).max(), np.abs(got[:, frc] - exp[:, frc]).max()
    assert pos_atol is None or dp <= pos_atol, (dp, pos_atol)
    assert frc_atol is None or df <= frc_atol, (df, frc_atol)
    np.testing.assert_array_equal(got[:, flag], exp[:, flag])
    return dp, df


def assert_loosely_close(got, exp, n_ee):
    """Check for solves that took different paths to a KKT point of the same NLP (stage 3 or 4 of badly conditioned
    clips): COM within 2 cm, fewer than 2 % of the contact flags differ (switch times moved by less than a frame).
    Returns the max |diff| of the COM."""
    base, _, _, flag = chd.phys.sample_columns(n_ee, n_ee)
    dcom = np.abs(got[:, base[:3]] - exp[:, base[:3]]).max()
    assert dcom < 0.02, dcom
    assert (got[:, flag] != exp[:, flag]).mean() < 0.02
    return dcom


def assert_solves_agree(ref, got, n_ee, n_ee_max=None):
    """Two forms of one solve (`PhysBatch.solve()` results; ref's rows hold n_ee end-effectors, `got` may hold more
    sequences after ref's, and its rows may be padded for n_ee_max end-effectors): equal status and iteration counts in stages 1.1-2.2 with snapshots 0 and 1
    within assert_samples_close's tolerances; equal status in stages 3 and 4; equal stage-3 iteration counts for at
    least 90 % of the sequences, and the final snapshot within the same tolerances where they are equal."""
    B = ref["stage_status"].shape[1]
    st, it = got["stage_status"][:, :B], got["stage_iters"][:, :B]
    cols = np.concatenate(chd.phys.sample_columns(n_ee, n_ee_max or n_ee))

    def close(snap, i):
        nf = ref["frames"][i]
        return assert_samples_close(got["samples"][snap, i, :nf][:, cols], ref["samples"][snap, i, :nf], n_ee)

    np.testing.assert_array_equal(st[:4], ref["stage_status"][:4])
    np.testing.assert_array_equal(it[:4], ref["stage_iters"][:4])
    fixed = np.array([close(snap, i) for snap in (0, 1) for i in range(B)])
    print("stages 1.1-2.2: max |diff| positions %.2e, forces %.2e" % tuple(fixed.max(axis=0)))
    np.testing.assert_array_equal(st[4], ref["stage_status"][4])
    np.testing.assert_array_equal(st[5], ref["stage_status"][5])
    same = np.nonzero(it[4] == ref["stage_iters"][4])[0]
    print("stage 3: iteration counts equal for %d / %d sequences" % (len(same), B))
    assert len(same) >= 0.9 * B
    d3 = np.array([close(2, i) for i in same])
    print("stage 3: max |diff| positions %.2e, forces %.2e" % tuple(d3.max(axis=0)))


QUEUE_KEYS = chd.phys.SOLVE_KEYS + ("stage_stats",)   # what a queue solve writes, before `solved` and the cost terms


def random_result(n, fo, stride=20, terms=False, seed=5):
    """What a queue would compute for n clips (`QUEUE_KEYS`, with `terms` also `cost_terms`): integers in each field's
    range, normal floats with mixed signs and about one entry in ten -0.0 in every float field."""
    rng = np.random.default_rng(seed)
    out = chd.phys.result_arrays(n, QUEUE_KEYS + (("cost_terms",) if terms else ()), fo, stride)
    ints = dict(frames=(1, fo + 1), success=(0, 2), stage_status=(-3, 2), stage_iters=(0, 3000))
    for k, v in out.items():
        if k in ints:
            v[:] = rng.integers(*ints[k], v.shape)
        else:
            v[:] = rng.standard_normal(v.shape)
            v[rng.random(v.shape) < 0.1] = -0.0
    return out


class QueueLib:
    """Stands in for libchd's queue: records the clip order (`frames_in`) and the per-clip weights (`weights`, None
    without them) it is created with, and answers every clip a solve covers with its queue position k and frame count f:
    samples[:, k, :f, 0] = f, frames f, success (k, f), stage_status k, stage_iters f, stage_stats f and, into a buffer
    set with chd_phys_set_cost_terms_out, cost terms 100 k + column.  A solve covers every clip, or with a claim source
    (chd_phys_queue_set_claim) the positions it hands out: it is asked for `slots` positions, then for `wants` in turn (as
    finished slots would ask) until it returns fewer than asked."""

    def __init__(self, wants=()):
        self.wants, self.cb, self.asked = list(wants), None, []
        self.terms_ptr, self.set_calls = None, []

    def chd_phys_queue_create(self, arr, n, slots, w, dev, opt, out):
        self.n, self.slots = n, min(slots, n)
        self.frames_in = [arr[k].n_frames for k in range(n)]
        self.stride = chd.phys.sample_stride(max(arr[k].n_ee for k in range(n)))
        cw = opt._obj.clip_weights if opt is not None else None
        self.weights = [tuple(getattr(cw[k], f) for f, _ in cw[k]._fields_) for k in range(n)] if cw else None
        out._obj.value = 1
        return 0

    def chd_phys_get_dims(self, h, d):
        d._obj.batch, d._obj.frames_out_max = self.slots, max(self.frames_in)
        return 0

    def chd_phys_queue_set_claim(self, h, cb, ctx):
        self.cb = C.cast(cb, chd.phys.CLAIM_FN)
        return 0

    def chd_phys_set_cost_terms_out(self, h, p):
        self.terms_ptr = p
        self.set_calls.append(p is not None)
        return 0

    def _claimed(self):
        """positions handed out by the claim source, None: it failed"""
        given = []
        for want in [self.slots] + self.wants:
            first = C.c_int32(-7)
            k = self.cb(None, want, C.byref(first))
            self.asked.append(want)
            if k < 0:
                return None
            given += range(first.value, first.value + k)
            if k < want:
                break
        return given

    def chd_phys_queue_solve(self, h, *ptrs):
        given = range(self.n) if self.cb is None else self._claimed()
        if given is None:
            return -1
        res = chd.phys.result_arrays(self.n, QUEUE_KEYS + ("cost_terms",), max(self.frames_in), self.stride)
        view = lambda p, a: np.ctypeslib.as_array(C.cast(p, C.POINTER(np.ctypeslib.as_ctypes_type(a.dtype))), a.shape)
        out = {k: view(p, res[k]) for k, p in zip(QUEUE_KEYS, ptrs)}
        if self.terms_ptr is not None:
            out["cost_terms"] = view(self.terms_ptr, res["cost_terms"])
        for k in given:
            f = self.frames_in[k]
            out["samples"][:, k, :f, 0] = f
            out["frames"][k] = f
            out["success"][k] = (k, f)
            out["stage_status"][:, k], out["stage_iters"][:, k] = k, f
            out["stage_stats"][:, k, :] = f
            if "cost_terms" in out:
                out["cost_terms"][k] = 100 * k + np.arange(len(chd.phys.COST_TERMS))
        return 0

    def chd_phys_batch_destroy(self, h):
        pass
