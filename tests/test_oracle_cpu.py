"""Known-answer and finite-difference tests that validate the CPU oracle itself (the reference ships no golden
vectors for this path, so the oracle is pinned by closed forms: SURVEY.md 8(c))."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def prob(chd):
    from oracle.phys import OracleProblem
    p = chd.synth.make_problem(5, n_frames=60, n_ee=4)
    return p, OracleProblem(p)


def test_hermite_closed_form(prob):
    p, o = prob
    o.set_stage("2.2")
    T = o.spline_poly_durations(0)
    x = o.get_x()
    # base_lin nodes: [px,py,pz,vx,vy,vz] per node (towr NodesVariablesAll)
    k, tl = 3, 0.037
    t = T[:k].sum() + tl
    n0, n1 = x[6 * k:6 * k + 6], x[6 * (k + 1):6 * (k + 1) + 6]
    Tk = T[k]
    p0, v0, p1, v1 = n0[:3], n0[3:], n1[:3], n1[3:]
    a, b = p0, v0
    c = -(3 * (p0 - p1) + Tk * (2 * v0 + v1)) / Tk ** 2
    d = (2 * (p0 - p1) + Tk * (v0 + v1)) / Tk ** 3
    got = o.spline_point(0, t)
    np.testing.assert_allclose(got[0], a + b * tl + c * tl ** 2 + d * tl ** 3, rtol=1e-13)
    np.testing.assert_allclose(got[1], b + 2 * c * tl + 3 * d * tl ** 2, rtol=1e-12)
    np.testing.assert_allclose(got[2], 2 * c + 6 * d * tl, rtol=1e-11)
    # junction rule: at a knot the previous segment is used (t >= t_global - 1e-10)
    tj = T[:4].sum()
    np.testing.assert_allclose(o.spline_point(0, tj)[0], x[6 * 4:6 * 4 + 3], rtol=1e-12)


def test_euler_matches_scipy_rotation(prob):
    from scipy.spatial.transform import Rotation
    p, o = prob
    for t in (0.0, 0.31, 1.07):
        e = o.spline_point(1, t)[0]
        R, w, wd = o.euler(t)
        # extrinsic xyz == intrinsic ZYX: R = Rz Ry Rx
        np.testing.assert_allclose(R, Rotation.from_euler("xyz", e).as_matrix(), atol=1e-13)
        # omega from a finite difference of R: [w]x = Rdot R^T
        h = 1e-6
        Rp = o.euler(t + h)[0]
        Rm = o.euler(t - h)[0]
        S = (Rp - Rm) / (2 * h) @ R.T
        np.testing.assert_allclose([S[2, 1], S[0, 2], S[1, 0]], w, atol=1e-6)
        wp, wm = o.euler(t + h)[1], o.euler(t - h)[1]
        np.testing.assert_allclose((wp - wm) / (2 * h), wd, atol=1e-5)


def test_stance_variable_pins_foot(prob):
    """A stance phase is one xyz variable shared by both nodes: the spline is constant during contact and its
    Jacobian wrt that variable sums to one (nodes_variables_dynamic_phase_based.cpp:88-101)."""
    p, o = prob
    ee = 0 if p.ee_start_contact[0] else 1
    assert p.ee_start_contact[ee]
    d0 = p.ee_durations[ee][0]
    a, b = o.spline_point(2 + ee, 0.1 * d0)[0], o.spline_point(2 + ee, 0.8 * d0)[0]
    np.testing.assert_allclose(a, b, atol=1e-15)
    rows = o.var_set_sizes()[2 + ee]
    J = o.spline_jac(2 + ee, 0.5 * d0, 0, rows)
    np.testing.assert_allclose(J[:, :3], np.eye(3), atol=1e-14)
    assert np.abs(J[:, 3:]).max() == 0.0


@pytest.mark.parametrize("stage", ["2.2", "3"])
def test_jacobian_and_gradient_finite_differences(chd, stage):
    from oracle.phys import OracleProblem
    p = chd.synth.make_problem(11, n_frames=40, n_ee=4)
    o = OracleProblem(p)
    o.set_stage(stage)
    n, m = o.n, o.m
    rng = np.random.default_rng(1)
    x = o.get_x() + rng.normal(0, 0.005, n)
    o.set_x(x)
    J = o.jac().toarray()
    g = o.grad()
    eps = 1e-6
    cols = rng.choice(n, size=120, replace=False)
    for i in cols:
        xp, xm = x.copy(), x.copy()
        xp[i] += eps
        xm[i] -= eps
        o.set_x(xp)
        cp, fp = o.cons(), o.cost()
        o.set_x(xm)
        cm, fm = o.cons(), o.cost()
        fd = (cp - cm) / (2 * eps)
        np.testing.assert_allclose(J[:, i], fd, rtol=2e-5, atol=2e-5 * max(1.0, np.abs(fd).max()))
        assert abs(g[i] - (fp - fm) / (2 * eps)) <= 1e-6 * max(1.0, abs(g[i]))
    o.set_x(x)


def test_staging_tables(prob):
    """Constraint sets per stage follow phys_optim.cpp:554-749 (SURVEY Appendix B)."""
    p, o = prob
    names = {}
    for st in ("1.1", "1.2", "2.1", "2.2", "3", "4"):
        o.set_stage(st)
        names[st] = [n.split("-")[0] for n, _ in o.constraint_sets()]
    assert set(names["1.1"]) == {"splineacc"}
    assert "dynamic" not in names["1.2"] and "leg" in names["1.2"] and "ee" in names["1.2"]
    assert "dynamic" in names["2.1"] and "height" not in names["2.1"]
    assert names["2.2"][-1] == "height"                     # height rows are appended last in stage 2.2
    assert names["3"][-1] == "contactduration" and names["4"][-1] == "ee"
    o.set_stage("3")
    assert o.n == sum(o.var_set_sizes())                    # durations join the variable vector only in stage 3


def test_oracle_ipm_converges_and_satisfies_constraints(chd):
    from oracle.phys import OracleProblem
    p = chd.synth.make_problem(3, n_frames=60, n_ee=2)
    o = OracleProblem(p)
    res = o.solve()
    assert all(s["status"] == 0 for s in res["stages"]), [s["status"] for s in res["stages"]]
    o.set_stage("4")
    c = o.cons()
    lo, hi = o.con_bounds()
    viol = np.maximum(lo - c, 0) + np.maximum(c - hi, 0)
    assert viol.max() <= 1e-4                                # IPOPT constr_viol_tol
    assert res["durations"].shape == (60, chd.phys.sample_stride(2))
