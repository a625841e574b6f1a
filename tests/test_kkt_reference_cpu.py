"""CPU checks of the reference behind tests/test_kkt_factor_gpu.py (tests/kkt_reference.py) and of its harness build:
the tile format round-trips, the block LDL^T in the kernels' order solves small quasi-definite systems as
scipy.linalg.solve does, the generators produce the inertia they are meant to (one positive pivot per primal unknown,
one negative per multiplier), and tests/kkt/kkt_harness.cu cross-compiles for sm_90a."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.linalg

import tests.kkt_reference as R

SHAPES = [(5, 0, 0), (8, 6, 1), (9, 7, 7), (63, 8, 8), (64, 15, 9), (65, 31, 64), (200, 96, 150)]


@pytest.mark.parametrize("Na,nbl,w", SHAPES)
@pytest.mark.parametrize("zero_tiles", [False, True], ids=["dense", "zero-tiles"])
def test_pack_unpack_round_trip(Na, nbl, w, zero_tiles):
    rng = np.random.default_rng(Na + nbl + w)
    K, _ = R.make_kkt(rng, Na, nbl, w, zero_tiles=zero_tiles)
    r = rng.standard_normal(Na + nbl)
    st = R.strides(Na + 3, nbl + 9, w + 8, w)             # wider strides than the system needs
    buf = R.pack(K, r, Na, nbl, st, st["Q"])
    K2, r2 = R.unpack(buf, Na, nbl, st, st["Q"])
    assert abs(K2 - K).max() == 0
    np.testing.assert_array_equal(r2, r)
    band = R.views(buf, st)[0]
    for k in range(Na, (Na + 7) & ~7):                     # identity padding
        assert band[k >> 3, 0, k & 7, k & 7] == 1.0


@pytest.mark.parametrize("Na,nbl,w", SHAPES[:6])
def test_reference_ldl_matches_dense_solve(Na, nbl, w):
    rng = np.random.default_rng(7 * Na + nbl)
    K, _ = R.make_kkt(rng, Na, nbl, w, delta_w=1e-2)
    r = rng.standard_normal(Na + nbl)
    st = R.strides(Na, nbl, w, w)
    f = R.ldl_solve(R.pack(K, r, Na, nbl, st, st["Q"]), Na, nbl, st, st["Q"])
    assert not f["fail"]
    x = scipy.linalg.solve(K.toarray(), r, assume_a="sym")
    xr, kappa = R.refined_solution(K, r)
    assert np.abs(f["x"] - xr).max() <= 1e-13 * kappa * np.abs(xr).max() + 1e-300
    np.testing.assert_allclose(f["x"], x, rtol=0, atol=1e-12 * kappa * np.abs(x).max())
    # and the factors reproduce K
    Kd = K.toarray()
    L, D = _dense_factors(f, Na, nbl, st, st["Q"])
    assert L.shape == (Na + nbl,) * 2
    np.testing.assert_allclose((L * D) @ L.T, Kd, rtol=0, atol=1e-12 * np.abs(Kd).max() * max(1.0, f["E"].max() / np.abs(Kd).max()))


def _dense_factors(f, Na, nbl, st, Qst):
    """Dense L (unit lower) and d of the reference's factors, border Schur factor recomputed from its pivots."""
    band, bord, _ = R.views(f["fac"], st)
    n, Np = Na + nbl, (Na + 7) & ~7
    L, d = np.eye(Np + nbl), np.zeros(Np + nbl)
    for J in range(Np // 8):
        T = band[J, 0]
        L[8 * J:8 * J + 8, 8 * J:8 * J + 8] += np.tril(T, -1)
        d[8 * J:8 * J + 8] = np.diagonal(T)
        for t in range(1, min(Qst, Np // 8 - J)):
            L[8 * (J + t):8 * (J + t) + 8, 8 * J:8 * J + 8] = band[J, t]
        for b in range(nbl):
            L[Np + b, 8 * J:8 * J + 8] = bord[J, b >> 3, b & 7]
    # border block: LDL^T of the Schur complement
    S = _schur(f, Na, nbl, st)
    for k in range(nbl):
        d[Np + k] = S[k, k]
        L[Np + k + 1:, Np + k] = S[k + 1:, k] / S[k, k]
        S[k + 1:, k + 1:] -= np.outer(L[Np + k + 1:, Np + k], S[k + 1:, k])
    keep = np.concatenate([np.arange(Na), Np + np.arange(nbl)])
    return L[np.ix_(keep, keep)], d[keep]


def _schur(f, Na, nbl, st):
    corn = R.views(f["fac"], st)[2]
    S = np.tril(corn[:nbl, :nbl])
    return S + np.tril(S, -1).T


@pytest.mark.parametrize("Na,nbl,w", SHAPES)
def test_generator_inertia(Na, nbl, w):
    """Quasi-definite by construction: one positive pivot per primal unknown (border included), one negative pivot per
    multiplier, whatever the elimination order."""
    for zt in (False, True):
        rng = np.random.default_rng(3 * Na + w)
        K, mult = R.make_kkt(rng, Na, nbl, w, zero_tiles=zt)
        st = R.strides(Na, nbl, w, w)
        assert R.inertia(K, Na, nbl, st, st["Q"]) == (Na - int(mult.sum()) + nbl, int(mult.sum()))


def test_harness_cross_compiles_for_sm90a(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not available")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kkt", "kkt_harness.cu")
    out = tmp_path / "kkt_harness.cubin"
    p = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-cubin", "-o", str(out), src], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    # the harness kernels carve the same static shared memory as chd_k_kkt / chd_k_kkt_gwin (tests/test_kkt_plan_cpu.py)
    assert "9600 bytes smem" in p.stderr and "12144 bytes smem" in p.stderr, p.stderr[-3000:]
