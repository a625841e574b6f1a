"""CPU tests of banded switch times (`PhysBatch(stage3_band_above=...)`, `chd_phys_options`): host-only layouts.

Default layouts must not change; banded ones must put every switch time into the time-ordered band and size the band
for every coupling stage 3 can produce, which is recomputed here from the problem's phase table and the oracle's row
times and variable spans."""
import ctypes as C

import numpy as np
import pytest

from tests.util import master_to_oracle_perm

TRUST = 0.04   # CHD_TAU_TRUST [s]: how far stage 3 may move a switch time


def _tables(b):
    lay = b.layout()
    lay.update(b.slot_index())
    lay["x0"] = b.get_x()
    lay["sizes"] = b.sizes
    lay["sizes_fixed"] = b.sizes_fixed()
    lay["dims"] = np.array(list(b.dims.values()))
    return lay


def _problems(chd):
    return {"walk2": [chd.synth.make_problem(s, n_ee=2) for s in range(4)],
            "dense150": [chd.synth.make_problem(s, n_frames=150, n_ee=4, dense=True) for s in range(2)],
            "dense600": [chd.synth.make_problem(s, n_frames=600, n_ee=4, dense=True) for s in range(2)]}


@pytest.mark.parametrize("name", ["walk2", "dense150", "dense600"])
def test_option_unset_keeps_layout(chd, name):
    """-1 (and, for batches without more than 96 phase durations, 96) gives exactly the tables of chd_phys_batch_create without options."""
    ps = _problems(chd)[name]
    ref = _tables(chd.phys.PhysBatch(ps, host_only=True))
    values = [-1] + ([96] if all(sum(len(d) - 1 for d in p.ee_durations) <= 96 for p in ps) else [])
    for v in values:
        got = _tables(chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=v))
        assert got.keys() == ref.keys()
        for k in ref:
            np.testing.assert_array_equal(got[k], ref[k], err_msg="%s stage3_band_above=%d" % (k, v))


def _n_dur(p):
    return sum(len(d) - 1 for d in p.ee_durations)


@pytest.mark.parametrize("frames", [200, 600])
def test_banded_switch_times_layout(chd, frames):
    from oracle.phys import OracleProblem
    ps = [chd.synth.make_problem(s, n_frames=frames, n_ee=4, dense=True) for s in range(2)]
    b = chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=96)
    lay = b.layout()
    sf = b.sizes_fixed()
    for i, p in enumerate(ps):
        nd = _n_dur(p)
        assert nd > 96
        n, m, _, Na, nb, w = (int(v) for v in b.sizes[i])
        assert sf[i, 2] == nd and sf[i, 0] == nb            # true count of phase durations; no switch time in the border
        vk, rk = lay["var_kkt"][i, :n], lay["row_kkt"][i, :m]
        assert (vk[n - nd:] >= 0).all() and (vk[n - nd:] < Na).all()
        used = np.concatenate([vk[vk >= 0], rk[rk >= 0]])
        assert len(np.unique(used)) == len(used) == Na + nb
        # --- independent recomputation of the switch-time couplings ---
        o = OracleProblem(p)
        o.set_stage("3")
        assert o.n == n
        rt = o.row_times()
        t0, t1 = o.var_times()
        sizes = o.var_set_sizes()                           # base lin, base ang, ee motion x n_ee, ee force x n_ee, durations
        off = np.concatenate([[0], np.cumsum(sizes)])
        sl = chd.phys.master_row_slices(b, i, lay)
        im, io = master_to_oracle_perm(sl, o)
        row_time = np.full(m, np.nan)
        row_time[im] = rt[io]
        kinds = {nm: (a, e) for nm, a, e in sl}

        def part(nm, j, cnt):                               # rows of the j-th of `cnt` equally long sets of one type
            a, e = kinds[nm]
            L = (e - a) // cnt
            return a + j * L, a + (j + 1) * L
        checked = 0
        tau0 = n - nd                                       # first switch time of the foot
        for ee, d in enumerate(p.ee_durations):
            ends = np.cumsum(d)
            ends[-1] = max(ends[-1], o.total_time)
            for k in range(len(d) - 1):
                v = tau0 + k
                lo = (ends[k - 1] if k > 0 else 0.0) - TRUST
                hi = ends[k + 1] + TRUST
                pos = vk[v]
                # explicit time-located rows of this foot (leg length, dynamics, toe-heel distance) inside the window
                sets = [part("rom", ee, p.n_ee), kinds["dyn"]] + ([part("heel", ee % 2, 2)] if p.n_ee == 4 else [])
                for a, e in sets:
                    r = np.arange(a, e)
                    r = r[(rk[r] >= 0) & (row_time[r] >= lo) & (row_time[r] <= hi)]
                    assert (np.abs(rk[r] - pos) <= w).all(), (ee, k, np.abs(rk[r] - pos).max(), w)
                    checked += len(r)
                # duration bound row d_k = tau_k - tau_{k-1} >= 0 (and the duration cost w D^T D)
                if k > 0:
                    assert abs(pos - vk[v - 1]) <= w
                # foot-motion node values living inside the window (cost samples and the rows above see them)
                mv = np.arange(off[2 + ee], off[3 + ee])
                mv = mv[(vk[mv] >= 0) & (vk[mv] < Na) & (t0[mv] >= lo) & (t1[mv] <= hi)]
                assert (np.abs(vk[mv] - pos) <= w).all(), (ee, k, np.abs(vk[mv] - pos).max(), w)
                checked += len(mv)
            rr = kinds["tottime"][0] + ee                # total-time row of this foot: last switch time only
            assert rk[rr] < 0 or abs(rk[rr] - vk[tau0 + len(d) - 2]) <= w
            tau0 += len(d) - 1
        assert checked > 1000


def test_small_counts_banded_on_request(chd):
    """0 bands every sequence with phase durations, also those the dense border would hold."""
    ps = [chd.synth.make_problem(s, n_ee=2) for s in range(4)]
    ref = chd.phys.PhysBatch(ps, host_only=True)
    b = chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=0)
    lay = b.layout()
    sf, sf0 = b.sizes_fixed(), ref.sizes_fixed()
    for i, p in enumerate(ps):
        n, Na, nb = int(b.sizes[i, 0]), int(b.sizes[i, 3]), int(b.sizes[i, 4])
        nd = _n_dur(p)
        assert sf[i, 2] == sf0[i, 2] == nd
        assert nb == sf[i, 0] == sf0[i, 0]                  # border = the stance variables of the default layout
        assert (lay["var_kkt"][i, n - nd:n] < Na).all()
        assert sf[i, 1] <= b.sizes[i, 5]
    np.testing.assert_array_equal(b.get_x(), ref.get_x())


@pytest.mark.parametrize("value", [-2, 97, 1000, -(2 ** 31), None, -1, 0, 96])
def test_create_option_range(chd, value):
    """chd_phys_batch_create takes a NULL option pointer (the defaults) or stage3_band_above in -1 .. 96; any other value
    returns -1 and no batch, through the C call and through PhysBatch."""
    ps = [chd.synth.make_problem(0, n_ee=2)]
    L = chd.phys.load_lib()
    arr, keep = chd.phys.make_problem_array(ps)
    opt = None if value is None else C.byref(chd.phys._Options(value))
    h = C.c_void_p()
    if value is None or -1 <= value <= 96:
        assert L.chd_phys_batch_create(arr, 1, None, -2, opt, C.byref(h)) == 0
        assert h.value
        L.chd_phys_batch_destroy(h)
        chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=value).close()
        return
    assert L.chd_phys_batch_create(arr, 1, None, -2, opt, C.byref(h)) == -1
    assert not h.value
    with pytest.raises(RuntimeError):
        chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=value)


def _gwin_fits(dims):
    """Batch-wide limits of the global-window KKT kernel: 96 panel groups, dynamic + static shared memory <= 227 KB."""
    Q, nbt = (dims["w_max"] + 7) // 8 + 1, (dims["nb_max"] + 1 + 7) // 8
    smem = (512 + (8 * nbt) ** 2 + 2 * (Q + nbt) * 64 + 16) * 8
    return Q - 1 + nbt <= 96 and smem + 16384 <= 232448


def test_mixed_batch_drops_banding_to_fit(chd):
    """Each sequence fits on its own, the batch (widest band of one, largest border of the other) would not: the banded
    sequence is built without banded switch times (stage 3 not attempted, as without the option), the batch builds."""
    ps = [chd.synth.make_problem(1, n_frames=600, n_ee=4, dense=True),
          chd.synth.make_problem(2, n_frames=200, n_ee=4, dense=False)]
    alone = chd.phys.PhysBatch(ps[:1], host_only=True, stage3_band_above=96)
    assert alone.sizes_fixed()[0, 2] > 96 and _gwin_fits(alone.dims)      # banded on its own
    b = chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=96)
    assert _gwin_fits(b.dims)
    assert b.sizes_fixed()[0, 2] == 0                                        # 600 frames: stage 3 off again
    ref = _tables(chd.phys.PhysBatch(ps, host_only=True))
    got = _tables(b)
    for k in ref:
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    # two banded long sequences together still fit: both keep their switch times in the band
    ps2 = [chd.synth.make_problem(s, n_frames=600, n_ee=4, dense=True) for s in (0, 1)]
    b2 = chd.phys.PhysBatch(ps2, host_only=True, stage3_band_above=96)
    assert (b2.sizes_fixed()[:, 2] > 96).all() and _gwin_fits(b2.dims)
