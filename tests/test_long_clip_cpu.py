"""CPU check that the long-clip configurations of tests/test_long_clip_gpu.py and scripts/long_horizon.py really have
iterates longer than the evaluation and line-search kernels can hold in shared memory (so they run those kernels'
global-memory form), and that the KKT plan of every one of them fits (csrc/chd_kkt_plan.h through the host build in
tests/emu, as tests/test_kkt_plan_cpu.py): batch creation accepts them on an H100."""
import pytest

from tests.test_kkt_plan_cpu import FITS, plan  # noqa: F401  (module fixture: the host build of the KKT plan)

THREADS, OPTIN = 512, 232448
# chd_iter_form (csrc/chd_api.cu): the shared-memory form needs (2 n_max + CHD_THREADS) doubles + 1 KB of the opt-in limit
SMEM_N_MAX = ((OPTIN - 1024) // 8 - THREADS) // 2


def _configs(chd):
    walk = lambda s, f: chd.synth.make_problem(s, n_frames=f, n_ee=4)
    dense = lambda s, f: chd.synth.make_problem(s, n_frames=f, n_ee=4, dense=True)
    return {
        "golden clip, 1100 frames, 4 ee, walking": [walk(0, 1100)],
        "700 frames, 4 ee, dense": [dense(0, 700)],
        "16 benchmark seeds + the golden clip": [chd.synth.make_problem(s, n_ee=2) for s in range(16)] + [walk(0, 1100)],
        "long_horizon.py --frames 1200 --sparse --batch 8": [walk(s, 1200) for s in range(8)],
        "long_horizon.py --frames 900 --batch 8": [dense(s, 900) for s in range(8)],
    }


def test_shared_memory_limit():
    assert SMEM_N_MAX == 14208
    assert (2 * SMEM_N_MAX + THREADS) * 8 + 1024 <= OPTIN < (2 * (SMEM_N_MAX + 1) + THREADS) * 8 + 1024


@pytest.mark.parametrize("name", ["golden clip, 1100 frames, 4 ee, walking", "700 frames, 4 ee, dense",
                                  "16 benchmark seeds + the golden clip", "long_horizon.py --frames 1200 --sparse --batch 8",
                                  "long_horizon.py --frames 900 --batch 8"])
def test_long_clip_crosses_the_limit_and_fits_the_kkt_plan(chd, plan, name):  # noqa: F811
    ps = _configs(chd)[name]
    b = chd.phys.PhysBatch(ps, host_only=True)
    d = b.dims
    assert d["n_max"] > SMEM_N_MAX, (name, d["n_max"])
    args = (d["na_max"], d["nb_max"], d["w_max"], int(b.sizes_fixed()[:, 1].max()), d["n_max"])
    p = plan(*args)
    assert p["status"] == FITS, (name, args, p)
    assert p["win_smem"] == 0                                 # the wide 4-foot band: chd_k_kkt_gwin
    # more phase durations than the dense border holds: stage 3 is not attempted (status -3), stage 4 runs
    assert all(sum(len(x) - 1 for x in q.ee_durations) > 96 for q in ps if q.n_frames >= 700)
    b.close()
