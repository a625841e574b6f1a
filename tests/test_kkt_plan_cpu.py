"""CPU check of the KKT plan (csrc/chd_kkt_plan.h, reached through the host build in tests/emu): the tile counts, the
storage stride, the kernel choice, the shared-memory and scratch sizes and the errors equal what batch creation worked
out on its own before the plan existed; and the regions the KKT kernels carve from those sizes lie inside their space,
the ones that are not aliases are disjoint, and with the window in shared memory the back-substitution's staging ends
before the vectors that alias the window's tail."""
import ctypes as C
import itertools
import os
import re
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PLAN_H = os.path.join(HERE, "..", "contact-human-dynamics_b200", "csrc", "chd_kkt_plan.h")
THREADS, OPTIN, GWIN_STATIC_MAX = 512, 232448, 16384
KKT_STATIC, GWIN_STATIC = 9600, 12144          # ptxas (sm_90a) static shared memory of chd_k_kkt / chd_k_kkt_gwin
FITS, TOO_WIDE_COMPACT, TOO_WIDE_PAIRS, TOO_LARGE = 0, 1, 2, 3


def _plan_type():
    body = re.search(r"struct ChdKktPlan \{(.*?)\};", open(PLAN_H).read(), re.S).group(1)
    fields = []
    for typ, names in re.findall(r"^\s*(int|size_t)\s+([^;]+);", body, re.M):
        fields += [(n.strip(), C.c_int if typ == "int" else C.c_size_t) for n in names.split(",")]
    return type("ChdKktPlan", (C.Structure,), {"_fields_": fields})


@pytest.fixture(scope="module")
def plan():
    subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "emu")])
    L = C.CDLL(os.path.join(HERE, "emu", "libchd_emu.so"))
    T = _plan_type()
    L.chd_emu_kkt_plan.argtypes = [C.c_int] * 5 + [C.c_longlong] * 3 + [C.POINTER(T)]

    def f(Na, nb, w, w_fix, n, kkt_static=KKT_STATIC, gwin_static=GWIN_STATIC, optin=OPTIN):
        p = T()
        assert L.chd_emu_kkt_plan(Na, nb, w, w_fix, n, kkt_static, gwin_static, optin, C.byref(p)) == C.sizeof(T)
        return {k: getattr(p, k) for k, _ in T._fields_}
    return f


def parent_plan(Na, nb, w, w_fix, n, kkt_static=KKT_STATIC, gwin_static=GWIN_STATIC, optin=OPTIN):
    """What batch creation computed before the plan: the sizes it put into ChdDev, the kernel and its dynamic shared
    memory, the scratch stride and its errors."""
    nbc, Q, Qfix, nbt = (Na + 7) // 8, (w + 7) // 8 + 1, (w_fix + 7) // 8 + 1, (nb + 1 + 7) // 8
    nbp8 = 8 * nbt
    win_tiles = max(Q * (Q + 1) // 2, 2 * Q)
    r = dict(nbc_max=nbc, Q=Q, Qfix=Qfix, nbt=nbt, win_tiles=win_tiles,
             kstride=nbc * Q * 64 + nbc * nbt * 64 + 64 * nbt * nbt, scratch_stride=0)
    n_even, xs_len = (n + 1) & ~1, 8 * nbc + nbp8
    pan = max(2 * (Q + nbt) * 64, 8 * nbc)
    kkt_fixed = (THREADS + nbp8 * nbp8 + pan + 16) * 8
    kkt_win = (win_tiles * 64 + Q * nbt * 64) * 8
    vectors_fit = win_tiles * 64 + Q * nbt * 64 >= n_even + xs_len + 2 * Q * 64 + 3072
    if vectors_fit and kkt_fixed + kkt_win + kkt_static + 256 <= optin:
        r.update(win_smem=1, pan_doubles=pan, smem_bytes=kkt_fixed + kkt_win,
                 status=TOO_WIDE_COMPACT if Q - 1 + nbt > 64 else FITS)
    else:
        pan = 2 * (Q + nbt) * 64
        smem = (THREADS + nbp8 * nbp8 + pan + 16) * 8
        r.update(win_smem=0, pan_doubles=pan, smem_bytes=smem,
                 scratch_stride=n_even + xs_len + 8 * nbc + win_tiles * 64 + Q * nbt * 64,
                 status=TOO_WIDE_PAIRS if Q - 1 + nbt > 96 else (TOO_LARGE if smem + gwin_static + 256 > optin else FITS))
    return r


def kernel_regions(p, n_max):
    """The carve-up chd_kkt_ctx_init / chd_kkt_border / chd_kkt_backsub make of the plan's sizes: region -> (offset,
    length) in doubles, for a stage with Qs band tiles per block column, and the back-substitution chunk rows R."""
    nbc, Q, nbt, nbp8 = p["nbc_max"], p["Q"], p["nbt"], 8 * p["nbt"]
    n_even, xs_len = (n_max + 1) & ~1, 8 * nbc + nbp8
    win_region = p["win_tiles"] * 64 + Q * nbt * 64
    ypan = THREADS + nbp8 * nbp8
    dinv = ypan + p["pan_doubles"]
    if p["win_smem"]:
        win = dinv + 16
        vecn = win + win_region - n_even
        xs, xs2 = vecn - xs_len, ypan
    else:
        vecn, xs, xs2 = 0, n_even, n_even + xs_len
        win = n_even + xs_len + 8 * nbc
    out = {}
    for Qs in (p["Qfix"], Q):
        R = max(1, (win_region - (n_even + xs_len if p["win_smem"] else 0)) // 64 // (2 * Qs))
        out[Qs] = dict(
            shared={"red": (0, THREADS), "cc": (THREADS, nbp8 * nbp8), "ypan": (ypan, (Qs + nbt) * 64),
                    "xpan": (ypan + (Qs + nbt) * 64, (Qs + nbt) * 64), "dinv": (dinv, 16)},
            window={"win": (win, p["win_tiles"] * 64), "bwin": (win + p["win_tiles"] * 64, Q * nbt * 64)},
            vectors={"vecn": (vecn, n_max), "xs": (xs, 8 * nbc), "xb": (xs + 8 * nbc, nbp8)},
            accum={"xs2": (xs2, 8 * nbc)}, stage=(win, 2 * R * Qs * 64), dinv=dinv)
    return out


def _disjoint(regions):
    for (a, (oa, la)), (b, (ob, lb)) in itertools.combinations(regions.items(), 2):
        assert oa + la <= ob or ob + lb <= oa, (a, oa, la, b, ob, lb)


def _inside(regions, lo, hi):
    for name, (o, ln) in regions.items():
        assert lo <= o and o + ln <= hi, (name, o, ln, lo, hi)


def check_regions(p, n_max):
    """Every region inside its space, the non-aliases disjoint, the aliases clear of what is live beside them."""
    smem = p["smem_bytes"] // 8
    assert p["smem_bytes"] % 8 == 0
    for r in kernel_regions(p, n_max).values():
        win, win_len = r["window"]["win"]
        win_end = r["window"]["bwin"][0] + r["window"]["bwin"][1]
        stage_end = r["stage"][0] + r["stage"][1]   # back-substitution staging: two chunks of R block rows
        assert stage_end <= win_end
        if p["win_smem"]:
            _inside({**r["shared"], **r["window"]}, 0, smem)
            _disjoint({**r["shared"], **r["window"]})
            _inside(r["vectors"], win, win_end)     # aliases of the window's tail ...
            _disjoint(r["vectors"])
            assert stage_end <= r["vectors"]["xs"][0], (stage_end, r["vectors"]["xs"])   # ... clear of the staging
            _inside(r["accum"], r["shared"]["ypan"][0], r["dinv"])   # alias of the idle panel buffers
        else:
            _inside(r["shared"], 0, smem)
            _disjoint(r["shared"])
            _inside({**r["window"], **r["vectors"], **r["accum"]}, 0, p["scratch_stride"])
            _disjoint({**r["window"], **r["vectors"], **r["accum"]})


def _compare(plan, args):
    got, ref = plan(*args), parent_plan(*args)
    assert (got["status"], got["win_smem"]) == (ref["status"], ref["win_smem"]), args
    if ref["status"] == FITS:
        for k, v in ref.items():
            assert got[k] == v, (k, got[k], v, args)
        check_regions(got, args[4])
    return got


def test_plan_grid(plan):
    kinds = {0: 0, 1: 0}
    for Na, nb, w, fix, nfac, (ks, gs, op) in itertools.product(
            (8, 97, 977, 2500, 8000, 24000), (0, 5, 40, 96, 150, 400), (8, 30, 63, 100, 190, 400), (1, 2), (1, 3),
            ((KKT_STATIC, GWIN_STATIC, OPTIN), (0, 0, OPTIN), (KKT_STATIC, GWIN_STATIC, 101376))):
        p = _compare(plan, (Na, nb, w, w // fix, Na // nfac, ks, gs, op))
        if p["status"] == FITS:
            kinds[p["win_smem"]] += 1
    assert kinds[0] > 50 and kinds[1] > 50, kinds


def test_plan_bench_batches(chd, plan):
    """The layouts of the benchmark's workloads and of the banded stage 3."""
    configs = {"phys 64 x 120 frames, 2 ee": ([chd.synth.make_problem(s, 120, 2) for s in range(64)], None),
               "long 600 frames, 4 ee, dense": ([chd.synth.make_problem(s, 600, 4, dense=True) for s in range(16)], None),
               "banded stage 3, 200 frames": ([chd.synth.make_problem(s, 200, 4, dense=True) for s in range(2)], 96),
               "banded stage 3, 600 frames": ([chd.synth.make_problem(s, 600, 4, dense=True) for s in range(2)], 96)}
    for name, (ps, band) in configs.items():
        b = chd.phys.PhysBatch(ps, host_only=True, stage3_band_above=band)
        d = b.dims
        args = (d["na_max"], d["nb_max"], d["w_max"], int(b.sizes_fixed()[:, 1].max()), d["n_max"])
        p = _compare(plan, args)
        assert p["status"] == FITS, (name, args)
        b.close()


def test_layout_band_limit(plan):
    """chd_kkt_gwin_status at the static-size bound (the layout builder's kkt_fits; the plan of chd_k_kkt_gwin goes
    through it too) accepts exactly the bands kkt_fits accepted before: at most 96 panel groups, dynamic + bounded
    static shared memory within the opt-in limit."""
    for w, nb in itertools.product(range(0, 800, 7), range(0, 800, 9)):
        Q, nbt = (w + 7) // 8 + 1, (nb + 1 + 7) // 8
        before = Q - 1 + nbt <= 96 and (512 + (8 * nbt) ** 2 + 2 * (Q + nbt) * 64 + 16) * 8 + GWIN_STATIC_MAX <= OPTIN
        p = plan(0, nb, w, w, 0, OPTIN, GWIN_STATIC_MAX, OPTIN)
        assert p["win_smem"] == 0 and (p["status"] == FITS) == before, (w, nb)
