"""Host-side mirror of the reference's phys-optim operator for a batch of sequences.

`PhysBatch` binds libchd.so (hand-written sm_90a kernels behind a C ABI, include/chd.h) through ctypes.
There is NO CPU fallback: if the CUDA library is missing or no GPU is visible, construction fails loudly
(`host_only=True` builds only the host-side NLP layout tables, which is what the CPU tests exercise).

Reference interface mirrored (towr_phys_optim/phys_optim.cpp): one object per `ifopt::Problem` batch,
`solve_stage()` per `solver->Solve(nlp)` call, `solve()` for the staged schedule :554-749, `sample()` for
`SaveSolution` :63-143.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from .io_formats import PhysProblem

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

STAGES = {"1.1": 0, "1.2": 1, "2.1": 2, "2.2": 3, "3": 4, "4": 5}
SET_NAMES = {0: "acc", 1: "terrain", 2: "rom", 3: "dyn", 4: "force", 5: "heel", 6: "height", 7: "tottime", 8: "durpos"}


class _Problem(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("n_ee", C.c_int32), ("dt", C.c_double),
                ("hip_left", C.POINTER(C.c_double)), ("hip_right", C.POINTER(C.c_double)),
                ("max_leg_length", C.c_double), ("max_heel_length", C.c_double), ("heel_dist", C.c_double),
                ("body_mass", C.c_double), ("inertia", C.POINTER(C.c_double)), ("base_lin", C.POINTER(C.c_double)),
                ("base_ang", C.POINTER(C.c_double)), ("ee_pos", C.POINTER(C.c_double)),
                ("floor_normal", C.c_double * 3), ("floor_point", C.c_double * 3),
                ("ee_start_contact", C.POINTER(C.c_int32)), ("ee_n_phases", C.POINTER(C.c_int32)),
                ("ee_durations", C.POINTER(C.c_double))]


class _Weights(C.Structure):
    _fields_ = [("w_com_lin", C.c_double), ("w_com_ang", C.c_double), ("w_ee", C.c_double), ("w_smooth", C.c_double),
                ("w_dur", C.c_double)]


class _Options(C.Structure):
    _fields_ = [("stage3_band_above", C.c_int32)]


class _Dims(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("batch", "n_max", "m_max", "slots_max", "n_splines", "p_max", "sets_max",
                                          "na_max", "nb_max", "w_max", "frames_out_max")]


_vp, _i32, _i64, _int, _f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_int, C.c_double

# Every function of include/chd.h, name -> (restype, argtypes); load_lib applies it.  Arrays, handles and streams are
# passed as c_void_p.
SIGNATURES = {
    "chd_phys_batch_create": (_int, [C.POINTER(_Problem), _i32, C.POINTER(_Weights), _i32, C.POINTER(_Options),
                                     C.POINTER(_vp)]),
    "chd_phys_batch_destroy": (None, [_vp]),
    "chd_phys_get_dims": (_int, [_vp, C.POINTER(_Dims)]),
    "chd_phys_get_sizes": (_int, [_vp, _vp]),
    "chd_phys_get_sizes_fixed": (_int, [_vp, _vp]),
    "chd_phys_get_x": (_int, [_vp, _vp]),
    "chd_phys_set_x": (_int, [_vp, _vp]),
    "chd_phys_eval": (_int, [_vp, _i32, _vp, _vp, _vp, _vp]),
    "chd_phys_get_layout": (_int, [_vp] * 8),
    "chd_phys_get_slot_index": (_int, [_vp] * 4),
    "chd_phys_get_ent_col": (_int, [_vp, _vp]),
    "chd_phys_get_duals": (_int, [_vp] * 7),
    "chd_phys_stage_stats": (_int, [_vp, _vp]),
    "chd_phys_solve_stage": (_int, [_vp, _i32, _i32, _vp, _vp, _vp]),
    "chd_phys_solve": (_int, [_vp] * 6),
    "chd_phys_sample": (_int, [_vp, _vp, _vp]),
    "chd_phys_sample_device": (_int, [_vp, _vp, _vp]),
    "chd_phys_launch_count": (_i64, [_vp]),
    "chd_phys_h2d_bytes": (_i64, [_vp]),
    "chd_phys_reset": (_int, [_vp]),
    "chd_phys_kernel_times": (_int, [_vp, _vp, _vp, _int]),
    "chd_phys_set_timing": (_int, [_vp, _int]),
    "chd_contact_create": (_int, [_vp, _vp, _vp, C.c_float, _i32, C.POINTER(_vp)]),
    "chd_contact_destroy": (None, [_vp]),
    "chd_contact_forward": (_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "chd_contact_forward_device": (_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "chd_contact_preprocess": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "chd_contact_detect": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "chd_contact_launch_count": (_i64, [_vp]),
    "chd_contact_set_precision": (_int, [_vp, _i32]),
    "chd_openpose_load": (_int, [C.POINTER(C.c_char_p), _i32, _i32, _vp, _i32]),
    "chd_kin_solve": (_int, [_vp] * 7 + [_i32] * 3 + [_vp] * 4),
    "chd_kin_work_bytes": (_i64, [_i32]),
    "chd_ik_solve": (_int, [_i32, _vp, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _f64, _f64, _i32, _vp, _vp]),
    "chd_ik_work_bytes": (_i64, [_i32] * 3),
    "chd_version": (C.c_char_p, []),
    "chd_measure_fp64_peak": (_int, [C.POINTER(_f64), C.POINTER(_f64)]),
}


def measure_fp64_peak():
    """(DFMA GFLOP/s, DMMA GFLOP/s) sustained on the current device (`chd_measure_fp64_peak`)."""
    L = load_lib()
    a, b = C.c_double(0), C.c_double(0)
    rc = L.chd_measure_fp64_peak(C.byref(a), C.byref(b))
    if rc != 0:
        raise RuntimeError("chd_measure_fp64_peak failed with code %d" % rc)
    return a.value, b.value


def lib_path() -> str:
    return os.path.join(_HERE, "libchd.so")


def load_lib():
    """Loads libchd.so; raises if it has not been built (no fallback path exists)."""
    global _LIB
    if _LIB is None:
        path = lib_path()
        if not os.path.exists(path):
            raise RuntimeError("libchd.so is missing (%s): run `python -c 'import __graft_entry__ as g; g.build()'`" % path)
        L = C.CDLL(path)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def make_problem_array(problems):
    """ctypes array of `chd_phys_problem` for a list of PhysProblem + the numpy buffers it points into."""
    B = len(problems)
    arr = (_Problem * B)()
    keep = []
    for i, p in enumerate(problems):
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        k = [f64(p.hip_left), f64(p.hip_right), f64(p.inertia), f64(p.base_lin), f64(p.base_ang), f64(p.ee_pos),
             np.ascontiguousarray(p.ee_start_contact, dtype=np.int32),
             np.ascontiguousarray([len(d) for d in p.ee_durations], dtype=np.int32),
             f64(np.concatenate([np.asarray(d, dtype=np.float64) for d in p.ee_durations]))]
        keep.append(k)
        q = arr[i]
        q.n_frames, q.n_ee, q.dt = p.n_frames, p.n_ee, p.dt
        q.hip_left, q.hip_right, q.inertia = _dp(k[0]), _dp(k[1]), _dp(k[2])
        q.base_lin, q.base_ang, q.ee_pos = _dp(k[3]), _dp(k[4]), _dp(k[5])
        q.max_leg_length, q.max_heel_length, q.heel_dist, q.body_mass = (p.max_leg_length, p.max_heel_length,
                                                                          p.heel_dist, p.body_mass)
        for d in range(3):
            q.floor_normal[d] = float(p.floor_normal[d])
            q.floor_point[d] = float(p.floor_point[d])
        q.ee_start_contact, q.ee_n_phases, q.ee_durations = _ip(k[6]), _ip(k[7]), _dp(k[8])
    return arr, keep


class PhysBatch:
    """`stage3_band_above`: sequences with more phase-duration variables than this carry their switch times as banded
    KKT unknowns, which lets stage 3 run beyond the 96 the dense border holds (0 bands every sequence; None: none)."""

    def __init__(self, problems: Sequence[PhysProblem], weights=(0.4, 1.7, 0.3, 0.1, 0.1), device: int = -1,
                 host_only: bool = False, stage3_band_above: Optional[int] = None):
        self.L = load_lib()
        self.problems = list(problems)
        B = len(self.problems)
        arr, self._keep = make_problem_array(self.problems)
        w = _Weights(*[float(x) for x in weights])
        h = C.c_void_p()
        dev = -2 if host_only else device
        # values outside 0..96 are rejected by the library (code -1)
        opt = None if stage3_band_above is None else C.byref(_Options(int(stage3_band_above)))
        rc = self.L.chd_phys_batch_create(arr, B, C.byref(w), dev, opt, C.byref(h))
        if rc != 0:
            raise RuntimeError("chd_phys_batch_create failed with code %d (no CUDA device? no CPU fallback exists)" % rc)
        self.h = h
        self.host_only = host_only
        d = _Dims()
        self.L.chd_phys_get_dims(self.h, C.byref(d))
        self.dims = {k: getattr(d, k) for k, _ in _Dims._fields_}
        self.B = B
        sz = np.zeros((B, 6), dtype=np.int32)
        self.L.chd_phys_get_sizes(self.h, _ptr(sz))
        self.sizes = sz  # n, m, nslots, Na, nb, w
        self.n_ee_max = max(p.n_ee for p in self.problems)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self):
        if getattr(self, "h", None):
            self.L.chd_phys_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- iterate -------------------------------------------------------------------------------
    def get_x(self) -> np.ndarray:
        x = np.zeros((self.B, self.dims["n_max"]))
        self._chk(self.L.chd_phys_get_x(self.h, _ptr(x)))
        return x

    def set_x(self, x: np.ndarray):
        x = np.ascontiguousarray(x, dtype=np.float64)
        assert x.shape == (self.B, self.dims["n_max"])
        self._chk(self.L.chd_phys_set_x(self.h, _ptr(x)))

    def layout(self) -> dict:
        B, d = self.B, self.dims
        out = dict(ent_ptr=np.zeros((B, d["m_max"] + 1), np.int32), ent_col=np.zeros((B, d["slots_max"]), np.int32),
                   row_lo=np.zeros((B, d["m_max"])), row_hi=np.zeros((B, d["m_max"])),
                   row_set=np.zeros((B, d["m_max"]), np.int32), var_kkt=np.zeros((B, d["n_max"]), np.int32),
                   row_kkt=np.zeros((B, d["m_max"]), np.int32))
        self._chk(self.L.chd_phys_get_layout(self.h, *[_ptr(out[k]) for k in ("ent_ptr", "ent_col", "row_lo", "row_hi",
                                                                              "row_set", "var_kkt", "row_kkt")]))
        return out

    def sizes_fixed(self) -> np.ndarray:
        """(B, 3): border unknowns / half bandwidth of the fixed-duration stages, number of phase-duration variables."""
        out = np.zeros((self.B, 3), np.int32)
        self._chk(self.L.chd_phys_get_sizes_fixed(self.h, _ptr(out)))
        return out

    def ent_col(self) -> np.ndarray:
        """Jacobian slot columns as they stand on the device (run-time pattern once stage 3 has moved a duration)."""
        out = np.zeros((self.B, self.dims["slots_max"]), np.int32)
        self._chk(self.L.chd_phys_get_ent_col(self.h, _ptr(out)))
        return out

    def duals(self) -> dict:
        """Interior-point state of the last solved stage (scaled problem), master row order."""
        B, d = self.B, self.dims
        out = {k: np.zeros((B, d["m_max"])) for k in ("y", "zL", "zU", "s", "row_scale")}
        out["obj_scale"] = np.zeros(B)
        self._chk(self.L.chd_phys_get_duals(self.h, *[_ptr(out[k]) for k in ("y", "zL", "zU", "s", "row_scale", "obj_scale")]))
        return out

    def stage_stats(self) -> np.ndarray:
        """(6, B, 4): objective, scaled NLP error, unscaled constraint violation, unscaled dual infeasibility per stage."""
        out = np.zeros((6, self.B, 4))
        self._chk(self.L.chd_phys_stage_stats(self.h, _ptr(out)))
        return out

    def slot_index(self) -> dict:
        """Column-oriented view of the Jacobian slots: ent_row (B,slots_max), col_ptr (B,n_max+1), col_ent (B,slots_max)."""
        B, d = self.B, self.dims
        out = dict(ent_row=np.zeros((B, d["slots_max"]), np.int32), col_ptr=np.zeros((B, d["n_max"] + 1), np.int32),
                   col_ent=np.zeros((B, d["slots_max"]), np.int32))
        self._chk(self.L.chd_phys_get_slot_index(self.h, *[_ptr(out[k]) for k in ("ent_row", "col_ptr", "col_ent")]))
        return out

    def eval(self, stage) -> dict:
        """cost (B,), grad (B,n_max), g (B,m_max) in master row order, jac slot values (B,slots_max)."""
        B, d = self.B, self.dims
        out = dict(cost=np.zeros(B), grad=np.zeros((B, d["n_max"])), g=np.zeros((B, d["m_max"])),
                   jac=np.zeros((B, d["slots_max"])))
        self._chk(self.L.chd_phys_eval(self.h, STAGES.get(stage, stage), _ptr(out["cost"]), _ptr(out["grad"]), _ptr(out["g"]),
                                       _ptr(out["jac"])))
        return out

    def jac_csr(self, i: int, jac_vals: np.ndarray, lay: Optional[dict] = None):
        """Expands sequence i's block-row slots into a scipy CSR matrix (m x n), master row order."""
        import scipy.sparse as sp
        lay = lay or self.layout()
        n, m = int(self.sizes[i, 0]), int(self.sizes[i, 1])
        ptr = lay["ent_ptr"][i, :m + 1]
        cols = lay["ent_col"][i, :ptr[-1]]
        vals = jac_vals[i, :ptr[-1]]
        rows = np.repeat(np.arange(m), np.diff(ptr))
        keep = cols >= 0
        return sp.csr_matrix((vals[keep], (rows[keep], cols[keep])), shape=(m, n))

    # ---- solves --------------------------------------------------------------------------------
    def solve_stage(self, stage, max_iter: int = 0) -> dict:
        B = self.B
        st, it, stats = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros((B, 8))
        self._chk(self.L.chd_phys_solve_stage(self.h, STAGES.get(stage, stage), int(max_iter), _ptr(st), _ptr(it), _ptr(stats)))
        return dict(status=st, iters=it, f=stats[:, 0], E0=stats[:, 1], viol=stats[:, 2], dual=stats[:, 3],
                    compl=stats[:, 4], mu=stats[:, 5], delta_w=stats[:, 6], ls_fail=stats[:, 7])

    def solve(self) -> dict:
        """Full staged schedule.  Returns the three SaveSolution snapshots, frame counts, success flags."""
        B, d = self.B, self.dims
        stride = 6 + 7 * self.n_ee_max
        samples = np.zeros((3, B, d["frames_out_max"], stride))
        frames = np.zeros(B, np.int32)
        success = np.zeros((B, 2), np.int32)
        sstat = np.zeros((6, B), np.int32)
        siter = np.zeros((6, B), np.int32)
        self._chk(self.L.chd_phys_solve(self.h, _ptr(samples), _ptr(frames), _ptr(success), _ptr(sstat), _ptr(siter)))
        return dict(samples=samples, frames=frames, success=success, stage_status=sstat, stage_iters=siter)

    def sample(self):
        B, d = self.B, self.dims
        out = np.zeros((B, d["frames_out_max"], 6 + 7 * self.n_ee_max))
        frames = np.zeros(B, np.int32)
        self._chk(self.L.chd_phys_sample(self.h, _ptr(out), _ptr(frames)))
        return out, frames

    # ---- instrumentation -----------------------------------------------------------------------
    def launch_count(self) -> int:
        return int(self.L.chd_phys_launch_count(self.h))

    def h2d_bytes(self) -> int:
        return int(self.L.chd_phys_h2d_bytes(self.h))

    def reset(self):
        self._chk(self.L.chd_phys_reset(self.h))

    def set_timing(self, on: bool):
        self.L.chd_phys_set_timing(self.h, int(on))

    def kernel_times(self, reset=False):
        ms, cnt = np.zeros(8), np.zeros(8, np.int64)
        self.L.chd_phys_kernel_times(self.h, _ptr(ms), _ptr(cnt), int(reset))
        names = ["eval", "kkt", "linesearch", "init", "sample"]
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(names)}

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError("libchd call failed with code %d" % rc)


SOLUTION_FILES = ("sol_out_no_dynamics.txt", "sol_out_dynamics.txt", "sol_out_durations.txt")


def write_outputs(out: dict, i: int, problem: PhysProblem, out_dir: str, n_ee_max: Optional[int] = None) -> None:
    """The four files `phys_optim` leaves in --out_dir (phys_optim.cpp:63-153, 756-761) for sequence i of a `solve()` result."""
    import os
    from .io_formats import write_solution, write_success_log
    n_ee = problem.n_ee
    ne_max = n_ee_max if n_ee_max is not None else (out["samples"].shape[-1] - 6) // 7
    nf = int(out["frames"][i])
    # strip the padding columns of a mixed n_ee batch
    cols = list(range(6)) + [6 + 3 * e + d for e in range(n_ee) for d in range(3)] + \
        [6 + 3 * ne_max + 3 * e + d for e in range(n_ee) for d in range(3)] + [6 + 6 * ne_max + e for e in range(n_ee)]
    for snap, name in enumerate(SOLUTION_FILES):
        write_solution(os.path.join(out_dir, name), problem.dt, out["samples"][snap, i, :nf][:, cols], n_ee)
    write_success_log(os.path.join(out_dir, "success_log.txt"), out["success"][i, 0], out["success"][i, 1])


def master_row_slices(batch: PhysBatch, i: int, lay: Optional[dict] = None):
    """[(set type name, start, stop)] of sequence i's master rows, in master order."""
    lay = lay or batch.layout()
    m = int(batch.sizes[i, 1])
    rs = lay["row_set"][i, :m]
    out, a = [], 0
    for r in range(1, m + 1):
        if r == m or rs[r] != rs[a]:
            out.append((SET_NAMES[int(rs[a])], a, r))
            a = r
    return out
