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
import dataclasses
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .io_formats import PhysProblem

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

STAGES = {"1.1": 0, "1.2": 1, "2.1": 2, "2.2": 3, "3": 4, "4": 5}
SET_NAMES = {0: "acc", 1: "terrain", 2: "rom", 3: "dyn", 4: "force", 5: "heel", 6: "height", 7: "tottime", 8: "durpos"}
# The unweighted cost terms of `PhysBatch.cost_terms` / `solve(cost_terms=True)`, in column order (chd_phys_cost_terms):
# data fit, velocity smoothing and acceleration smoothing of the base position, the base orientation and the feet, then
# the change of the phase durations.
COST_TERMS = ("data_lin", "data_ang", "data_ee", "vel_lin", "vel_ang", "vel_ee", "acc_lin", "acc_ang", "acc_ee", "dur")
DEFAULT_WEIGHTS = (0.4, 1.7, 0.3, 0.1, 0.1)   # w_com_lin, w_com_ang, w_ee, w_smooth, w_dur (phys_optim.cpp:27-31)
# The values of `SolverOptions.last_stage`, named after the SaveSolution snapshot each one ends with (SOLUTION_FILES).
LAST_STAGES = ("no_dynamics", "dynamics", "durations")
SNAPSHOT_STAGES = ("1.2", "2.2", "3")         # the stage after which each snapshot is taken (stage 4 replaces 3's)


@dataclasses.dataclass(frozen=True)
class SolverOptions:
    """Solver options of one clip (chd_phys_solver_options).  The defaults are the reference's solve.

    `tol`, `constr_viol_tol`, `dual_inf_tol`, `compl_inf_tol`: IPOPT's termination tolerances of every stage (a stage
    converges when the scaled NLP error is within `tol` and the unscaled constraint violation, dual infeasibility and
    complementarity within the other three); each must be finite and > 0.
    `max_iter`: the iteration cap of stages 1.1, 1.2, 2.1, 2.2, 3, 4; 0 keeps the stage's own (7000, 7000, 7000, 2500,
    2000, 7000).  A capped stage ends with status -1 and the schedule goes on.
    `last_stage`: "no_dynamics" stops after stage 1.2, "dynamics" after stage 2.2, "durations" runs the whole schedule.
    The stages a clip does not run report status -9 and 0 iterations, and the snapshots it does not take are NaN."""
    tol: float = 1e-3
    constr_viol_tol: float = 1e-4
    dual_inf_tol: float = 1.0
    compl_inf_tol: float = 1e-4
    max_iter: Tuple[int, ...] = (0, 0, 0, 0, 0, 0)
    last_stage: str = "durations"

    def __post_init__(self):
        if self.last_stage not in LAST_STAGES:
            raise ValueError("last_stage: one of %s, not %r" % (", ".join(LAST_STAGES), self.last_stage))
        if len(self.max_iter) != 6:
            raise ValueError("max_iter: one cap for each of the six stages, not %r" % (self.max_iter,))
        object.__setattr__(self, "max_iter", tuple(int(k) for k in self.max_iter))


def sample_stride(n_ee_max: int) -> int:
    """Columns of a SaveSolution sample row (phys_optim.cpp:63-143) of a batch with up to n_ee_max end-effectors:
    base_lin (3), base_ang in degrees (3), foot positions (3 n_ee_max), foot forces (3 n_ee_max), contact flags (n_ee_max)."""
    return 6 + 7 * n_ee_max


def sample_columns(n_ee: int, n_ee_max: int):
    """(base, pos, frc, flag): column indices of the base (6), foot positions (3 n_ee), foot forces (3 n_ee) and contact
    flags (n_ee) of the first n_ee end-effectors in a sample row padded for n_ee_max (`sample_stride`)."""
    return (np.arange(6), np.arange(6, 6 + 3 * n_ee), np.arange(6 + 3 * n_ee_max, 6 + 3 * n_ee_max + 3 * n_ee),
            np.arange(6 + 6 * n_ee_max, 6 + 6 * n_ee_max + n_ee))


# Every per-clip result a solve can return: name -> (dtype, shape), "N" marking the clip axis ("fo": SaveSolution frames
# of the longest clip, "stride": `sample_stride`).  The batch, the queue and the merges of `chd.parallel` allocate,
# reorder, concatenate and pack results through the functions below, so that no caller needs a field's clip axis.
RESULT_FIELDS = {
    "samples": (np.float64, (3, "N", "fo", "stride")),   # the three SaveSolution snapshots (SOLUTION_FILES)
    "frames": (np.int32, ("N",)),
    "success": (np.int32, ("N", 2)),                     # dynamics, durations (success_log.txt)
    "stage_status": (np.int32, (6, "N")),
    "stage_iters": (np.int32, (6, "N")),
    "stage_stats": (np.float64, (6, "N", 4)),            # `PhysBatch.stage_stats`
    "cost_terms": (np.float64, ("N", len(COST_TERMS))),
    "solved": (np.bool_, ("N",)),
}
SOLVE_KEYS = ("samples", "frames", "success", "stage_status", "stage_iters")   # chd_phys_solve's outputs, in its order


def clip_axis(key: str) -> int:
    """The clip axis of result field `key`."""
    return RESULT_FIELDS[key][1].index("N")


def result_arrays(n: int, keys, fo: int = 0, stride: int = 0) -> dict:
    """Zeroed arrays of the result fields `keys` for n clips."""
    size = dict(N=n, fo=fo, stride=stride)
    return {k: np.zeros([size.get(s, s) for s in RESULT_FIELDS[k][1]], RESULT_FIELDS[k][0]) for k in keys}


def take_clips(res: dict, idx) -> dict:
    """Every field of `res` for the clips `idx` (an index array: selects or reorders)."""
    return {k: np.take(v, idx, axis=clip_axis(k)) for k, v in res.items()}


def concat_results(parts) -> dict:
    """Results of consecutive batches as one, clips in batch order; `samples` padded to the largest fo."""
    fo = max((p["samples"].shape[2] for p in parts if "samples" in p), default=0)
    pad = lambda k, v: np.pad(v, ((0, 0), (0, 0), (0, fo - v.shape[2]), (0, 0))) if k == "samples" else v
    return {k: np.concatenate([pad(k, p[k]) for p in parts], axis=clip_axis(k)) for k in parts[0]}


def _clips_first(res: dict, key: str) -> np.ndarray:
    """View of field `key` of `res` with its clip axis first."""
    return np.moveaxis(res[key], clip_axis(key), 0)


def pack_rows(res: dict, keys, idx, width: Optional[int] = None) -> np.ndarray:
    """Fields `keys` of the clips `idx` as one float64 row per clip: the fields side by side in the order of `keys`, each
    in C order with its clip axis removed; zero-padded to `width` columns.  Exact: int32 values and -0.0 pass through
    float64 unchanged, and `unpack_rows` writes them back."""
    idx = np.asarray(idx, np.int64)
    blocks = [_clips_first(res, k)[idx] for k in keys]
    cols = [int(np.prod(b.shape[1:])) for b in blocks]
    rows = np.zeros((len(idx), sum(cols) if width is None else width))
    c = 0
    for b, w in zip(blocks, cols):
        rows[:, c:c + w] = b.reshape(len(idx), w)
        c += w
    return rows


def unpack_rows(rows: np.ndarray, res: dict, keys, idx) -> None:
    """Writes rows packed by `pack_rows(..., keys, ...)` into the clips `idx` of the arrays of `res`; columns after the
    fields are ignored."""
    idx = np.asarray(idx, np.int64)
    c = 0
    for k in keys:
        dst = _clips_first(res, k)
        w = int(np.prod(dst.shape[1:]))
        dst[idx] = rows[:, c:c + w].reshape((len(idx),) + dst.shape[1:])
        c += w


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


class _SolverOptions(C.Structure):
    _fields_ = [("tol", C.c_double), ("constr_viol_tol", C.c_double), ("dual_inf_tol", C.c_double),
                ("compl_inf_tol", C.c_double), ("max_iter", C.c_int32 * 6), ("last_stage", C.c_int32)]

    @classmethod
    def of(cls, o: SolverOptions) -> "_SolverOptions":
        return cls(o.tol, o.constr_viol_tol, o.dual_inf_tol, o.compl_inf_tol, (C.c_int32 * 6)(*o.max_iter),
                   LAST_STAGES.index(o.last_stage))

    def value(self) -> SolverOptions:
        return SolverOptions(self.tol, self.constr_viol_tol, self.dual_inf_tol, self.compl_inf_tol, tuple(self.max_iter),
                             LAST_STAGES[self.last_stage])


class _Options(C.Structure):
    _fields_ = [("stage3_band_above", C.c_int32), ("clip_weights", C.POINTER(_Weights)),
                ("clip_options", C.POINTER(_SolverOptions))]


def clip_weights(weights, n: int) -> Optional[np.ndarray]:
    """`weights` as the batch classes take it: one 5-tuple (w_com_lin, w_com_ang, w_ee, w_smooth, w_dur) for every
    problem -> None, or one 5-tuple per problem -> an (n, 5) array.  Any other shape raises ValueError; the library
    refuses a weight that is negative or not finite."""
    w = np.asarray(weights, dtype=np.float64)
    if w.shape == (5,):
        return None
    if w.shape != (n, 5):
        raise ValueError("weights: one 5-tuple, or one 5-tuple per problem (%d), not an array of shape %s" % (n, w.shape))
    return w


def clip_options(options, n: int) -> Optional[List[SolverOptions]]:
    """`options` as the batch classes take it: None -> None (the library's defaults), one `SolverOptions` -> n copies
    of it, or one per problem.  Anything else raises ValueError; the library refuses a bad tolerance or cap."""
    if options is None:
        return None
    if isinstance(options, SolverOptions):
        return [options] * n
    options = list(options)
    if len(options) != n or not all(isinstance(o, SolverOptions) for o in options):
        raise ValueError("options: one SolverOptions, or one per problem (%d)" % n)
    return options


def _create_args(weights, n: int, stage3_band_above: Optional[int], order=None, options=None):
    """(weights argument, options argument, buffers to keep alive) of chd_phys_batch_create / chd_phys_queue_create;
    `order`: problem i of the call is problems[order[i]]."""
    per, per_opt = clip_weights(weights, n), clip_options(options, n)
    band = -1 if stage3_band_above is None else int(stage3_band_above)   # outside -1..96: refused by the library (-1)
    if order is not None:
        per = per[order] if per is not None else None
        per_opt = [per_opt[i] for i in order] if per_opt is not None else None
    w = _Weights(*[float(x) for x in weights]) if per is None else None
    warr = None if per is None else (_Weights * n)(*[_Weights(*[float(x) for x in row]) for row in per])
    oarr = None if per_opt is None else (_SolverOptions * n)(*[_SolverOptions.of(o) for o in per_opt])
    opt = None
    if stage3_band_above is not None or warr is not None or oarr is not None:
        opt = _Options(band, None if warr is None else C.cast(warr, C.POINTER(_Weights)),
                       None if oarr is None else C.cast(oarr, C.POINTER(_SolverOptions)))
    return (None if w is None else C.byref(w)), (None if opt is None else C.byref(opt)), (w, warr, oarr, opt)


class _Dims(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("batch", "n_max", "m_max", "slots_max", "n_splines", "p_max", "sets_max",
                                          "na_max", "nb_max", "w_max", "frames_out_max")]


_vp, _i32, _i64, _int, _f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_int, C.c_double

# chd_phys_claim_fn: (ctx, want, *first) -> k; passed to chd_phys_queue_set_claim as c_void_p (C.cast)
CLAIM_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32))

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
    "chd_phys_get_stage_weights": (_int, [_vp, _vp]),
    "chd_phys_get_solver_options": (_int, [_vp, C.POINTER(_SolverOptions)]),
    "chd_phys_cost_terms": (_int, [_vp, _vp]),
    "chd_phys_set_cost_terms_out": (_int, [_vp, _vp]),
    "chd_phys_solve_stage": (_int, [_vp, _i32, _i32, _vp, _vp, _vp]),
    "chd_phys_solve": (_int, [_vp] * 6),
    "chd_phys_sample": (_int, [_vp, _vp, _vp]),
    "chd_phys_sample_device": (_int, [_vp, _vp, _vp]),
    "chd_phys_launch_count": (_i64, [_vp]),
    "chd_phys_h2d_bytes": (_i64, [_vp]),
    "chd_phys_reset": (_int, [_vp]),
    "chd_phys_kernel_times": (_int, [_vp, _vp, _vp, _int]),
    "chd_phys_set_timing": (_int, [_vp, _int]),
    "chd_phys_queue_create": (_int, [C.POINTER(_Problem), _i32, _i32, C.POINTER(_Weights), _i32, C.POINTER(_Options),
                                     C.POINTER(_vp)]),
    "chd_phys_queue_solve": (_int, [_vp] * 7),
    "chd_phys_queue_set_claim": (_int, [_vp] * 3),
    "chd_contact_create": (_int, [_vp, _vp, _vp, C.c_float, _i32, C.POINTER(_vp)]),
    "chd_contact_destroy": (None, [_vp]),
    "chd_contact_forward": (_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "chd_contact_forward_device": (_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "chd_contact_preprocess": (_int, [_vp, _vp, _vp, _i32, _f64, _f64, _vp, _vp]),
    "chd_contact_score_device": (_int, [_vp, _vp, _i32, _i32, _vp, _vp, C.c_float, _vp, _vp, _vp, _vp]),
    "chd_contact_detect": (_int, [_vp, _vp, _vp, _i32, _f64, _f64, _vp, _vp, C.c_float, _vp, _vp, _vp, _vp, _vp]),
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


class _Handle:
    """A libchd phys handle (`h`, from chd_phys_batch_create or chd_phys_queue_create): its dims, its release and its
    instrumentation.  `KERNELS`: the kernel groups of chd_phys_kernel_times the handle reports."""
    KERNELS = ("eval", "kkt", "linesearch", "init", "sample")

    def _read_dims(self):
        d = _Dims()
        self.L.chd_phys_get_dims(self.h, C.byref(d))
        self.dims = {k: getattr(d, k) for k, _ in _Dims._fields_}

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

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError("libchd call failed with code %d" % rc)

    def launch_count(self) -> int:
        return int(self.L.chd_phys_launch_count(self.h))

    def h2d_bytes(self) -> int:
        """Bytes uploaded so far: the tables at creation, and in a queue the records of every admitted clip."""
        return int(self.L.chd_phys_h2d_bytes(self.h))

    def set_timing(self, on: bool):
        self.L.chd_phys_set_timing(self.h, int(on))

    def kernel_times(self, reset=False):
        ms, cnt = np.zeros(8), np.zeros(8, np.int64)
        self.L.chd_phys_kernel_times(self.h, _ptr(ms), _ptr(cnt), int(reset))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.KERNELS)}


class PhysBatch(_Handle):
    """`weights`: one 5-tuple (w_com_lin, w_com_ang, w_ee, w_smooth, w_dur) for every sequence, or one per sequence
    (`clip_weights`).  `options`: one `SolverOptions` for every sequence, or one per sequence (`clip_options`); None:
    the defaults.  `stage3_band_above`: sequences with more phase-duration variables than this carry their switch
    times as banded KKT unknowns, which lets stage 3 run beyond the 96 the dense border holds (0 bands every sequence;
    None: none)."""

    def __init__(self, problems: Sequence[PhysProblem], weights=DEFAULT_WEIGHTS, device: int = -1,
                 host_only: bool = False, stage3_band_above: Optional[int] = None, options=None):
        self.L = load_lib()
        self.problems = list(problems)
        B = len(self.problems)
        arr, self._keep = make_problem_array(self.problems)
        w, opt, _ = _create_args(weights, B, stage3_band_above, options=options)
        h = C.c_void_p()
        dev = -2 if host_only else device
        rc = self.L.chd_phys_batch_create(arr, B, w, dev, opt, C.byref(h))
        if rc != 0:
            raise RuntimeError("chd_phys_batch_create failed with code %d (no CUDA device? no CPU fallback exists)" % rc)
        self.h = h
        self.host_only = host_only
        self._read_dims()
        self.B = B
        sz = np.zeros((B, 6), dtype=np.int32)
        self.L.chd_phys_get_sizes(self.h, _ptr(sz))
        self.sizes = sz  # n, m, nslots, Na, nb, w
        self.n_ee_max = max(p.n_ee for p in self.problems)

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

    def stage_weights(self) -> np.ndarray:
        """(B, 6, 10): the cost weights of every sequence's six stages: w_data, w_vel, w_acc (base lin, base ang, feet
        each) and w_dur, so that a stage's cost is `cost_terms() @ stage_weights()[:, stage]` row by row."""
        out = np.zeros((self.B, 6, 10))
        self._chk(self.L.chd_phys_get_stage_weights(self.h, _ptr(out)))
        return out

    def solver_options(self) -> List[SolverOptions]:
        """Every sequence's `SolverOptions` as the solver uses them, each cap of 0 resolved to the stage's own."""
        out = (_SolverOptions * self.B)()
        self._chk(self.L.chd_phys_get_solver_options(self.h, out))
        return [o.value() for o in out]

    def cost_terms(self) -> np.ndarray:
        """(B, 10): the unweighted cost terms at the current x, columns `COST_TERMS` (chd_phys_cost_terms)."""
        out = np.zeros((self.B, len(COST_TERMS)))
        self._chk(self.L.chd_phys_cost_terms(self.h, _ptr(out)))
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

    def solve(self, cost_terms: bool = False) -> dict:
        """Full staged schedule.  Returns the three SaveSolution snapshots, frame counts, success flags; with
        `cost_terms` also `cost_terms` (B, 10): the unweighted cost terms (`COST_TERMS`) of every final iterate."""
        out = result_arrays(self.B, SOLVE_KEYS, self.dims["frames_out_max"], sample_stride(self.n_ee_max))
        with _terms_out(self, self.B, cost_terms) as terms:
            self._chk(self.L.chd_phys_solve(self.h, *[_ptr(out[k]) for k in SOLVE_KEYS]))
        if terms is not None:
            out["cost_terms"] = terms
        return out

    def sample(self):
        B, d = self.B, self.dims
        out = np.zeros((B, d["frames_out_max"], sample_stride(self.n_ee_max)))
        frames = np.zeros(B, np.int32)
        self._chk(self.L.chd_phys_sample(self.h, _ptr(out), _ptr(frames)))
        return out, frames

    def reset(self):
        self._chk(self.L.chd_phys_reset(self.h))


class _terms_out:
    """Points the handle's cost-terms output (chd_phys_set_cost_terms_out) at a fresh (n, 10) array for one solve, and
    back to NULL afterwards, so that the library never holds a pointer into freed memory."""

    def __init__(self, obj, n: int, on: bool):
        self.obj, self.terms = obj, (result_arrays(n, ("cost_terms",))["cost_terms"] if on else None)

    def __enter__(self):
        if self.terms is not None:
            self.obj._chk(self.obj.L.chd_phys_set_cost_terms_out(self.obj.h, _ptr(self.terms)))
        return self.terms

    def __exit__(self, *exc):
        if self.terms is not None:
            self.obj.L.chd_phys_set_cost_terms_out(self.obj.h, None)


class PhysQueue(_Handle):
    """Any number of clips solved through `slots` device slots: a slot takes the next clip as soon as its clip has
    finished, so device memory scales with `slots` and the slowest clip's tail is paid once per queue rather than once
    per batch.  The clips enter in descending `chd.parallel.work_estimate` order (the longest first, so that the queue's
    final tail is short); `solve()` returns `PhysBatch.solve()`'s dict plus `stage_stats` (6, N, 4) and `solved` (N),
    in input order.  Each clip's results are those of a `PhysBatch` of the same clips (`stage3_band_above`: see
    `PhysBatch`).

    `claim`: a callable `want -> (first, k)` that decides which queue positions this queue solves
    (`chd_phys_queue_set_claim`): it is asked for `slots` positions when a solve starts and for as many as there are
    finished slots at every refill check point, and hands out the k consecutive positions first .. first + k - 1
    (0 <= k <= want; fewer than asked: nothing is left).  Queue positions are the `work_estimate` order (`order`), which
    is the same in every process that holds the same problem list, so processes that share one source
    (`chd.parallel.StoreClaim`) split the clips between them.  Only the clips handed out are solved: `solved` marks
    them, the other clips' rows stay zero.

    `weights` and `options`: as `PhysBatch`'s, one per problem in input order (each clip keeps its own through every
    slot).  A clip that stops early (`SolverOptions.last_stage`) frees its slot for the next clip at once."""
    KERNELS = _Handle.KERNELS + ("admit",)

    def __init__(self, problems: Sequence[PhysProblem], slots: int, weights=DEFAULT_WEIGHTS, device: int = -1,
                 stage3_band_above: Optional[int] = None, claim=None, options=None):
        from .parallel import work_estimate
        self.L = load_lib()
        self.problems = list(problems)
        N = len(self.problems)
        # queue position k holds problems[order[k]]; stable, so equal estimates keep their input order
        self.order = np.argsort(-np.asarray(work_estimate(self.problems), dtype=np.float64), kind="stable")
        arr, self._keep = make_problem_array([self.problems[i] for i in self.order])
        w, opt, _ = _create_args(weights, N, stage3_band_above, self.order, options)
        h = C.c_void_p()
        rc = self.L.chd_phys_queue_create(arr, N, int(slots), w, device, opt, C.byref(h))
        if rc != 0:
            raise RuntimeError("chd_phys_queue_create failed with code %d" % rc)
        self.h = h
        self._read_dims()
        self.N, self.slots = N, self.dims["batch"]
        self.n_ee_max = max(p.n_ee for p in self.problems)
        self.claim, self._claimed, self._claim_error = claim, [], None
        self._claim_cb = None                  # the ctypes callback: alive as long as the handle holds it
        if claim is not None:
            self._claim_cb = CLAIM_FN(self._on_claim)
            rc = self.L.chd_phys_queue_set_claim(self.h, C.cast(self._claim_cb, C.c_void_p), None)
            if rc != 0:
                self.close()
                raise RuntimeError("chd_phys_queue_set_claim failed with code %d" % rc)

    def _on_claim(self, ctx, want, first):
        """chd_phys_claim_fn over `claim`: records the positions handed out; an exception in `claim` becomes -1 and is
        raised again by solve()."""
        try:
            f, k = (int(v) for v in self.claim(int(want)))
        except BaseException as e:            # must not cross the C frames
            self._claim_error = e
            return -1
        first[0] = f
        if k > 0:
            self._claimed.append((f, k))
        return k

    def solve(self, cost_terms: bool = False) -> dict:
        """Full staged schedule of every clip (with `claim`: of the clips it hands out); the same keys and shapes as
        `PhysBatch.solve()` for N sequences (`cost_terms` included), plus stage_stats (6, N, 4)
        (`PhysBatch.stage_stats`) and solved (N bools)."""
        N = self.N
        keys = SOLVE_KEYS + ("stage_stats",)      # chd_phys_queue_solve's outputs, in its order
        out = result_arrays(N, keys, self.dims["frames_out_max"], sample_stride(self.n_ee_max))
        self._claimed, self._claim_error = [], None
        with _terms_out(self, N, cost_terms) as terms:
            rc = self.L.chd_phys_queue_solve(self.h, *[_ptr(out[k]) for k in keys])
        if self._claim_error is not None:
            e, self._claim_error = self._claim_error, None
            raise RuntimeError("the claim source of the queue failed") from e
        self._chk(rc)
        solved = np.ones(N, bool)
        if self.claim is not None:
            solved[:] = False
            for f, k in self._claimed:
                solved[f:f + k] = True
        out["solved"] = solved
        if terms is not None:
            out["cost_terms"] = terms
        return take_clips(out, np.argsort(self.order))   # queue position of every input clip


SOLUTION_FILES = ("sol_out_no_dynamics.txt", "sol_out_dynamics.txt", "sol_out_durations.txt")


def snapshots_taken(out: dict, i: int) -> List[bool]:
    """Which of the three SaveSolution snapshots (SOLUTION_FILES) sequence i of a `solve()` result took: those whose
    stage ran (a snapshot after the clip's `last_stage` is NaN)."""
    return [int(out["stage_status"][STAGES[s], i]) != -9 for s in SNAPSHOT_STAGES]


def write_outputs(out: dict, i: int, problem: PhysProblem, out_dir: str, n_ee_max: Optional[int] = None) -> None:
    """The files `phys_optim` leaves in --out_dir (phys_optim.cpp:63-153, 756-761) for sequence i of a `solve()` result:
    the solution file of every snapshot the clip took (all three unless it stopped early, `SolverOptions.last_stage`)
    and success_log.txt, whose flag is 0 for a stage that did not run."""
    import os
    from .io_formats import write_solution, write_success_log
    n_ee = problem.n_ee
    ne_max = n_ee_max if n_ee_max is not None else (out["samples"].shape[-1] - 6) // 7
    nf = int(out["frames"][i])
    cols = np.concatenate(sample_columns(n_ee, ne_max))     # strips the padding columns of a mixed n_ee batch
    for snap, (name, taken) in enumerate(zip(SOLUTION_FILES, snapshots_taken(out, i))):
        if taken:
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
