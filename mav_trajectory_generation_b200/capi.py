"""ctypes binding of the C-ABI (include/mtg_b200.h) for tests, bench.py and smoke().

This is plumbing only: device memory comes from torch tensors (data_ptr), streams from
torch.cuda.  There is NO fallback: if libmtg_b200.so is missing or no sm_90 device is present
every entry point raises.
"""
import ctypes as C
import os

import numpy as np

from . import _build

MTG_OK = 0
KERNEL_WAYPOINT, KERNEL_GENERIC, KERNEL_NOFREE = 1, 2, 3
STATUS_BAD_TIME, STATUS_NOT_SPD = 1, 2
OPT_WAYPOINT_VARIANT = 1
OPT_RING_DEPTH, OPT_CTAS_PER_SM, OPT_STAGGER_US, OPT_DYNAMIC_TILES, OPT_CHUNK_BLOCKS = 2, 3, 4, 5, 6
OPT_GENERIC_VARIANT = 7
OPT_MELLINGER_UNFUSED = 8
OPT_TMA_INPUTS = 9
OPT_EARLY_REFILL = 10
OPT_CHUNK_WARPS = 11
OPT_L2_HINTS = 12

EXPORTED_SYMBOLS = [
    "mtg_create", "mtg_destroy", "mtg_last_error", "mtg_launch_count", "mtg_device_is_sm90",
    "mtg_problem_layout", "mtg_solve_linear_batch_f64", "mtg_coeffs_from_constraints_batch_f64",
    "mtg_compute_cost_batch_f64", "mtg_solve_linear_batch_host_f64",
    "mtg_coeffs_from_constraints_batch_host_f64", "mtg_compute_cost_batch_host_f64",
    "mtg_host_alloc", "mtg_host_free", "mtg_device_alloc", "mtg_device_free", "mtg_memcpy_h2d",
    "mtg_memcpy_d2h", "mtg_stream_synchronize", "mtg_version", "mtg_set_option",
    "mtg_solve_waypoints_nfabian_batch_f64", "mtg_solve_waypoints_nfabian_batch_host_f64",
    "mtg_cost_gradient_mellinger_batch_f64", "mtg_evaluate_batch_f64", "mtg_evaluate_range_batch_f64",
    "mtg_cost_gradient_mellinger_batch_host_f64", "mtg_evaluate_range_batch_host_f64",
    "mtg_memcpy_d2d", "mtg_ipc_export", "mtg_ipc_import", "mtg_ipc_close",
    "mtg_max_magnitude_batch_f64", "mtg_time_objective_batch_f64", "mtg_max_magnitude_batch_host_f64",
    "mtg_time_objective_batch_host_f64", "mtg_scale_to_constraints_batch_f64",
    "mtg_scale_times_with_violation_batch_f64", "mtg_scale_to_constraints_batch_host_f64",
    "mtg_scale_times_with_violation_batch_host_f64", "mtg_input_feasibility_batch_f64",
    "mtg_input_feasibility_batch_host_f64", "mtg_half_plane_feasibility_batch_f64",
    "mtg_half_plane_feasibility_batch_host_f64", "mtg_input_feasibility_recursive_batch_f64",
    "mtg_input_feasibility_recursive_batch_host_f64", "mtg_input_feasibility_sampling_batch_f64",
    "mtg_input_feasibility_sampling_batch_host_f64", "mtg_sample_flat_states_batch_f64",
    "mtg_sample_flat_state_at_time_batch_f64", "mtg_sample_flat_states_batch_host_f64",
    "mtg_sample_flat_state_at_time_batch_host_f64", "mtg_optimize_time_mellinger_batch_f64",
    "mtg_optimize_time_mellinger_batch_host_f64", "mtg_optimize_time_batch_f64", "mtg_optimize_time_batch_host_f64",
]
# mav_msgs::EigenTrajectoryPoint as one record of MTG_FLAT_STATE_DOUBLES doubles: the slice of each field
FLAT_STATE_DOUBLES = 25
FLAT_STATE_FIELDS = {
    "position_W": slice(0, 3), "velocity_W": slice(3, 6), "acceleration_W": slice(6, 9), "jerk_W": slice(9, 12),
    "snap_W": slice(12, 15), "orientation_W_B": slice(15, 19),  # (w, x, y, z)
    "angular_velocity_W": slice(19, 22), "angular_acceleration_W": slice(22, 25),
}
TIME_COST_SQUARED, TIME_COST_RICHTER = 0, 1
STATUS_FEAS_CAPACITY = 4
# InputFeasibilityResult
(FEAS_FEASIBLE, FEAS_INDETERMINABLE, FEAS_THRUST_HIGH, FEAS_THRUST_LOW, FEAS_VELOCITY, FEAS_ROLL_PITCH_RATES,
 FEAS_YAW_RATES, FEAS_YAW_ACC) = range(8)
FEAS_NAMES = ("Feasible", "Indeterminable", "InfeasibleThrustHigh", "InfeasibleThrustLow", "InfeasibleVelocity",
              "InfeasibleRollPitchRates", "InfeasibleYawRates", "InfeasibleYawAcc")
# InputConstraintType order: the bit of mtg_input_constraints::present
INPUT_LIMITS = ("f_min", "f_max", "v_max", "omega_xy_max", "omega_z_max", "omega_z_dot_max")
# Gravity of the host mirror's InputConstraints / FeasibilityAnalytic default (the reference uses mav_msgs::kGravity;
# mav_comm is not part of this project, so this value was not checked against it).
GRAVITY = 9.81


class MtgProblem(C.Structure):
    _fields_ = [("N", C.c_int32), ("r", C.c_int32), ("K", C.c_int32), ("D", C.c_int32),
                ("fixed_mask", C.POINTER(C.c_uint8))]


class MtgMellingerParams(C.Structure):
    _fields_ = [("f_abs", C.c_double), ("f_rel", C.c_double), ("x_rel", C.c_double), ("x_abs", C.c_double),
                ("initial_stepsize_rel", C.c_double), ("max_iterations", C.c_int32)]


# nlopt_result values of mtg_optimize_time_mellinger_batch_f64
(OPTIMIZE_RESULT_FAILURE, OPTIMIZE_RESULT_ROUNDOFF_LIMITED, OPTIMIZE_RESULT_SUCCESS, OPTIMIZE_RESULT_FTOL_REACHED, OPTIMIZE_RESULT_XTOL_REACHED,
 OPTIMIZE_RESULT_MAXEVAL_REACHED) = (-1, -4, 1, 3, 4, 5)
# NonlinearOptimizationParameters' defaults
MELLINGER_DEFAULTS = dict(f_abs=-1.0, f_rel=0.05, x_rel=-1.0, x_abs=-1.0, initial_stepsize_rel=0.1,
                          max_iterations=3000)


def mellinger_params(**kw):
    """mtg_mellinger_params: MELLINGER_DEFAULTS updated by kw."""
    unknown = set(kw) - set(MELLINGER_DEFAULTS)
    if unknown:
        raise ValueError(f"unknown Mellinger parameters {sorted(unknown)}")
    v = dict(MELLINGER_DEFAULTS, **kw)
    return MtgMellingerParams(float(v["f_abs"]), float(v["f_rel"]), float(v["x_rel"]), float(v["x_abs"]),
                              float(v["initial_stepsize_rel"]), int(v["max_iterations"]))


class MtgLayout(C.Structure):
    _fields_ = [("n_all", C.c_int32), ("n_fixed", C.c_int32), ("n_free", C.c_int32), ("kernel", C.c_int32)]


class MtgSoftConstraint(C.Structure):
    _fields_ = [("derivative", C.c_int32), ("max_value", C.c_double)]


class MtgTimeObjective(C.Structure):
    _fields_ = [("time_cost", C.c_int32), ("time_penalty", C.c_double), ("soft_constraint_weight", C.c_double),
                ("maximum_cost", C.c_double), ("n_constraints", C.c_int32),
                ("constraints", C.POINTER(MtgSoftConstraint))]


class MtgInputConstraints(C.Structure):
    _fields_ = [("present", C.c_uint32)] + [(n, C.c_double) for n in INPUT_LIMITS] + \
               [("gravity", C.c_double), ("min_section_time", C.c_double)]


def default_input_limits(gravity=GRAVITY):
    """InputConstraints::setDefaultValues(): every limit present."""
    return dict(f_min=0.5 * gravity, f_max=1.5 * gravity, v_max=3.0, omega_xy_max=np.pi / 2, omega_z_max=np.pi / 2,
                omega_z_dot_max=2.0 * np.pi)


def input_constraints(limits, min_section_time=0.05, gravity=GRAVITY):
    """mtg_input_constraints from {name: value} (names of INPUT_LIMITS; a missing name is an absent limit).  The values
    are passed as given: they are the final limits."""
    unknown = set(limits) - set(INPUT_LIMITS)
    if unknown:
        raise ValueError(f"unknown input constraints {sorted(unknown)}")
    c = MtgInputConstraints()
    for q, n in enumerate(INPUT_LIMITS):
        if n in limits:
            c.present |= 1 << q
            setattr(c, n, float(limits[n]))
    c.gravity = float(gravity)
    c.min_section_time = float(min_section_time)
    return c


class MtgHalfPlane(C.Structure):
    _fields_ = [("point", C.c_double * 3), ("normal", C.c_double * 3)]


MAX_HALF_PLANES = 64


def _normalized(v):
    """Eigen's normalized() of a 3-vector: v / sqrt((v0 v0 + v1 v1) + v2 v2), each step rounded once."""
    v = np.asarray(v, dtype=np.float64)
    sq = np.float64(0.0)
    for x in v:
        sq = sq + x * x
    if not sq > 0.0:
        return v.copy()
    return v / np.sqrt(sq)


def half_plane(point, normal):
    """HalfPlane(point, normal): [1][6] float64 (point, then the normal normalised as the reference does)."""
    point = np.asarray(point, dtype=np.float64).reshape(3)
    normal = np.asarray(normal, dtype=np.float64).reshape(3)
    if not np.linalg.norm(normal) > 0.0:
        raise ValueError("invalid normal")
    return np.concatenate([point, _normalized(normal)])[None, :]


def half_plane_from_points(a, b, c):
    """HalfPlane(a, b, c): the plane through a, b and c with normal (b - a) x (c - a), normalised; [1][6] float64."""
    a, b, c = (np.asarray(x, dtype=np.float64).reshape(3) for x in (a, b, c))
    if np.array_equal(a, b) or np.array_equal(a, c):
        raise ValueError("the three points must differ from the first")
    u, v = b - a, c - a
    n = np.array([u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]])
    return np.concatenate([a, _normalized(n)])[None, :]


def bounding_box(center, size):
    """HalfPlane::createBoundingBox(center, size): for each axis, (center - size / 2, +e_axis) then
    (center + size / 2, -e_axis); [6][6] float64."""
    center = np.asarray(center, dtype=np.float64).reshape(3)
    size = np.asarray(size, dtype=np.float64).reshape(3)
    lo, hi = center - size / 2.0, center + size / 2.0
    rows = []
    for axis in range(3):
        e = np.zeros(3)
        e[axis] = 1.0
        rows.append(half_plane(lo, e))
        rows.append(half_plane(hi, -e))
    return np.concatenate(rows)


def half_plane_array(planes):
    """An MtgHalfPlane array (and its length) from [P][6] float64 rows: point, normal."""
    planes = np.asarray(planes, dtype=np.float64).reshape(-1, 6)
    arr = (MtgHalfPlane * max(len(planes), 1))()
    for i, row in enumerate(planes):
        arr[i].point[:] = [float(x) for x in row[:3]]
        arr[i].normal[:] = [float(x) for x in row[3:]]
    return arr, len(planes)


def time_objective_params(time_cost=TIME_COST_SQUARED, time_penalty=500.0, soft_constraint_weight=100.0,
                          maximum_cost=1e12, constraints=()):
    """mtg_time_objective for `constraints` = [(derivative, max_value), ...] (reference defaults otherwise)."""
    arr = (MtgSoftConstraint * max(len(constraints), 1))(*[MtgSoftConstraint(int(k), float(v)) for k, v in constraints])
    obj = MtgTimeObjective(int(time_cost), float(time_penalty), float(soft_constraint_weight), float(maximum_cost),
                           len(constraints), C.cast(arr, C.POINTER(MtgSoftConstraint)))
    obj._keep = arr  # the array must outlive the call
    return obj


_lib = None


def load():
    """Load libmtg_b200.so (built in-tree by __graft_entry__.build()).  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_CUDA
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(the CUDA extension is the only compute path; there is no fallback)")
    L = C.CDLL(path)
    vp, i64, dp = C.c_void_p, C.c_int64, C.c_void_p
    L.mtg_create.restype = C.c_int
    L.mtg_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.mtg_destroy.argtypes = [vp]
    L.mtg_destroy.restype = None
    L.mtg_last_error.restype = C.c_char_p
    L.mtg_last_error.argtypes = [vp]
    L.mtg_launch_count.restype = i64
    L.mtg_launch_count.argtypes = [vp]
    L.mtg_device_is_sm90.argtypes = [vp]
    L.mtg_problem_layout.argtypes = [C.POINTER(MtgProblem), C.POINTER(MtgLayout), vp]
    L.mtg_solve_linear_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp, dp, vp]
    L.mtg_coeffs_from_constraints_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp, vp]
    L.mtg_compute_cost_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, vp]
    L.mtg_solve_linear_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp, dp]
    L.mtg_coeffs_from_constraints_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp]
    L.mtg_compute_cost_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp]
    L.mtg_host_alloc.restype = vp
    L.mtg_host_alloc.argtypes = [vp, C.c_uint64]
    L.mtg_host_free.argtypes = [vp, vp]
    L.mtg_device_alloc.restype = vp
    L.mtg_device_alloc.argtypes = [vp, C.c_uint64]
    L.mtg_device_free.argtypes = [vp, vp]
    L.mtg_memcpy_h2d.argtypes = [vp, vp, vp, C.c_uint64, vp]
    L.mtg_memcpy_d2h.argtypes = [vp, vp, vp, C.c_uint64, vp]
    L.mtg_stream_synchronize.argtypes = [vp, vp]
    L.mtg_memcpy_d2d.argtypes = [vp, vp, vp, C.c_uint64, vp]
    L.mtg_ipc_export.argtypes = [vp, vp, C.c_char_p, C.POINTER(C.c_uint64)]
    L.mtg_ipc_import.argtypes = [vp, C.c_char_p, C.c_uint64, C.POINTER(vp), C.POINTER(vp)]
    L.mtg_ipc_close.argtypes = [vp, vp]
    L.mtg_version.restype = C.c_int
    L.mtg_set_option.argtypes = [vp, C.c_int, C.c_int]
    L.mtg_evaluate_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_int32, C.c_double,
                                         C.c_double, C.c_int32, dp, vp]
    L.mtg_evaluate_range_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_double, C.c_double,
                                               C.c_double, C.c_int32, C.POINTER(C.c_int32), C.c_int32, dp, dp, dp, vp]
    L.mtg_cost_gradient_mellinger_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp, vp]
    L.mtg_cost_gradient_mellinger_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, dp]
    L.mtg_evaluate_range_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_double,
                                                    C.c_double, C.c_double, C.c_int32, C.POINTER(C.c_int32),
                                                    C.c_int32, dp, dp, dp]
    L.mtg_solve_waypoints_nfabian_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, i64, dp,
                                                             C.c_double, C.c_double, C.c_double, dp, dp, dp]
    L.mtg_solve_waypoints_nfabian_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, i64, dp,
                                                        C.c_double, C.c_double, C.c_double, dp, dp, dp, vp]
    i32p = C.POINTER(C.c_int32)
    L.mtg_max_magnitude_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_int32, i32p, dp, dp,
                                              dp, dp, vp]
    L.mtg_max_magnitude_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_int32, i32p,
                                                   dp, dp, dp, dp]
    L.mtg_time_objective_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp, C.POINTER(MtgTimeObjective),
                                               dp, dp, dp, dp, vp]
    L.mtg_time_objective_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dp,
                                                    C.POINTER(MtgTimeObjective), dp, dp, dp, dp]
    dbl = C.c_double
    L.mtg_scale_to_constraints_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, dbl, dbl, dp,
                                                     dp, dp, dp, dp, vp]
    L.mtg_scale_to_constraints_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, dbl, dbl,
                                                          dp, dp, dp, dp, dp]
    L.mtg_scale_times_with_violation_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dbl, dbl, dp, dp,
                                                           dp, dp, dp, vp]
    L.mtg_scale_times_with_violation_batch_host_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, dbl, dbl, dp,
                                                                dp, dp, dp, dp]
    L.mtg_input_feasibility_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp,
                                                  C.POINTER(MtgInputConstraints), dp, dp, dp, vp]
    L.mtg_input_feasibility_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp,
                                                       C.POINTER(MtgInputConstraints), dp, dp, dp]
    L.mtg_input_feasibility_recursive_batch_f64.argtypes = L.mtg_input_feasibility_batch_f64.argtypes
    L.mtg_input_feasibility_recursive_batch_host_f64.argtypes = L.mtg_input_feasibility_batch_host_f64.argtypes
    L.mtg_input_feasibility_sampling_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp,
                                                           C.POINTER(MtgInputConstraints), dbl, dp, dp, dp, vp]
    L.mtg_input_feasibility_sampling_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp,
                                                                C.POINTER(MtgInputConstraints), dbl, dp, dp, dp]
    L.mtg_half_plane_feasibility_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, C.c_int32,
                                                       C.POINTER(MtgHalfPlane), dp, dp, dp, dp, vp]
    L.mtg_half_plane_feasibility_batch_host_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp,
                                                            C.c_int32, C.POINTER(MtgHalfPlane), dp, dp, dp, dp]
    L.mtg_sample_flat_states_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, dbl, dbl, dbl,
                                                   C.c_int32, C.c_int32, dp, dp, dp, vp]
    L.mtg_sample_flat_states_batch_host_f64.argtypes = L.mtg_sample_flat_states_batch_f64.argtypes[:-1]
    L.mtg_sample_flat_state_at_time_batch_f64.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, i64, dp, dp, dp, dp,
                                                          dp, dp, vp]
    L.mtg_sample_flat_state_at_time_batch_host_f64.argtypes = L.mtg_sample_flat_state_at_time_batch_f64.argtypes[:-1]
    L.mtg_optimize_time_mellinger_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp,
                                                        C.POINTER(MtgMellingerParams), dbl, dbl, dp, dp, dp, dp, dp,
                                                        dp, dp, dp, dp, vp]
    L.mtg_optimize_time_mellinger_batch_host_f64.argtypes = L.mtg_optimize_time_mellinger_batch_f64.argtypes[:-1]
    L.mtg_optimize_time_batch_f64.argtypes = [vp, C.POINTER(MtgProblem), i64, dp, dp, C.POINTER(MtgTimeObjective),
                                              C.POINTER(MtgMellingerParams), dp, dp, dp, dp, dp, dp, dp, vp]
    L.mtg_optimize_time_batch_host_f64.argtypes = L.mtg_optimize_time_batch_f64.argtypes[:-1]
    for name in EXPORTED_SYMBOLS:
        getattr(L, name)  # AttributeError if the library does not export what the header declares
    _lib = L
    return L


class Problem:
    """A constraint topology: N, derivative_to_optimize r, K segments, D dimensions and the
    per-vertex fixed mask ([K+1][N/2], None = createRandomVertices topology)."""

    def __init__(self, N, r, K, D, fixed_mask=None):
        self.N, self.r, self.K, self.D = int(N), int(r), int(K), int(D)
        self._mask = None
        self.c = MtgProblem(self.N, self.r, self.K, self.D, None)
        if fixed_mask is not None:
            self._mask = np.ascontiguousarray(fixed_mask, dtype=np.uint8).reshape(self.K + 1, self.N // 2)
            self.c.fixed_mask = self._mask.ctypes.data_as(C.POINTER(C.c_uint8))
        lay = MtgLayout()
        slot = np.zeros(max(self.K * self.N, 1), dtype=np.int32)
        rc = load().mtg_problem_layout(C.byref(self.c), C.byref(lay), slot.ctypes.data)
        if rc != MTG_OK:
            raise ValueError(f"invalid problem N={N} r={r} K={K} D={D} (rc={rc})")
        self.n_all, self.n_fixed, self.n_free, self.kernel = lay.n_all, lay.n_fixed, lay.n_free, lay.kernel
        self.slot_col = slot[: self.K * self.N]

    @property
    def bytes_per_trajectory(self):
        """Algorithmic HBM bytes: seg_times + d_fixed in, coeffs out (SURVEY.md 8d)."""
        return 8 * (self.K + self.D * self.n_fixed) + 8 * self.K * self.D * self.N


class Solver:
    """One handle on one CUDA device (single caller)."""

    def __init__(self, device=0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.mtg_create(int(device), C.byref(h))
        if rc != MTG_OK:
            raise RuntimeError(f"mtg_create failed (rc={rc}): {self.lib.mtg_last_error(None).decode()}")
        self.h = h
        self.device = int(device)

    def close(self):
        if getattr(self, "h", None):
            self.lib.mtg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != MTG_OK:
            raise RuntimeError(f"{what} failed (rc={rc}): {self.lib.mtg_last_error(self.h).decode()}")

    def set_option(self, key, value):
        self._check(self.lib.mtg_set_option(self.h, int(key), int(value)), "mtg_set_option")

    @property
    def launch_count(self):
        return int(self.lib.mtg_launch_count(self.h))

    # ---- device-pointer path (torch CUDA tensors, float64, contiguous) --------------------
    def solve_linear(self, prob, seg_times, d_fixed, coeffs=None, d_free=None, status=None, stream=None):
        import torch
        B = seg_times.shape[0]
        assert seg_times.is_cuda and seg_times.dtype == torch.float64 and seg_times.is_contiguous()
        assert d_fixed.is_cuda and d_fixed.dtype == torch.float64 and d_fixed.is_contiguous()
        assert tuple(seg_times.shape) == (B, prob.K) and tuple(d_fixed.shape) == (B, prob.D, prob.n_fixed)
        if coeffs is None:
            coeffs = torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=seg_times.device)
        assert coeffs.is_contiguous() and tuple(coeffs.shape) == (B, prob.K, prob.D, prob.N)
        s = stream if stream is not None else torch.cuda.current_stream(seg_times.device).cuda_stream
        rc = self.lib.mtg_solve_linear_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(), coeffs.data_ptr(),
            d_free.data_ptr() if d_free is not None else None,
            status.data_ptr() if status is not None else None, s)
        self._check(rc, "mtg_solve_linear_batch_f64")
        return coeffs

    # ---- raw device pointers (peer memory imported with ipc_import has no torch tensor behind it) ----
    def solve_linear_ptr(self, prob, B, seg_times_ptr, d_fixed_ptr, coeffs_ptr, stream):
        rc = self.lib.mtg_solve_linear_batch_f64(self.h, C.byref(prob.c), int(B), int(seg_times_ptr), int(d_fixed_ptr),
                                                 int(coeffs_ptr), None, None, int(stream))
        self._check(rc, "mtg_solve_linear_batch_f64")

    def memcpy_d2d(self, dst_ptr, src_ptr, nbytes, stream):
        self._check(self.lib.mtg_memcpy_d2d(self.h, int(dst_ptr), int(src_ptr), int(nbytes), int(stream)), "mtg_memcpy_d2d")

    def ipc_export(self, tensor):
        """(handle bytes [64], offset) of a CUDA tensor's storage position, for ipc_import on another rank."""
        buf = C.create_string_buffer(64)
        off = C.c_uint64(0)
        self._check(self.lib.mtg_ipc_export(self.h, tensor.data_ptr(), buf, C.byref(off)), "mtg_ipc_export")
        return bytes(buf.raw), int(off.value)

    def ipc_import(self, handle, offset):
        """-> (pointer to the exported position, base pointer to pass to ipc_close)."""
        ptr, base = C.c_void_p(), C.c_void_p()
        self._check(self.lib.mtg_ipc_import(self.h, handle, int(offset), C.byref(ptr), C.byref(base)), "mtg_ipc_import")
        return int(ptr.value), int(base.value)

    def ipc_close(self, base):
        self._check(self.lib.mtg_ipc_close(self.h, int(base)), "mtg_ipc_close")

    def solve_waypoints_nfabian(self, N, r, positions, v_max, a_max, magic=6.5, coeffs=None, seg_times_out=None,
                                status=None, stream=None):
        """positions: CUDA float64 [B][K+1][D] -> coeffs [B][K][D][N] (fused Nfabian times + packing)."""
        import torch
        B, K1, D = positions.shape
        K = K1 - 1
        assert positions.is_cuda and positions.dtype == torch.float64 and positions.is_contiguous()
        if coeffs is None:
            coeffs = torch.empty((B, K, D, N), dtype=torch.float64, device=positions.device)
        s = stream if stream is not None else torch.cuda.current_stream(positions.device).cuda_stream
        rc = self.lib.mtg_solve_waypoints_nfabian_batch_f64(
            self.h, N, r, K, D, B, positions.data_ptr(), float(v_max), float(a_max), float(magic), coeffs.data_ptr(),
            seg_times_out.data_ptr() if seg_times_out is not None else None,
            status.data_ptr() if status is not None else None, s)
        self._check(rc, "mtg_solve_waypoints_nfabian_batch_f64")
        return coeffs

    def evaluate(self, seg_times, coeffs, derivative, t_start, dt, n_samples, stream=None, out=None):
        """coeffs [B][K][D][N] -> samples [B][n_samples][D] of the given derivative (Trajectory::evaluate)."""
        import torch
        B, K, D, N = coeffs.shape
        if out is None:
            out = torch.empty((B, n_samples, D), dtype=torch.float64, device=coeffs.device)
        assert out.is_contiguous() and tuple(out.shape) == (B, n_samples, D)
        s = stream if stream is not None else torch.cuda.current_stream(coeffs.device).cuda_stream
        rc = self.lib.mtg_evaluate_batch_f64(self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(),
                                             int(derivative), float(t_start), float(dt), int(n_samples),
                                             out.data_ptr(), s)
        self._check(rc, "mtg_evaluate_batch_f64")
        return out

    def evaluate_range(self, seg_times, coeffs, t_start, t_end, dt, derivs=(0,), max_samples=None, want_times=False,
                       stream=None):
        """Batched Trajectory::evaluateRange: (out [B][S][len(derivs)][D], n_samples [B] int32, sampling_times or None)."""
        import torch
        B, K, D, N = coeffs.shape
        if max_samples is None:
            max_samples = int((t_end - t_start) / dt + 1) + 2
        derivs = [int(x) for x in derivs]
        arr = (C.c_int32 * len(derivs))(*derivs)
        out = torch.empty((B, max_samples, len(derivs), D), dtype=torch.float64, device=coeffs.device)
        n = torch.empty((B,), dtype=torch.int32, device=coeffs.device)
        st = torch.zeros((B, max_samples), dtype=torch.float64, device=coeffs.device) if want_times else None
        s = stream if stream is not None else torch.cuda.current_stream(coeffs.device).cuda_stream
        rc = self.lib.mtg_evaluate_range_batch_f64(self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(),
                                                   float(t_start), float(t_end), float(dt), len(derivs), arr,
                                                   int(max_samples), out.data_ptr(), n.data_ptr(),
                                                   st.data_ptr() if want_times else None, s)
        self._check(rc, "mtg_evaluate_range_batch_f64")
        return out, n, st

    def sample_flat_states(self, seg_times, coeffs, min_time, max_time, sampling_interval, max_samples=None,
                           stream=None, _whole=0):
        """Batched sampleTrajectoryInRange: (states [B][S][FLAT_STATE_DOUBLES], time_ns [B][S] int64, n_samples [B]
        int32).  Fields are the FLAT_STATE_FIELDS slices of the last axis; records past n_samples[b] are zero and
        n_samples[b] is -1 where the reference returns false.  max_samples=None sizes S to the largest count, which
        takes a counting pass and waits for it."""
        import torch
        B, K, D, N = coeffs.shape
        s = stream if stream is not None else torch.cuda.current_stream(coeffs.device).cuda_stream
        n = torch.empty((B,), dtype=torch.int32, device=coeffs.device)

        def run(S, states, time_ns):
            rc = self.lib.mtg_sample_flat_states_batch_f64(
                self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(), float(min_time), float(max_time),
                float(sampling_interval), int(_whole), int(S), states.data_ptr() if states is not None else None,
                time_ns.data_ptr() if time_ns is not None else None, n.data_ptr(), s)
            self._check(rc, "mtg_sample_flat_states_batch_f64")

        if max_samples is None:
            run(0, None, None)
            max_samples = max(int(n.max().item()), 0) if B else 0
        states = torch.empty((B, max_samples, FLAT_STATE_DOUBLES), dtype=torch.float64, device=coeffs.device)
        time_ns = torch.empty((B, max_samples), dtype=torch.int64, device=coeffs.device)
        run(max_samples, states, time_ns)
        return states, time_ns, n

    def sample_whole_trajectories(self, seg_times, coeffs, sampling_interval, max_samples=None, stream=None):
        """Batched sampleWholeTrajectory: sample_flat_states over [0, each row's total time]."""
        return self.sample_flat_states(seg_times, coeffs, 0.0, 0.0, sampling_interval, max_samples, stream, _whole=1)

    def sample_flat_state_at_time(self, seg_times, coeffs, sample_times, stream=None):
        """Batched sampleTrajectoryAtTime, row b at sample_times[b]: (states [B][FLAT_STATE_DOUBLES], time_ns [B] int64,
        ok [B] int32; 0 with a zero record where the reference returns false)."""
        import torch
        B, K, D, N = coeffs.shape
        states = torch.empty((B, FLAT_STATE_DOUBLES), dtype=torch.float64, device=coeffs.device)
        time_ns = torch.empty((B,), dtype=torch.int64, device=coeffs.device)
        ok = torch.empty((B,), dtype=torch.int32, device=coeffs.device)
        s = stream if stream is not None else torch.cuda.current_stream(coeffs.device).cuda_stream
        rc = self.lib.mtg_sample_flat_state_at_time_batch_f64(self.h, N, K, D, B, seg_times.data_ptr(),
                                                              coeffs.data_ptr(), sample_times.data_ptr(),
                                                              states.data_ptr(), time_ns.data_ptr(), ok.data_ptr(), s)
        self._check(rc, "mtg_sample_flat_state_at_time_batch_f64")
        return states, time_ns, ok

    def cost_gradient_mellinger(self, prob, seg_times, d_fixed, stream=None):
        """(cost [B], grad [B][K]) -- batched getCostAndGradientMellinger."""
        import torch
        B = seg_times.shape[0]
        cost = torch.empty((B,), dtype=torch.float64, device=seg_times.device)
        grad = torch.empty((B, prob.K), dtype=torch.float64, device=seg_times.device)
        s = stream if stream is not None else torch.cuda.current_stream(seg_times.device).cuda_stream
        rc = self.lib.mtg_cost_gradient_mellinger_batch_f64(self.h, C.byref(prob.c), B, seg_times.data_ptr(),
                                                            d_fixed.data_ptr(), cost.data_ptr(), grad.data_ptr(), s)
        self._check(rc, "mtg_cost_gradient_mellinger_batch_f64")
        return cost, grad

    def max_magnitude(self, seg_times, coeffs, derivs=(1, 2), stream=None):
        """Batched computeMaximumOfMagnitude: (value, time, segment) [B][len(derivs)] and status [B] (int32)."""
        import torch
        B, K, D, N = coeffs.shape
        derivs = [int(x) for x in derivs]
        arr = (C.c_int32 * max(len(derivs), 1))(*derivs)
        dev = coeffs.device
        value = torch.empty((B, len(derivs)), dtype=torch.float64, device=dev)
        time = torch.empty((B, len(derivs)), dtype=torch.float64, device=dev)
        segment = torch.empty((B, len(derivs)), dtype=torch.int32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_max_magnitude_batch_f64(self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(),
                                                  len(derivs), arr, value.data_ptr(), time.data_ptr(),
                                                  segment.data_ptr(), status.data_ptr(), s)
        self._check(rc, "mtg_max_magnitude_batch_f64")
        return value, time, segment, status

    def time_objective(self, prob, seg_times, d_fixed, d_free=None, constraints=(), time_cost=TIME_COST_SQUARED,
                       time_penalty=500.0, soft_constraint_weight=100.0, maximum_cost=1e12, stream=None):
        """Batched objectiveFunctionTime (d_free None) / objectiveFunctionTimeAndConstraints: (objective [B],
        terms [B][3] = (trajectory, time, soft), coeffs [B][K][D][N], status [B]).  constraints: [(derivative,
        max_value), ...]."""
        import torch
        B = seg_times.shape[0]
        dev = seg_times.device
        obj = time_objective_params(time_cost, time_penalty, soft_constraint_weight, maximum_cost, constraints)
        coeffs = torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=dev)
        objective = torch.empty((B,), dtype=torch.float64, device=dev)
        terms = torch.empty((B, 3), dtype=torch.float64, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_time_objective_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(),
            d_free.data_ptr() if d_free is not None else None, C.byref(obj), coeffs.data_ptr(), objective.data_ptr(),
            terms.data_ptr(), status.data_ptr(), s)
        self._check(rc, "mtg_time_objective_batch_f64")
        return objective, terms, coeffs, status

    def scale_to_constraints(self, seg_times, coeffs, v_max, a_max, seg_times_out=None, coeffs_out=None, stream=None):
        """Batched Trajectory::scaleSegmentTimesToMeetConstraints: (seg_times_out [B][K], coeffs_out [B][K][D][N],
        within_range [B] int32, maxima [B][2] = (max |v|, max |a|) at the last check, status [B] int32).  Pass the
        input tensors as the outputs to stretch in place; v_max / a_max = inf means no limit on that order."""
        import torch
        B, K, D, N = coeffs.shape
        dev = coeffs.device
        if seg_times_out is None:
            seg_times_out = torch.empty_like(seg_times)
        if coeffs_out is None:
            coeffs_out = torch.empty_like(coeffs)
        within = torch.empty((B,), dtype=torch.int32, device=dev)
        maxima = torch.empty((B, 2), dtype=torch.float64, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_scale_to_constraints_batch_f64(
            self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(), float(v_max), float(a_max),
            seg_times_out.data_ptr(), coeffs_out.data_ptr(), within.data_ptr(), maxima.data_ptr(), status.data_ptr(), s)
        self._check(rc, "mtg_scale_to_constraints_batch_f64")
        return seg_times_out, coeffs_out, within, maxima, status

    def scale_times_with_violation(self, prob, seg_times, d_fixed, v_max, a_max, seg_times_out=None, stream=None):
        """Batched PolynomialOptimizationNonLinear::scaleSegmentTimesWithViolation: solve, stretch, re-solve at the
        stretched times.  -> (coeffs [B][K][D][N], seg_times_out [B][K], within_range [B], maxima [B][2], status [B])."""
        import torch
        B = seg_times.shape[0]
        dev = seg_times.device
        coeffs = torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=dev)
        if seg_times_out is None:
            seg_times_out = torch.empty_like(seg_times)
        within = torch.empty((B,), dtype=torch.int32, device=dev)
        maxima = torch.empty((B, 2), dtype=torch.float64, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_scale_times_with_violation_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(), float(v_max), float(a_max),
            coeffs.data_ptr(), seg_times_out.data_ptr(), within.data_ptr(), maxima.data_ptr(), status.data_ptr(), s)
        self._check(rc, "mtg_scale_times_with_violation_batch_f64")
        return coeffs, seg_times_out, within, maxima, status

    def optimize_time_mellinger(self, prob, seg_times, d_fixed, v_max, a_max, params=None, seg_times_out=None,
                                stream=None):
        """Batched PolynomialOptimizationNonLinear::optimize() with kMellingerOuterLoop (mtg_b200.h states the
        descent): -> dict of coeffs [B][K][D][N], seg_times (scaled) [B][K], relative_times [B][K], cost [B],
        iterations [B], result [B] (OPTIMIZE_RESULT_*), within_range [B], maxima [B][2], status [B].  params: a
        mellinger_params() (defaults: the reference's).  Waits on the stream once per iteration."""
        import torch
        B = seg_times.shape[0]
        dev = seg_times.device
        if params is None:
            params = mellinger_params()
        out = dict(coeffs=torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=dev),
                   seg_times=seg_times_out if seg_times_out is not None else torch.empty_like(seg_times),
                   relative_times=torch.empty_like(seg_times),
                   cost=torch.empty((B,), dtype=torch.float64, device=dev),
                   iterations=torch.empty((B,), dtype=torch.int32, device=dev),
                   result=torch.empty((B,), dtype=torch.int32, device=dev),
                   within_range=torch.empty((B,), dtype=torch.int32, device=dev),
                   maxima=torch.empty((B, 2), dtype=torch.float64, device=dev),
                   status=torch.empty((B,), dtype=torch.int32, device=dev))
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_optimize_time_mellinger_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(), C.byref(params), float(v_max),
            float(a_max), *[out[k].data_ptr() for k in self._MELLINGER_OUTPUTS], s)
        self._check(rc, "mtg_optimize_time_mellinger_batch_f64")
        return out

    _MELLINGER_OUTPUTS = ("coeffs", "seg_times", "relative_times", "cost", "iterations", "result", "within_range",
                          "maxima", "status")

    def optimize_time(self, prob, seg_times, d_fixed, constraints=(), time_cost=TIME_COST_SQUARED, params=None,
                      time_penalty=500.0, soft_constraint_weight=100.0, maximum_cost=1e12, seg_times_out=None,
                      stream=None):
        """Batched PolynomialOptimizationNonLinear::optimize() with kSquaredTime (time_cost TIME_COST_SQUARED) or
        kRichterTime (TIME_COST_RICHTER), as the compass search of mtg_b200.h: -> dict of coeffs [B][K][D][N],
        seg_times [B][K] (the best point), objective [B], terms [B][3], evaluations [B], result [B]
        (OPTIMIZE_RESULT_*), status [B].  constraints: soft [(derivative, max_value), ...]; params: a mellinger_params()
        whose max_iterations counts objective evaluations.  Waits on the stream once per poll."""
        import torch
        B = seg_times.shape[0]
        dev = seg_times.device
        if params is None:
            params = mellinger_params()
        obj = time_objective_params(time_cost, time_penalty, soft_constraint_weight, maximum_cost, constraints)
        out = dict(coeffs=torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=dev),
                   seg_times=seg_times_out if seg_times_out is not None else torch.empty_like(seg_times),
                   objective=torch.empty((B,), dtype=torch.float64, device=dev),
                   terms=torch.empty((B, 3), dtype=torch.float64, device=dev),
                   evaluations=torch.empty((B,), dtype=torch.int32, device=dev),
                   result=torch.empty((B,), dtype=torch.int32, device=dev),
                   status=torch.empty((B,), dtype=torch.int32, device=dev))
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_optimize_time_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(), C.byref(obj), C.byref(params),
            *[out[k].data_ptr() for k in self._OPTIMIZE_TIME_OUTPUTS], s)
        self._check(rc, "mtg_optimize_time_batch_f64")
        return out

    _OPTIMIZE_TIME_OUTPUTS = ("coeffs", "seg_times", "objective", "terms", "evaluations", "result", "status")

    def check_input_feasibility(self, seg_times, coeffs, limits, min_section_time=0.05, gravity=GRAVITY, stream=None):
        """Batched FeasibilityAnalytic::checkInputFeasibilityTrajectory: (result [B], segment [B], status [B]), int32.
        limits: {name: value} over INPUT_LIMITS (absent name = no limit; default_input_limits() gives the reference's
        defaults) or an MtgInputConstraints."""
        return self._input_feasibility("mtg_input_feasibility_batch_f64", seg_times, coeffs, limits, min_section_time,
                                       gravity, stream)

    def check_input_feasibility_recursive(self, seg_times, coeffs, limits, min_section_time=0.05, gravity=GRAVITY,
                                          stream=None):
        """Batched FeasibilityRecursive::checkInputFeasibilityTrajectory: (result [B], segment [B], status [B]), int32,
        with the arguments of check_input_feasibility."""
        return self._input_feasibility("mtg_input_feasibility_recursive_batch_f64", seg_times, coeffs, limits,
                                       min_section_time, gravity, stream)

    def check_input_feasibility_sampling(self, seg_times, coeffs, limits, sampling_interval=0.01, gravity=GRAVITY,
                                         stream=None):
        """Batched FeasibilitySampling::checkInputFeasibilityTrajectory: (result [B], segment [B], status [B]), int32.
        limits as for check_input_feasibility; samples every sampling_interval seconds from the start of each
        segment (an MtgInputConstraints' min_section_time is ignored)."""
        return self._input_feasibility("mtg_input_feasibility_sampling_batch_f64", seg_times, coeffs, limits, 0.05,
                                       gravity, stream, (float(sampling_interval),))

    def _input_feasibility(self, entry, seg_times, coeffs, limits, min_section_time, gravity, stream, extra=()):
        import torch
        B, K, D, N = coeffs.shape
        dev = coeffs.device
        ic = limits if isinstance(limits, MtgInputConstraints) else input_constraints(limits, min_section_time, gravity)
        result = torch.empty((B,), dtype=torch.int32, device=dev)
        segment = torch.empty((B,), dtype=torch.int32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = getattr(self.lib, entry)(self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(), C.byref(ic), *extra,
                                      result.data_ptr(), segment.data_ptr(), status.data_ptr(), s)
        self._check(rc, entry)
        return result, segment, status

    def check_half_plane_feasibility(self, seg_times, coeffs, planes, stream=None):
        """Batched FeasibilityBase::checkHalfPlaneFeasibility: (feasible, segment, plane, status), each [B] int32.
        planes: [P][6] float64 rows (point, normal; see half_plane / bounding_box), used as given."""
        import torch
        B, K, D, N = coeffs.shape
        dev = coeffs.device
        arr, P = half_plane_array(planes)
        out = [torch.empty((B,), dtype=torch.int32, device=dev) for _ in range(4)]
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.mtg_half_plane_feasibility_batch_f64(self.h, N, K, D, B, seg_times.data_ptr(), coeffs.data_ptr(),
                                                           P, arr, *(o.data_ptr() for o in out), s)
        self._check(rc, "mtg_half_plane_feasibility_batch_f64")
        return tuple(out)

    def coeffs_from_constraints(self, prob, seg_times, d_fixed, d_free, coeffs=None, stream=None):
        import torch
        B = seg_times.shape[0]
        if coeffs is None:
            coeffs = torch.empty((B, prob.K, prob.D, prob.N), dtype=torch.float64, device=seg_times.device)
        s = stream if stream is not None else torch.cuda.current_stream(seg_times.device).cuda_stream
        rc = self.lib.mtg_coeffs_from_constraints_batch_f64(
            self.h, C.byref(prob.c), B, seg_times.data_ptr(), d_fixed.data_ptr(),
            d_free.data_ptr() if d_free is not None else None, coeffs.data_ptr(), s)
        self._check(rc, "mtg_coeffs_from_constraints_batch_f64")
        return coeffs

    def compute_cost(self, prob, seg_times, coeffs, cost=None, stream=None):
        import torch
        B = seg_times.shape[0]
        if cost is None:
            cost = torch.empty((B,), dtype=torch.float64, device=seg_times.device)
        s = stream if stream is not None else torch.cuda.current_stream(seg_times.device).cuda_stream
        rc = self.lib.mtg_compute_cost_batch_f64(self.h, C.byref(prob.c), B, seg_times.data_ptr(),
                                                 coeffs.data_ptr(), cost.data_ptr(), s)
        self._check(rc, "mtg_compute_cost_batch_f64")
        return cost

    # ---- host-pointer path (numpy arrays or pinned torch CPU tensors) ----------------------
    @staticmethod
    def _hptr(a):
        if a is None:
            return None
        if isinstance(a, np.ndarray):
            assert a.flags["C_CONTIGUOUS"]
            return a.ctypes.data
        assert a.is_contiguous() and not a.is_cuda
        return a.data_ptr()

    def solve_linear_host(self, prob, seg_times, d_fixed, coeffs, d_free=None, status=None):
        B = seg_times.shape[0]
        rc = self.lib.mtg_solve_linear_batch_host_f64(
            self.h, C.byref(prob.c), B, self._hptr(seg_times), self._hptr(d_fixed), self._hptr(coeffs),
            self._hptr(d_free), self._hptr(status))
        self._check(rc, "mtg_solve_linear_batch_host_f64")
        return coeffs

    def solve_waypoints_nfabian_host(self, N, r, positions, v_max, a_max, magic, coeffs, seg_times_out=None,
                                     status=None):
        """positions host [B][K+1][D] -> coeffs host [B][K][D][N] (pipelined H2D / fused solve / D2H)."""
        B, K1, D = positions.shape
        rc = self.lib.mtg_solve_waypoints_nfabian_batch_host_f64(
            self.h, N, r, K1 - 1, D, B, self._hptr(positions), float(v_max), float(a_max), float(magic),
            self._hptr(coeffs), self._hptr(seg_times_out), self._hptr(status))
        self._check(rc, "mtg_solve_waypoints_nfabian_batch_host_f64")
        return coeffs

    def coeffs_from_constraints_host(self, prob, seg_times, d_fixed, d_free, coeffs):
        B = seg_times.shape[0]
        rc = self.lib.mtg_coeffs_from_constraints_batch_host_f64(
            self.h, C.byref(prob.c), B, self._hptr(seg_times), self._hptr(d_fixed), self._hptr(d_free),
            self._hptr(coeffs))
        self._check(rc, "mtg_coeffs_from_constraints_batch_host_f64")
        return coeffs

    def compute_cost_host(self, prob, seg_times, coeffs, cost):
        B = seg_times.shape[0]
        rc = self.lib.mtg_compute_cost_batch_host_f64(self.h, C.byref(prob.c), B, self._hptr(seg_times),
                                                      self._hptr(coeffs), self._hptr(cost))
        self._check(rc, "mtg_compute_cost_batch_host_f64")
        return cost

    def cost_gradient_mellinger_host(self, prob, seg_times, d_fixed, cost, grad):
        """cost [B] (or None) and grad [B][K] host buffers -- batched getCostAndGradientMellinger."""
        B = seg_times.shape[0]
        rc = self.lib.mtg_cost_gradient_mellinger_batch_host_f64(
            self.h, C.byref(prob.c), B, self._hptr(seg_times), self._hptr(d_fixed), self._hptr(cost), self._hptr(grad))
        self._check(rc, "mtg_cost_gradient_mellinger_batch_host_f64")
        return grad

    def evaluate_range_host(self, seg_times, coeffs, t_start, t_end, dt, derivs, out, n_samples, sampling_times=None):
        """Batched Trajectory::evaluateRange into host buffers: out [B][max_samples][len(derivs)][D], n_samples [B]
        int32, sampling_times [B][max_samples] or None (max_samples is out.shape[1])."""
        B, K, D, N = coeffs.shape
        derivs = [int(x) for x in derivs]
        arr = (C.c_int32 * len(derivs))(*derivs)
        rc = self.lib.mtg_evaluate_range_batch_host_f64(
            self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs), float(t_start), float(t_end), float(dt),
            len(derivs), arr, int(out.shape[1]), self._hptr(out), self._hptr(n_samples), self._hptr(sampling_times))
        self._check(rc, "mtg_evaluate_range_batch_host_f64")
        return n_samples

    def sample_flat_states_host(self, seg_times, coeffs, min_time, max_time, sampling_interval, states, n_samples,
                                time_ns=None, whole=False):
        """sample_flat_states (whole=True: sample_whole_trajectories) into host buffers: states
        [B][max_samples][FLAT_STATE_DOUBLES], n_samples [B] int32, time_ns [B][max_samples] int64 or None
        (max_samples is states.shape[1])."""
        B, K, D, N = coeffs.shape
        rc = self.lib.mtg_sample_flat_states_batch_host_f64(
            self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs), float(min_time), float(max_time),
            float(sampling_interval), int(bool(whole)), int(states.shape[1]), self._hptr(states), self._hptr(time_ns),
            self._hptr(n_samples))
        self._check(rc, "mtg_sample_flat_states_batch_host_f64")
        return n_samples

    def sample_flat_state_at_time_host(self, seg_times, coeffs, sample_times, states, ok, time_ns=None):
        """sample_flat_state_at_time into host buffers: states [B][FLAT_STATE_DOUBLES], ok [B] int32, time_ns [B]
        int64 or None."""
        B, K, D, N = coeffs.shape
        rc = self.lib.mtg_sample_flat_state_at_time_batch_host_f64(
            self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs), self._hptr(sample_times),
            self._hptr(states), self._hptr(time_ns), self._hptr(ok))
        self._check(rc, "mtg_sample_flat_state_at_time_batch_host_f64")
        return ok

    def max_magnitude_host(self, seg_times, coeffs, derivs, value, time=None, segment=None, status=None):
        B, K, D, N = coeffs.shape
        derivs = [int(x) for x in derivs]
        arr = (C.c_int32 * max(len(derivs), 1))(*derivs)
        rc = self.lib.mtg_max_magnitude_batch_host_f64(self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs),
                                                       len(derivs), arr, self._hptr(value), self._hptr(time),
                                                       self._hptr(segment), self._hptr(status))
        self._check(rc, "mtg_max_magnitude_batch_host_f64")
        return value

    def time_objective_host(self, prob, seg_times, d_fixed, d_free, obj, coeffs, objective, terms=None, status=None):
        """obj: time_objective_params(...)."""
        B = seg_times.shape[0]
        rc = self.lib.mtg_time_objective_batch_host_f64(
            self.h, C.byref(prob.c), B, self._hptr(seg_times), self._hptr(d_fixed), self._hptr(d_free), C.byref(obj),
            self._hptr(coeffs), self._hptr(objective), self._hptr(terms), self._hptr(status))
        self._check(rc, "mtg_time_objective_batch_host_f64")
        return objective

    def scale_to_constraints_host(self, seg_times, coeffs, v_max, a_max, seg_times_out, coeffs_out, within_range=None,
                                  maxima=None, status=None):
        B, K, D, N = coeffs.shape
        rc = self.lib.mtg_scale_to_constraints_batch_host_f64(
            self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs), float(v_max), float(a_max),
            self._hptr(seg_times_out), self._hptr(coeffs_out), self._hptr(within_range), self._hptr(maxima),
            self._hptr(status))
        self._check(rc, "mtg_scale_to_constraints_batch_host_f64")
        return seg_times_out

    def optimize_time_mellinger_host(self, prob, seg_times, d_fixed, v_max, a_max, params=None):
        """optimize_time_mellinger on host numpy arrays (one copy in, the loop, one copy out): a dict of numpy
        arrays with the same keys."""
        B, K = seg_times.shape
        if params is None:
            params = mellinger_params()
        seg_times = np.ascontiguousarray(seg_times, dtype=np.float64)
        d_fixed = np.ascontiguousarray(d_fixed, dtype=np.float64)
        f8, i4 = np.float64, np.int32
        out = dict(coeffs=np.empty((B, K, prob.D, prob.N), f8), seg_times=np.empty((B, K), f8),
                   relative_times=np.empty((B, K), f8), cost=np.empty(B, f8), iterations=np.empty(B, i4),
                   result=np.empty(B, i4), within_range=np.empty(B, i4), maxima=np.empty((B, 2), f8),
                   status=np.empty(B, i4))
        rc = self.lib.mtg_optimize_time_mellinger_batch_host_f64(
            self.h, C.byref(prob.c), B, seg_times.ctypes.data, d_fixed.ctypes.data, C.byref(params), float(v_max),
            float(a_max), *[out[k].ctypes.data for k in self._MELLINGER_OUTPUTS])
        self._check(rc, "mtg_optimize_time_mellinger_batch_host_f64")
        return out

    def optimize_time_host(self, prob, seg_times, d_fixed, constraints=(), time_cost=TIME_COST_SQUARED, params=None,
                           time_penalty=500.0, soft_constraint_weight=100.0, maximum_cost=1e12):
        """optimize_time on host numpy arrays (one copy in, the search, one copy out): a dict of numpy arrays with
        the same keys."""
        B, K = seg_times.shape
        if params is None:
            params = mellinger_params()
        obj = time_objective_params(time_cost, time_penalty, soft_constraint_weight, maximum_cost, constraints)
        seg_times = np.ascontiguousarray(seg_times, dtype=np.float64)
        d_fixed = np.ascontiguousarray(d_fixed, dtype=np.float64)
        f8, i4 = np.float64, np.int32
        out = dict(coeffs=np.empty((B, K, prob.D, prob.N), f8), seg_times=np.empty((B, K), f8),
                   objective=np.empty(B, f8), terms=np.empty((B, 3), f8), evaluations=np.empty(B, i4),
                   result=np.empty(B, i4), status=np.empty(B, i4))
        rc = self.lib.mtg_optimize_time_batch_host_f64(
            self.h, C.byref(prob.c), B, seg_times.ctypes.data, d_fixed.ctypes.data, C.byref(obj), C.byref(params),
            *[out[k].ctypes.data for k in self._OPTIMIZE_TIME_OUTPUTS])
        self._check(rc, "mtg_optimize_time_batch_host_f64")
        return out

    def scale_times_with_violation_host(self, prob, seg_times, d_fixed, v_max, a_max, coeffs, seg_times_out,
                                        within_range=None, maxima=None, status=None):
        B = seg_times.shape[0]
        rc = self.lib.mtg_scale_times_with_violation_batch_host_f64(
            self.h, C.byref(prob.c), B, self._hptr(seg_times), self._hptr(d_fixed), float(v_max), float(a_max),
            self._hptr(coeffs), self._hptr(seg_times_out), self._hptr(within_range), self._hptr(maxima),
            self._hptr(status))
        self._check(rc, "mtg_scale_times_with_violation_batch_host_f64")
        return coeffs

    def check_input_feasibility_host(self, seg_times, coeffs, limits, result, segment=None, status=None,
                                     min_section_time=0.05, gravity=GRAVITY):
        """check_input_feasibility into host buffers: result [B], segment [B] or None, status [B] or None (int32)."""
        return self._input_feasibility_host("mtg_input_feasibility_batch_host_f64", seg_times, coeffs, limits, result,
                                            segment, status, min_section_time, gravity)

    def check_input_feasibility_recursive_host(self, seg_times, coeffs, limits, result, segment=None, status=None,
                                               min_section_time=0.05, gravity=GRAVITY):
        """check_input_feasibility_recursive into host buffers: result [B], segment [B] or None, status [B] or None
        (int32)."""
        return self._input_feasibility_host("mtg_input_feasibility_recursive_batch_host_f64", seg_times, coeffs,
                                            limits, result, segment, status, min_section_time, gravity)

    def check_input_feasibility_sampling_host(self, seg_times, coeffs, limits, result, segment=None, status=None,
                                              sampling_interval=0.01, gravity=GRAVITY):
        """check_input_feasibility_sampling into host buffers: result [B], segment [B] or None, status [B] or None
        (int32)."""
        return self._input_feasibility_host("mtg_input_feasibility_sampling_batch_host_f64", seg_times, coeffs,
                                            limits, result, segment, status, 0.05, gravity,
                                            (float(sampling_interval),))

    def _input_feasibility_host(self, entry, seg_times, coeffs, limits, result, segment, status, min_section_time,
                                gravity, extra=()):
        B, K, D, N = coeffs.shape
        ic = limits if isinstance(limits, MtgInputConstraints) else input_constraints(limits, min_section_time, gravity)
        rc = getattr(self.lib, entry)(self.h, N, K, D, B, self._hptr(seg_times), self._hptr(coeffs), C.byref(ic),
                                      *extra,
                                      self._hptr(result), self._hptr(segment), self._hptr(status))
        self._check(rc, entry)
        return result

    def check_half_plane_feasibility_host(self, seg_times, coeffs, planes, feasible, segment=None, plane=None,
                                          status=None):
        """check_half_plane_feasibility into host buffers: feasible [B]; segment, plane, status [B] or None (int32)."""
        B, K, D, N = coeffs.shape
        arr, P = half_plane_array(planes)
        rc = self.lib.mtg_half_plane_feasibility_batch_host_f64(self.h, N, K, D, B, self._hptr(seg_times),
                                                                self._hptr(coeffs), P, arr, self._hptr(feasible),
                                                                self._hptr(segment), self._hptr(plane),
                                                                self._hptr(status))
        self._check(rc, "mtg_half_plane_feasibility_batch_host_f64")
        return feasible
