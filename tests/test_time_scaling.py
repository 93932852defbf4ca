"""Batched Trajectory::scaleSegmentTimesToMeetConstraints (mtg_scale_to_constraints_batch_f64) and
PolynomialOptimizationNonLinear::scaleSegmentTimesWithViolation (mtg_scale_times_with_violation_batch_f64).

`replay` restates the reference loop (src/trajectory.cpp:382-429) in NumPy with std::max semantics, over any maxima
function.  On the CPU it is pinned to closed forms with the binary128 maxima of tests/extrema_exact.cpp; on the GPU the
kernel must equal the replay over mtg_max_magnitude_batch_f64 bit for bit, and its decisions must agree with the
binary128 maxima wherever they are not within the maxima's forward-error bound of the threshold."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import extrema_oracle as X
from test_time_objective import EPS, random_segments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_time_scaling.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_time_scaling")
LIMIT = 1.0 + 1e-3  # 1.0 + kTolerance (trajectory.cpp:386)
MAX_ROUNDS = 20


def build_binary():
    """C++ check of the batch class against the single-object host mirror (tests/cpp/test_time_scaling.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


def _std_max(x, y):
    """std::max(x, y) = (x < y) ? y : x, elementwise (NaN in x is kept, NaN in y is not)."""
    return np.where(x < y, y, x)


def replay(times, coeffs, v_max, a_max, maxima_fn):
    """The reference loop for B trajectories.  maxima_fn(times, coeffs) -> (v [B], a [B]).  A row with a segment time
    <= 0 or non-finite stops with status 1 (MTG_STATUS_BAD_TIME), within 0, maxima NaN, untouched.
    -> (times, coeffs, within [B], maxima [B][2], status [B], stretches [B], first_scale [B])."""
    times = np.array(times, dtype=np.float64)
    coeffs = np.array(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    within = np.zeros(B, dtype=np.int32)
    maxima = np.full((B, 2), np.nan)
    status = np.zeros(B, dtype=np.int32)
    stretches = np.zeros(B, dtype=np.int64)
    first_scale = np.ones(B)
    active = np.ones(B, dtype=bool)
    for rnd in range(MAX_ROUNDS):
        rows = np.nonzero(active)[0]
        if rows.size == 0:
            break
        bad = (~(times[rows] > 0.0) | ~np.isfinite(times[rows])).any(axis=1)
        status[rows[bad]] = 1
        within[rows[bad]] = 0
        active[rows[bad]] = False
        rows = rows[~bad]
        if rows.size == 0:
            break
        v, a = maxima_fn(times[rows], coeffs[rows])
        maxima[rows, 0], maxima[rows, 1] = v, a
        with np.errstate(invalid="ignore"):  # inf / inf: a NaN violation, as in the reference
            vv, av = v / v_max, a / a_max
        ok = (vv <= LIMIT) & (av <= LIMIT)
        within[rows] = ok
        active[rows[ok]] = False
        go = rows[~ok]
        s = _std_max(np.ones(go.size), _std_max(vv[~ok], np.sqrt(av[~ok])))
        if rnd == 0:
            first_scale[go] = s
        inv = 1.0 / s
        times[go] = times[go] * s[:, None]
        f = np.ones(go.size)
        for n in range(N):  # Polynomial::scalePolynomialInTime
            coeffs[go, :, :, n] = coeffs[go, :, :, n] * f[:, None, None]
            f = f * inv
        stretches[go] += 1
    return times, coeffs, within, maxima, status, stretches, first_scale


def exact_maxima(times, coeffs):
    return X.max_magnitude(times, coeffs, 1)["value"], X.max_magnitude(times, coeffs, 2)["value"]


# ---- CPU: the replay pinned with the binary128 maxima -------------------------------------------------------------
def _one(N, coeffs_row, T=1.0):
    c = np.zeros((1, 1, 1, N))
    c[0, 0, 0, :len(coeffs_row)] = coeffs_row
    return np.array([[T]]), c


def test_replay_closed_form_acceleration_bound():
    # p = t^2 on [0, 1]: max |a| = 2 against 0.5 -> s = sqrt(4) = 2, T = 2, p = 0.25 t^2, then a = 0.5: within
    times, c = _one(4, (0, 0, 1))
    t, co, w, mx, st, n, s0 = replay(times, c, np.inf, 0.5, exact_maxima)
    assert t[0, 0] == 2.0 and co[0, 0, 0].tolist() == [0.0, 0.0, 0.25, 0.0]
    assert w[0] == 1 and n[0] == 1 and s0[0] == 2.0 and st[0] == 0
    assert mx[0].tolist() == [1.0, 0.5]  # the last check: v = 2 * 0.25 * 2, a = 0.5


def test_replay_velocity_and_acceleration_dominated():
    # velocity-bound: p = 3t + t^2 / 2 on [0, 1], v = 4 at t = 1 against 2 (a = 1 against 10): s = 2
    times, c = _one(6, (0, 3, 0.5))
    t, co, w, mx, st, n, s0 = replay(times, c, 2.0, 10.0, exact_maxima)
    assert s0[0] == 2.0 and t[0, 0] == 2.0 and w[0] == 1 and n[0] == 1
    assert co[0, 0, 0, :3].tolist() == [0.0, 1.5, 0.125]
    # acceleration-bound: same polynomial, a = 1 against 1 / 9 -> sqrt(9) = 3 beats v / v_max = 4 / 100
    t, co, w, mx, st, n, s0 = replay(times, c, 100.0, 1.0 / 9.0, exact_maxima)
    assert s0[0] == np.sqrt(1.0 / (1.0 / 9.0)) and n[0] == 1 and w[0] == 1 and t[0, 0] == s0[0]


def test_replay_feasible_and_infinite_limits():
    rng = np.random.default_rng(1)
    times, c = random_segments(rng, 6, 3, 2, 8)
    v, a = exact_maxima(times, c)
    t, co, w, mx, st, n, _ = replay(times, c, float(v.max()) * 2, float(a.max()) * 2, exact_maxima)
    assert (n == 0).all() and (w == 1).all() and np.array_equal(t, times) and np.array_equal(co, c)
    assert np.array_equal(mx[:, 0], v) and np.array_equal(mx[:, 1], a)
    t, co, w, mx, st, n, _ = replay(times, c, np.inf, np.inf, exact_maxima)  # violation 0: no limit
    assert (n == 0).all() and (w == 1).all() and np.array_equal(t, times)


def test_replay_nan_violation_keeps_stretching_by_one():
    # a NaN maximum (or inf / inf) makes std::max(vv, sqrt(av)) NaN and std::max(1, NaN) = 1: 20 unchanged rounds
    times, c = _one(4, (0, 1, 1))
    t, co, w, mx, st, n, s0 = replay(times, c, 1.0, 1.0, lambda tt, cc: (np.full(len(tt), np.nan), np.zeros(len(tt))))
    assert n[0] == MAX_ROUNDS and w[0] == 0 and s0[0] == 1.0 and np.array_equal(t, times) and np.array_equal(co, c)
    t, co, w, mx, st, n, s0 = replay(times, c, np.inf, 1.0, lambda tt, cc: (np.full(len(tt), np.inf), np.zeros(len(tt))))
    assert n[0] == MAX_ROUNDS and w[0] == 0 and np.array_equal(t, times)


def test_replay_bad_time_rows_stop():
    times, c = _one(4, (0, 1, 1))
    for T in (0.0, -1.0, np.nan, np.inf, -np.inf):
        t, co, w, mx, st, n, _ = replay(np.array([[T]]), c, 0.1, 0.1, exact_maxima)
        assert st[0] == 1 and w[0] == 0 and np.isnan(mx[0]).all() and n[0] == 0
        assert np.array_equal(t, np.array([[T]]), equal_nan=True)


def test_null_handle_is_rejected():
    import mav_trajectory_generation_b200 as m
    lib = m.load()
    p = m.Problem(10, 4, 2, 3)
    assert lib.mtg_scale_to_constraints_batch_f64(None, 10, 2, 3, 1, None, None, 1.0, 1.0, None, None, None, None, None,
                                                  None) != 0
    assert lib.mtg_scale_times_with_violation_batch_f64(None, C.byref(p.c), 1, None, None, 1.0, 1.0, None, None, None,
                                                        None, None, None) != 0
    assert lib.mtg_scale_to_constraints_batch_host_f64(None, 10, 2, 3, 1, None, None, 1.0, 1.0, None, None, None, None,
                                                       None) != 0
    assert lib.mtg_scale_times_with_violation_batch_host_f64(None, C.byref(p.c), 1, None, None, 1.0, 1.0, None, None,
                                                             None, None, None) != 0


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def solver():
    """A handle of this module's own, with every option at its default (other modules' tests set options)."""
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (no CPU fallback exists)")
    import mav_trajectory_generation_b200 as m
    s = m.Solver(0)
    yield s
    s.close()


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_maxima(solver):
    def fn(times, coeffs):
        import torch
        v, _, _, st = solver.max_magnitude(_cuda(times), _cuda(coeffs), (1, 2))
        torch.cuda.synchronize()
        v = v.cpu().numpy()
        return v[:, 0], v[:, 1]
    return fn


def run_scale(solver, times, coeffs, v_max, a_max):
    import torch
    t, c, w, mx, st = solver.scale_to_constraints(_cuda(times), _cuda(coeffs), v_max, a_max)
    torch.cuda.synchronize()
    return t.cpu().numpy(), c.cpu().numpy(), w.cpu().numpy(), mx.cpu().numpy(), st.cpu().numpy()


def check_composition(solver, times, coeffs, v_max, a_max, what):
    """The kernel against the replay over mtg_max_magnitude_batch_f64, bit for bit; returns the replay."""
    got = run_scale(solver, times, coeffs, v_max, a_max)
    ref = replay(times, coeffs, v_max, a_max, gpu_maxima(solver))
    for name, g, r in zip(("times", "coeffs", "within", "maxima", "status"), got, ref):
        same = np.array_equal(g, r, equal_nan=True)
        if not same:
            rows = np.nonzero(~np.all((g == r) | (np.isnan(g) & np.isnan(r)), axis=tuple(range(1, g.ndim))))[0]
            raise AssertionError(f"{what}: {name} differs from the replay at rows {rows[:8]}")
    return ref


def mixed_limits(solver, times, coeffs):
    """Limits that leave feasible, velocity-bound and acceleration-bound rows side by side."""
    v, a = gpu_maxima(solver)(times, coeffs)
    return float(np.quantile(v, 0.6)), float(np.quantile(a, 0.6))


def solved_fixtures(solver, oracle, N, K, D, B, seed):
    import torch
    import mav_trajectory_generation_b200 as m
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    prob = m.Problem(N, N // 2 - 1, K, D)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    coeffs = solver.solve_linear(prob, _cuda(times), _cuda(d_fixed))
    torch.cuda.synchronize()
    return prob, pos, times, d_fixed, coeffs.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 6, 8, 10, 12))
@pytest.mark.parametrize("K", (1, 3, 16, 50))
def test_bitwise_equal_to_its_composition(solver, oracle, N, K):
    rng = np.random.default_rng(10 * N + K)
    kinds = np.zeros(3, dtype=np.int64)  # feasible, velocity-bound, acceleration-bound rows
    for D in (1, 2, 3, 4):
        inputs = [random_segments(rng, 40, K, D, N)]
        inputs.append(solved_fixtures(solver, oracle, N, K, D, 40, 6000 + 100 * N + K)[2::2])
        for kind, (times, coeffs) in zip(("random", "solved"), inputs):
            v_max, a_max = mixed_limits(solver, times, coeffs)
            check_composition(solver, times, coeffs, v_max, a_max, f"{kind} N={N} K={K} D={D}")
            first_v, first_a = gpu_maxima(solver)(times, coeffs)
            vv, av = first_v / v_max, first_a / a_max
            feasible = (vv <= LIMIT) & (av <= LIMIT)
            kinds += [feasible.sum(), (~feasible & (vv >= np.sqrt(av))).sum(), (~feasible & (vv < np.sqrt(av))).sum()]
            if kind == "random":  # K >= 3 puts rows of every kind in one CTA tile of 128 / K rows
                assert feasible.any() and (~feasible).any(), (N, K, D)
    assert (kinds > 0).all(), kinds


def exact_decision(times, coeffs, v_max, a_max):
    """First-round violations from binary128 maxima, with the forward-error bound of check_against_exact."""
    N = coeffs.shape[3]
    out = {}
    for k, lim, name in ((1, v_max, "v"), (2, a_max, "a")):
        ex = X.max_magnitude(times, coeffs, k)
        bound = 1e-13 * ex["value"] + 8 * max(N - 1 - k, 1) * EPS * ex["scale"]
        out[name] = ex["value"] / lim
        out["d" + name] = bound / lim
    near = (np.abs(out["v"] - LIMIT) <= out["dv"]) | (np.abs(out["a"] - LIMIT) <= out["da"])
    return out, near


@pytest.mark.gpu
@pytest.mark.parametrize("N", (6, 10, 12))
def test_against_binary128(solver, oracle, N):
    rng = np.random.default_rng(N)
    D, K = 3, 5
    times, coeffs = random_segments(rng, 64, K, D, N)
    v_max, a_max = mixed_limits(solver, times, coeffs)
    # one row placed on the threshold on purpose: its exact velocity violation is 1.001
    ve = X.max_magnitude(times[:1], coeffs[:1], 1)["value"][0]
    vn = v_max * LIMIT
    coeffs[0] = coeffs[0] * (vn / ve)
    t, c, w, mx, st = run_scale(solver, times, coeffs, v_max, a_max)
    assert (st == 0).all()
    ref = replay(times, coeffs, v_max, a_max, gpu_maxima(solver))
    ex, near = exact_decision(times, coeffs, v_max, a_max)
    assert near[0] and near.sum() >= 1
    keep = ~near
    first_within = ref[5] == 0
    exact_within = (ex["v"] <= LIMIT) & (ex["a"] <= LIMIT)
    assert np.array_equal(first_within[keep], exact_within[keep])
    s_exact = np.maximum(1.0, np.maximum(ex["v"], np.sqrt(ex["a"])))
    tol = s_exact * (np.maximum(ex["dv"] / np.maximum(ex["v"], 1e-300), ex["da"] / np.maximum(ex["a"], 1e-300)) + 4 * EPS)
    st_rows = keep & ~exact_within
    assert (np.abs(ref[6] - s_exact)[st_rows] <= tol[st_rows]).all()
    # every row reported within range is within range by the exact maxima of its output
    exo_v, exo_a = X.max_magnitude(t, c, 1), X.max_magnitude(t, c, 2)
    for exo, lim, k in ((exo_v, v_max, 1), (exo_a, a_max, 2)):
        slack = 1e-13 * exo["value"] + 8 * (N - 1 - k) * EPS * exo["scale"]
        assert (exo["value"][w == 1] <= lim * LIMIT + slack[w == 1]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("K", (1, 16, 50))
def test_solved_fixtures_need_one_stretch(solver, oracle, K):
    N, D, B = 10, 3, 64
    _, _, times, _, coeffs = solved_fixtures(solver, oracle, N, K, D, B, 7000 + K)
    v_max, a_max = mixed_limits(solver, times, coeffs)
    ref = check_composition(solver, times, coeffs, v_max, a_max, f"fixture K={K}")
    _, near = exact_decision(times, coeffs, v_max, a_max)
    assert (ref[5] >= 1).any()
    assert (ref[5][~near] <= 1).all(), ref[5].max()
    assert (ref[2] == 1).all()


def velocity_ramp_times(positions, v_max, a_max):
    """estimateSegmentTimesVelocityRamp (reference src/vertex.cpp:233-290), one trajectory."""
    out = []
    for i in range(positions.shape[0] - 1):
        distance = np.linalg.norm(positions[i] - positions[i + 1])
        acc_time = v_max / a_max
        acc_distance = 0.5 * v_max * acc_time
        if distance < 2.0 * acc_distance:
            t = 2.0 * np.sqrt(distance / a_max)
        else:
            t = 2.0 * acc_time + (distance - 2.0 * acc_distance) / v_max
        out.append(max(0.1, t))
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize("D,r,K,seed,bounds,v_max,a_max", __import__("test_oracle").REF_PARAMS)
def test_reference_time_scaling_assertions(solver, oracle, D, r, K, seed, bounds, v_max, a_max):
    """TimeScalingInTrajectory and TimeScaling (reference test/test_polynomial_optimization.cpp:608-729)."""
    import torch
    import mav_trajectory_generation_b200 as m
    N = 10
    pos = oracle.create_random_positions(K, D, -bounds, bounds, seed)
    prob = m.Problem(N, r, K, D)
    d_fixed = oracle.waypoint_d_fixed(N, pos[None])
    # TimeScalingInTrajectory: ramp times for (2v, 2a), solve, scale to (v, a)
    times = velocity_ramp_times(pos, 2 * v_max, 2 * a_max)[None]
    coeffs = solver.solve_linear(prob, _cuda(times), _cuda(d_fixed)).cpu().numpy()
    t, c, w, mx, st = run_scale(solver, times, coeffs, v_max, a_max)
    assert st[0] == 0
    ve, ae = exact_maxima(t, c)
    assert ve[0] <= v_max + 1e-3 and ae[0] <= a_max + 1e-3, (ve, ae)
    # TimeScaling: ramp times for (v, a), scaleSegmentTimesWithViolation, the cost does not grow
    times = velocity_ramp_times(pos, v_max, a_max)[None]
    tt, df = _cuda(times), _cuda(d_fixed)
    before = solver.compute_cost(prob, tt, solver.solve_linear(prob, tt, df))
    co, t2, w2, mx2, st2 = solver.scale_times_with_violation(prob, tt, df, v_max, a_max)
    after = solver.compute_cost(prob, t2, co)
    torch.cuda.synchronize()
    assert int(st2[0]) == 0
    assert float(after[0]) <= float(before[0])
    ve, ae = exact_maxima(t2.cpu().numpy(), co.cpu().numpy())
    assert ve[0] <= (v_max + 1e-3) * (1 + 1e-9) and ae[0] <= (a_max + 1e-3) * (1 + 1e-9), (ve, ae)


@pytest.mark.gpu
def test_scale_times_with_violation_composition(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    from test_gpu_parity import check_parity, global_rel_err
    N, r, K, D, B = 10, 4, 16, 3, 64
    prob, pos, times, d_fixed, coeffs = solved_fixtures(solver, oracle, N, K, D, B, 8000)
    v_max, a_max = mixed_limits(solver, times, coeffs)
    co, t_out, w, mx, st = solver.scale_times_with_violation(prob, _cuda(times), _cuda(d_fixed), v_max, a_max)
    t_s, c_s, w_s, mx_s, st_s = run_scale(solver, times, coeffs, v_max, a_max)
    again = solver.solve_linear(prob, t_out, _cuda(d_fixed))
    torch.cuda.synchronize()
    co, t_out = co.cpu().numpy(), t_out.cpu().numpy()
    assert np.array_equal(t_out, t_s) and np.array_equal(w.cpu().numpy(), w_s)
    assert np.array_equal(mx.cpu().numpy(), mx_s) and (st.cpu().numpy() == 0).all()
    assert np.array_equal(co, again.cpu().numpy())
    assert (t_out != times).any(axis=1).sum() >= B // 4
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, t_out, n_threads=oracle.hardware_threads())
    exact = oracle.exact_solve_batch(N, r, t_out, d_fixed)
    check_parity(co, ref, exact, "scale_times_with_violation re-solve")
    # the min-snap solution of the waypoint topology is time-scale invariant: re-solved == stretched
    assert (global_rel_err(co, c_s) <= 1e-10).all()
    # an arbitrary-mask problem (masked block kernel): composition only
    rng = np.random.RandomState(5)
    Km, Nm = 5, 8
    h = Nm // 2
    mask = (rng.rand(Km + 1, h) < 0.35).astype(np.uint8)
    mask[:, 0] = 1
    mask[0, :] = 1
    mask[-1, :] = 1
    mask[2, 1] = 1
    pm = m.Problem(Nm, h - 1, Km, 2, fixed_mask=mask)
    assert pm.kernel == m.KERNEL_GENERIC
    tm = rng.uniform(1.0, 3.0, size=(33, Km))
    dm = rng.uniform(-3, 3, size=(33, 2, pm.n_fixed))
    c0 = solver.solve_linear(pm, _cuda(tm), _cuda(dm)).cpu().numpy()
    vm, am = mixed_limits(solver, tm, c0)
    co, t_out, w, mx, st = solver.scale_times_with_violation(pm, _cuda(tm), _cuda(dm), vm, am)
    t_s, c_s, w_s, mx_s, st_s = run_scale(solver, tm, c0, vm, am)
    again = solver.solve_linear(pm, t_out, _cuda(dm))
    torch.cuda.synchronize()
    assert np.array_equal(t_out.cpu().numpy(), t_s) and np.array_equal(w.cpu().numpy(), w_s)
    assert np.array_equal(co.cpu().numpy(), again.cpu().numpy())


@pytest.mark.gpu
def test_edge_rows_and_arguments(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, K, D = 10, 4, 3
    rng = np.random.default_rng(3)
    times, coeffs = random_segments(rng, 8, K, D, N)
    bad_t = {1: 0.0, 2: -1.0, 3: np.nan, 4: np.inf, 5: -np.inf}
    for b, T in bad_t.items():
        times[b, b % K] = T
    coeffs[6, 1, 0, 3] = np.inf  # infinite maximum against an infinite limit: NaN violation, s = 1 every round
    t, c, w, mx, st = run_scale(solver, times, coeffs, np.inf, 0.5)
    for b in bad_t:
        assert st[b] == m.STATUS_BAD_TIME and w[b] == 0 and np.isnan(mx[b]).all()
        assert np.array_equal(t[b], times[b], equal_nan=True) and np.array_equal(c[b], coeffs[b])
    assert st[6] == 0 and w[6] == 0 and np.array_equal(t[6], times[6]) and np.array_equal(c[6], coeffs[6])
    check_composition(solver, times, coeffs, np.inf, 0.5, "edge rows")
    # in place == out of place
    tt, cc = _cuda(times), _cuda(coeffs)
    t2, c2, w2, mx2, st2 = solver.scale_to_constraints(tt, cc, np.inf, 0.5, seg_times_out=tt, coeffs_out=cc)
    torch.cuda.synchronize()
    assert t2.data_ptr() == tt.data_ptr()
    assert np.array_equal(tt.cpu().numpy(), t, equal_nan=True) and np.array_equal(cc.cpu().numpy(), c)
    assert np.array_equal(w2.cpu().numpy(), w) and np.array_equal(mx2.cpu().numpy(), mx, equal_nan=True)
    # a failed first solve keeps its input times
    r, Kf, B = 4, 4, 8
    pos, tf = oracle.make_waypoint_batch(Kf, D, B, base_seed=4100)
    prob = m.Problem(N, r, Kf, D)
    df = oracle.waypoint_d_fixed(N, pos)
    tf[5, 2] = np.inf  # the factorisation meets a non-finite pivot: STATUS_NOT_SPD
    co, t_out, w, mx, st = solver.scale_times_with_violation(prob, _cuda(tf), _cuda(df), 1.0, 1.0)
    torch.cuda.synchronize()
    st, w, t_out = st.cpu().numpy(), w.cpu().numpy(), t_out.cpu().numpy()
    assert st[5] & m.STATUS_NOT_SPD and st[5] & m.STATUS_BAD_TIME and w[5] == 0
    assert np.array_equal(t_out[5], tf[5]) and (st[np.arange(B) != 5] == 0).all()
    # arguments
    lib, h = solver.lib, solver.h
    out_t, out_c = torch.empty_like(tt), torch.empty_like(cc)

    def call(N_, vm, am, t_ptr=tt.data_ptr(), B_=8):
        return lib.mtg_scale_to_constraints_batch_f64(h, N_, K, D, B_, t_ptr, cc.data_ptr(), vm, am, out_t.data_ptr(),
                                                      out_c.data_ptr(), None, None, None, None)
    for vm, am in ((0.0, 1.0), (-1.0, 1.0), (np.nan, 1.0), (1.0, 0.0), (1.0, -2.0), (1.0, np.nan)):
        assert call(N, vm, am) == -1
    assert call(9, 1.0, 1.0) == -1 and call(2, 1.0, 1.0) == -1 and call(N, 1.0, 1.0, t_ptr=None) == -1
    assert call(N, 1.0, 1.0, t_ptr=None, B_=0) == 0
    p2 = m.Problem(2, 0, Kf, D)
    assert lib.mtg_scale_times_with_violation_batch_f64(h, C.byref(p2.c), B, _cuda(tf).data_ptr(), _cuda(df).data_ptr(),
                                                        1.0, 1.0, out_c.data_ptr(), out_t.data_ptr(), None, None, None,
                                                        None) == -1
    assert lib.mtg_scale_times_with_violation_batch_f64(h, C.byref(prob.c), B, _cuda(tf).data_ptr(), None, 1.0, 1.0,
                                                        out_c.data_ptr(), out_t.data_ptr(), None, None, None, None) == -1
    assert lib.mtg_scale_times_with_violation_batch_f64(h, C.byref(prob.c), B, _cuda(tf).data_ptr(),
                                                        _cuda(df).data_ptr(), np.nan, 1.0, out_c.data_ptr(),
                                                        out_t.data_ptr(), None, None, None, None) == -1


@pytest.mark.gpu
def test_tiling_rows_alone_equal_the_batch(solver, oracle):
    N, K, D, B = 10, 16, 3, 20011
    _, _, times, _, coeffs = solved_fixtures(solver, oracle, N, K, D, B, 9000)
    rng = np.random.default_rng(9)
    # rows that finish in different rounds: feasible (0 stretches), stretched once, a bad time (stops at once) and an
    # infinite coefficient against an infinite velocity limit (NaN violation: all 20 rounds)
    times[rng.choice(B, size=40, replace=False), 3] = -1.0
    inf_rows = rng.choice(B, size=40, replace=False)
    coeffs[inf_rows, 2, 1, 4] = np.inf
    v, a = gpu_maxima(solver)(times[:2000], coeffs[:2000])
    v_max, a_max = np.inf, float(np.nanquantile(a, 0.5))
    t, c, w, mx, st = run_scale(solver, times, coeffs, v_max, a_max)
    sample = rng.choice(B, size=24, replace=False)
    for b in np.concatenate([sample, inf_rows[:2]]):
        t1, c1, w1, mx1, st1 = run_scale(solver, times[b:b + 1], coeffs[b:b + 1], v_max, a_max)
        assert np.array_equal(t1[0], t[b]) and np.array_equal(c1[0], c[b]) and w1[0] == w[b]
        assert np.array_equal(mx1[0], mx[b], equal_nan=True) and st1[0] == st[b]
    part = slice(0, 3000)
    ref = replay(times[part], coeffs[part], v_max, a_max, gpu_maxima(solver))
    assert np.array_equal(ref[0], t[part], equal_nan=True) and np.array_equal(ref[1], c[part])
    assert np.array_equal(ref[2], w[part]) and np.array_equal(ref[4], st[part])
    assert {0, 1, MAX_ROUNDS} <= set(ref[5].tolist()), np.unique(ref[5])


@pytest.mark.gpu
def test_host_variants_match_device(solver, oracle):
    import torch
    N, r, K, D, B = 10, 4, 5, 3, 4099
    prob, pos, times, d_fixed, coeffs = solved_fixtures(solver, oracle, N, K, D, B, 9500)
    v_max, a_max = mixed_limits(solver, times, coeffs)
    dev = run_scale(solver, times, coeffs, v_max, a_max)
    co, t_out, w, mx, st = solver.scale_times_with_violation(prob, _cuda(times), _cuda(d_fixed), v_max, a_max)
    torch.cuda.synchronize()
    dev_nl = [x.cpu().numpy() for x in (co, t_out, w, mx, st)]
    for pinned in (False, True):
        def buf(shape, dtype=np.float64):
            a = torch.empty(shape, dtype=torch.float64 if dtype == np.float64 else torch.int32)
            return a.pin_memory() if pinned else a.numpy()
        h_t, h_c, h_w, h_m, h_s = buf((B, K)), buf((B, K, D, N)), buf((B,), np.int32), buf((B, 2)), buf((B,), np.int32)
        solver.scale_to_constraints_host(times, coeffs, v_max, a_max, h_t, h_c, h_w, h_m, h_s)
        for a, b in zip((h_t, h_c, h_w, h_m, h_s), dev):
            assert np.array_equal(np.asarray(a), b)
        # in place on host buffers
        it, ic = times.copy(), coeffs.copy()
        solver.scale_to_constraints_host(it, ic, v_max, a_max, it, ic)
        assert np.array_equal(it, dev[0]) and np.array_equal(ic, dev[1])
        h_co, h_to = buf((B, K, D, N)), buf((B, K))
        solver.scale_times_with_violation_host(prob, times, d_fixed, v_max, a_max, h_co, h_to, h_w, h_m, h_s)
        for a, b in zip((h_co, h_to, h_w, h_m, h_s), dev_nl):
            assert np.array_equal(np.asarray(a), b)


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    out = subprocess.run([build_binary()], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert " 0 failures" in out.stdout
