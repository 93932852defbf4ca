"""Batched FeasibilityRecursive::checkInputFeasibilityTrajectory (mtg_input_feasibility_recursive_batch_f64).

The exact reference is tests/feasibility_recursive_exact.cpp: binary128 roots and root values, the section walk in fp64
as the reference runs it, and a per-row decision margin (the smallest relative gap of any comparison it made, less the
error the compared values can carry).  On the CPU it is pinned to closed forms and to an mpmath replay, and the host
mirror is checked against it; on the GPU the kernel must give the replay's result and segment on every row whose margin
exceeds the root-time tolerance; at most 1 % of rows may fall under it, and they are reported."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import feasibility_oracle
import feasibility_recursive_oracle as F
from test_input_feasibility import limit_sets, reference_distribution, waypoint_fixtures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility_recursive.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility_recursive")

G = 9.81
DEFAULTS = dict(f_min=0.5 * G, f_max=1.5 * G, v_max=3.0, omega_xy_max=np.pi / 2, omega_z_max=np.pi / 2,
                omega_z_dot_max=2 * np.pi)
FEASIBLE, INDET, THRUST_HIGH, THRUST_LOW, VELOCITY, ROLL_PITCH, YAW_RATES, YAW_ACC = range(8)
REACHABLE = (FEASIBLE, INDET, THRUST_HIGH, THRUST_LOW, VELOCITY, YAW_RATES, YAW_ACC)
STATUS_BAD_TIME, STATUS_FEAS_CAPACITY = 1, 4
# the analytic check's limit sets, and three that make Indeterminable, ThrustLow and YawAcc common in the fixtures
PARITY_SETS = limit_sets(0.7) + [{"omega_xy_max": 0.05}, dict(f_min=0.95 * G, f_max=1.05 * G, v_max=2.0),
                                 {"omega_z_max": 0.5, "omega_z_dot_max": 0.05}]
# The replay's margin already has the forward error of every root value taken off; what is left must also clear the
# root times, which the GPU finds to about 1e-15 T (a double root only to sqrt(u) ~ 1e-8 T, but its value is
# stationary there).
MARGIN_BOUND = 1e-9


def build_binary():
    """The C++ driver of the host FeasibilityRecursive and the batch class
    (tests/cpp/test_input_feasibility_recursive.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


def host_mirror(times, coeffs, limits, mst, gravity=G):
    """FeasibilityRecursive of the C++ host mirror on every row: (result [B], segment [B])."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    present = sum(1 << q for q, n in enumerate(F.LIMITS) if n in limits)
    lim = np.array([float(limits.get(n, 0.0)) for n in F.LIMITS])
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([B, K, D, N, present], dtype=np.int32).tobytes())
            f.write(np.concatenate([lim, [gravity, mst]]).tobytes())
            f.write(times.tobytes())
            f.write(coeffs.tobytes())
        subprocess.check_call([build_binary(), "mirror", src, dst], timeout=600)
        out = np.fromfile(dst, dtype=np.int32)
    return out[:B], out[B:]


def _seg(N, D, rows, T):
    """One K = 1 trajectory from {dim: {power: coefficient}}."""
    c = np.zeros((1, 1, D, N))
    for d, row in rows.items():
        for j, v in row.items():
            c[0, 0, d, j] = v
    return np.array([[T]]), c


def exact(times, coeffs, limits, mst=0.05):
    return F.input_feasibility_recursive(times, coeffs, limits, mst, G)


# ---- CPU: the replay against closed forms and mpmath ---------------------------------------------------------------
@pytest.mark.parametrize("N", (4, 8, 12))
def test_replay_closed_forms(N):
    # hover: thrust g everywhere, nothing moves
    t, c = _seg(N, 3, {}, 2.0)
    assert exact(t, c, DEFAULTS)["result"][0] == FEASIBLE
    # constant z acceleration a: thrust |a + g|, out of range at the ends already
    t, c = _seg(N, 3, {2: {2: -0.3 * G}}, 2.0)  # a = -0.6 g -> 0.4 g < 0.5 g
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_LOW
    t, c = _seg(N, 3, {2: {2: 0.3 * G}}, 2.0)  # 1.6 g > 1.5 g
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_HIGH
    # constant speed 3.5 along x: the end points fail, and both sides compute them bit for bit
    t, c = _seg(N, 3, {0: {1: 3.5}}, 1.0)
    r = exact(t, c, DEFAULTS)
    assert r["result"][0] == VELOCITY and r["segment"][0] == 0 and r["margin"][0] == np.inf
    # v_x = 2.5 + 4 t - 4 t^2 on [0, 1]: 2.5 at both ends, 3.5 at the root t = 0.5 of p_x''
    t, c = _seg(N, 3, {0: {1: 2.5, 2: 2.0, 3: -4.0 / 3.0}}, 1.0)
    r = exact(t, c, {"v_max": 3.0})
    assert r["result"][0] == VELOCITY
    assert abs(r["margin"][0] - (3.5 ** 2 - 9.0) / 9.0) < 1e-12  # the single-axis speed squared against v_max^2
    assert exact(t, c, {"v_max": 3.6})["result"][0] == FEASIBLE
    # yaw rate 2 rad/s, yaw acceleration 7 rad/s^2 (D = 4); D = 3 ignores dim 3 entirely
    t, c = _seg(N, 4, {3: {1: 2.0}}, 1.0)
    assert exact(t, c, DEFAULTS)["result"][0] == YAW_RATES
    assert exact(t, c[:, :, :3].copy(), DEFAULTS)["result"][0] == FEASIBLE
    t, c = _seg(N, 4, {3: {2: 3.5}}, 0.1)  # yaw' <= 0.7, yaw'' = 7 > 2 pi
    assert exact(t, c, DEFAULTS)["result"][0] == YAW_ACC
    # a segment shorter than min_section_time is Indeterminable even with no limit at all
    t, c = _seg(N, 3, {}, 0.04)
    assert exact(t, c, {}, 0.05)["result"][0] == INDET
    assert exact(t, c, {}, 0.03)["result"][0] == FEASIBLE
    # free fall: f_min^2 = 0 makes the roll/pitch bound DBL_MAX, halved down to min_section_time
    t, c = _seg(N, 3, {2: {2: -G / 2}}, 1.0)
    assert exact(t, c, {"omega_xy_max": 1e6})["result"][0] == INDET
    # constant jerk J along x: on a section starting at t1 the bound is J / sqrt(J^2 t1^2 + g^2), J / g at t1 = 0
    # (the analytic check's sqrt(j_max / f_min) is sqrt(J / g) = 0.319 here)
    J = 1.0
    t, c = _seg(N, 3, {0: {3: J / 6}}, 2.0)
    assert exact(t, c, {"omega_xy_max": 1.02 * J / G})["result"][0] == FEASIBLE
    assert exact(t, c, {"omega_xy_max": 0.98 * J / G})["result"][0] == INDET
    assert feasibility_oracle.input_feasibility(t, c, {"omega_xy_max": 0.2}, 0.05, G)["result"][0] == INDET
    assert exact(t, c, {"omega_xy_max": 0.2})["result"][0] == FEASIBLE


def test_replay_quirks():
    N = 6
    # the end points are checked before the per-axis bounds, ThrustLow before ThrustHigh
    t, c = _seg(N, 3, {2: {2: -0.3 * G, 3: 2.2 * G / 6}}, 1.0)  # z acceleration from -0.6 g to 1.6 g
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_LOW
    assert exact(t, c, {"f_max": 1.5 * G})["result"][0] == THRUST_HIGH
    # f_i = a_i + gravity_i changes sign on x: x adds nothing to the lower bound, the row is decided by the split
    t, c = _seg(N, 3, {0: {2: 0.5, 3: -1.0 / 3.0}}, 1.0)  # a_x = 1 - 2 t
    r = exact(t, c, {"f_min": 0.5 * G, "omega_xy_max": 10.0})
    assert r["result"][0] == FEASIBLE and r["margin"][0] > MARGIN_BOUND
    # an all-zero axis: its exact comparisons do not pull the margin down
    t, c = _seg(N, 3, {0: {4: 0.01}}, 1.0)
    assert exact(t, c, DEFAULTS)["margin"][0] > MARGIN_BOUND
    # D = 2 and D = 5: Indeterminable at segment 0
    for D in (2, 5):
        t, c = _seg(N, D, {}, 1.0)
        r = exact(t, c, DEFAULTS)
        assert r["result"][0] == INDET and r["segment"][0] == 0
    # bad time: Indeterminable, segment -1
    for T in (0.0, -1.0, np.nan, np.inf):
        t, c = _seg(N, 3, {}, T)
        r = exact(t, c, DEFAULTS)
        assert r["result"][0] == INDET and r["segment"][0] == -1


def _mp_replay(c, T, limits, mst, mp):
    """An independent replay with mpmath.polyroots (50 digits) and mpmath values for one K = 1, D = 3 or 4 segment;
    the section ends are fp64 as in the reference."""
    mp.mp.dps = 50
    D, N = c.shape

    def poly(d, k):
        p = [mp.mpf(0)] * max(N - k, 1)
        for j in range(N - k):
            f = mp.mpf(1)
            for w in range(k):
                f *= j + k - w
            p[j] = f * mp.mpf(float(c[d, j + k]))
        return p

    def ev(p, t):
        a = mp.mpf(0)
        for x in reversed(p):
            a = a * t + x
        return a

    def roots(p):
        g = [j * p[j] for j in range(1, len(p))]
        while g and g[-1] == 0:
            g.pop()
        out = []
        if len(g) >= 2:
            for r in mp.polyroots(list(reversed(g)), maxsteps=400, extraprec=400):
                if abs(mp.im(r)) < mp.mpf(10) ** -30 and 0 <= mp.re(r) <= T:
                    out.append(mp.re(r))
        return out

    if D not in (3, 4):
        return INDET
    P = {k: [poly(i, k) for i in range(3)] for k in (1, 2, 3)}
    R = {k: [roots(p) for p in P[k]] for k in (1, 2, 3)}
    grav = [0, 0, G]
    has = {n: n in limits for n in F.LIMITS}

    def minmax(k, i, t1, t2):
        vs = [ev(P[k][i], t1), ev(P[k][i], t2)] + [ev(P[k][i], r) for r in R[k][i] if t1 <= r <= t2]
        return min(vs), max(vs)

    def walk(t1, t2):
        if t2 - t1 < mst:
            return INDET
        if has["f_min"] or has["f_max"]:
            f = [mp.sqrt(sum((ev(P[2][i], t) + grav[i]) ** 2 for i in range(3))) for t in (t1, t2)]
            if has["f_min"] and min(f) < limits["f_min"]:
                return THRUST_LOW
            if has["f_max"] and max(f) > limits["f_max"]:
                return THRUST_HIGH
        if has["v_max"] and max(mp.sqrt(sum(ev(P[1][i], t) ** 2 for i in range(3))) for t in (t1, t2)) > \
                limits["v_max"]:
            return VELOCITY
        f_min_sqr = f_max_sqr = v_max_sqr = j_max_sqr = mp.mpf(0)
        if has["v_max"]:
            for i in range(3):
                lo, hi = minmax(1, i, t1, t2)
                if max(lo ** 2, hi ** 2) > limits["v_max"] ** 2:
                    return VELOCITY
                v_max_sqr += max(abs(lo), abs(hi)) ** 2
        if has["f_min"] or has["f_max"] or has["omega_xy_max"]:
            for i in range(3):
                lo, hi = minmax(2, i, t1, t2)
                lo, hi = lo + grav[i], hi + grav[i]
                if has["f_max"] and max(abs(lo), abs(hi)) > limits["f_max"]:
                    return THRUST_HIGH
                if not lo * hi < 0:
                    f_min_sqr += min(abs(lo), abs(hi)) ** 2
                f_max_sqr += max(abs(lo), abs(hi)) ** 2
        if has["omega_xy_max"]:
            for i in range(3):
                lo, hi = minmax(3, i, t1, t2)
                j_max_sqr += max(abs(lo), abs(hi)) ** 2
        f_lower, f_upper, v_upper = mp.sqrt(f_min_sqr), mp.sqrt(f_max_sqr), mp.sqrt(v_max_sqr)
        omega = mp.sqrt(j_max_sqr / f_min_sqr) if f_min_sqr > 1e-6 else mp.mpf(np.finfo(float).max)
        if has["f_min"] and f_upper < limits["f_min"]:
            return THRUST_LOW
        if has["f_max"] and f_lower > limits["f_max"]:
            return THRUST_HIGH
        if (has["f_min"] and f_lower < limits["f_min"]) or (has["f_max"] and f_upper > limits["f_max"]) or \
                (has["v_max"] and v_upper > limits["v_max"]) or \
                (has["omega_xy_max"] and omega > limits["omega_xy_max"]):
            h = (t1 + t2) / 2
            r = walk(t1, h)
            return r if r != FEASIBLE else walk(h, t2)
        return FEASIBLE

    r = walk(0.0, float(T))
    if r != FEASIBLE or D != 4:
        return r
    for k, name, code in ((1, "omega_z_max", YAW_RATES), (2, "omega_z_dot_max", YAW_ACC)):
        if name in limits:
            p = poly(3, k)
            if max(abs(ev(p, t)) for t in [0, T] + roots(p)) > limits[name]:
                return code
    return FEASIBLE


def test_replay_against_mpmath():
    mp = pytest.importorskip("mpmath")
    rng = np.random.default_rng(43)
    checked = 0
    for i in range(24):
        N = (6, 8, 10)[i % 3]
        D = 3 + i % 2
        T = float(rng.uniform(0.3, 1.5))
        c = rng.normal(size=(D, N)) / np.maximum(1.0, np.arange(N)) ** 2 * np.array([1, 1, 1, 0.5][:D])[:, None]
        limits = limit_sets(0.8)[i % 9]
        mst = (0.05, 0.10)[i % 2]
        r = exact(np.array([[T]]), c[None, None], limits, mst)
        if r["margin"][0] < 1e-9:
            continue
        assert r["result"][0] == _mp_replay(c, T, limits, mst, mp), (i, limits)
        checked += 1
    assert checked >= 20


def test_host_mirror_matches_replay():
    """The single-object FeasibilityRecursive (host roots, no GPU) against the replay on margin-clear rows."""
    import oracle_lib as O
    checked = 0
    for N, K, D in ((6, 3, 3), (10, 4, 4), (12, 2, 3)):
        pos, times = O.make_waypoint_batch(K, D, 48, base_seed=900 + N)
        coeffs, _ = O.solve_waypoint_batch(N, N // 2 - 1, pos, times)
        for i, limits in enumerate(limit_sets(0.7)):
            mst = (0.01, 0.05, 0.10)[i % 3]
            r, s = host_mirror(times, coeffs, limits, mst)
            ex = exact(times, coeffs, limits, mst)
            ok = ex["margin"] > MARGIN_BOUND
            assert np.array_equal(r[ok], ex["result"][ok]), (N, limits)
            assert np.array_equal(s[ok], ex["segment"][ok]), (N, limits)
            checked += int(ok.sum())
    t, c = _seg(6, 3, {}, 0.04)  # quirks: T < min_section_time without limits, D = 5
    assert host_mirror(t, c, {}, 0.05)[0][0] == INDET
    t, c = _seg(6, 5, {}, 1.0)
    assert host_mirror(t, c, DEFAULTS, 0.05)[0][0] == INDET
    assert checked >= 1000


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def solver():
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


def gpu_check(solver, times, coeffs, limits, mst=0.05, analytic=False):
    import torch
    fn = solver.check_input_feasibility if analytic else solver.check_input_feasibility_recursive
    r, s, st = fn(_cuda(times), _cuda(coeffs), limits, mst, G)
    torch.cuda.synchronize()
    return r.cpu().numpy(), s.cpu().numpy(), st.cpu().numpy()


def check_parity(solver, times, coeffs, limits, mst, what, counts=None):
    r, s, st = gpu_check(solver, times, coeffs, limits, mst)
    ex = exact(times, coeffs, limits, mst)
    ok = ex["margin"] > MARGIN_BOUND
    bad = np.nonzero(ok & ((r != ex["result"]) | (s != ex["segment"])))[0]
    assert bad.size == 0, (f"{what}: rows {bad[:8]} gpu {r[bad[:8]]}/{s[bad[:8]]} exact {ex['result'][bad[:8]]}/"
                           f"{ex['segment'][bad[:8]]} margin {ex['margin'][bad[:8]]}")
    assert np.all(st[np.isfinite(times).all(axis=1) & (times > 0).all(axis=1)] == 0), what
    under = int((~ok).sum())
    if under:
        print(f"{what}: {under}/{len(r)} rows within the margin bound")
    if counts is not None:
        for code in range(8):
            counts[code] = counts.get(code, 0) + int((r == code).sum())
    return under, len(r)


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 6, 8, 10, 12))
def test_parity_with_binary128_replay(solver, N):
    under = total = 0
    counts = {}
    for D in (3, 4):
        for K in (1, 3, 16, 50):
            B = {1: 96, 3: 48, 16: 12, 50: 6}[K]
            times, coeffs = waypoint_fixtures(solver, N, K, D, B, 50000 + 100 * N + 10 * D + K)
            for i, limits in enumerate(PARITY_SETS):
                mst = (0.01, 0.05, 0.10)[i % 3]
                u, t = check_parity(solver, times, coeffs, limits, mst, f"N={N} D={D} K={K} set {i}", counts)
                under += u
                total += t
    print(f"N={N}: {under}/{total} rows within the margin bound; results {counts}")
    assert under <= 0.01 * total
    assert counts.get(ROLL_PITCH, 0) == 0
    for code in REACHABLE:
        assert counts.get(code, 0) > 0, (N, code, counts)


@pytest.mark.gpu
def test_reference_distribution_and_cross_checker_property(solver):
    times, coeffs = reference_distribution(solver, 8192, 7654321)
    counts = {}
    under = total = 0
    sets = [dict(DEFAULTS), dict(DEFAULTS, f_min=0.9 * G), dict(DEFAULTS, f_max=1.05 * G, f_min=0.5 * G),
            {"v_max": 1.5}, {"omega_z_max": 1.0}, {"omega_z_dot_max": 1.0}, {"omega_xy_max": 1.0}, {}]
    for i, limits in enumerate(sets):
        for mst in (0.01, 0.05, 0.10):
            u, t = check_parity(solver, times, coeffs, limits, mst, f"reference set {i} mst {mst}", counts)
            under += u
            total += t
    print(f"reference distribution: {under}/{total} rows within the margin bound; results {counts}")
    assert under <= 0.01 * total
    for code in REACHABLE:
        assert counts.get(code, 0) >= 20, (code, counts)
    assert counts.get(ROLL_PITCH, 0) == 0
    # the reference test's cross-check: FeasibilityAnalytic Feasible at 0.01 => FeasibilityRecursive Feasible or
    # Indeterminable at 0.01, 0.05 and 0.10 (on the rows both replays decide clear of rounding)
    analytic = gpu_check(solver, times, coeffs, DEFAULTS, 0.01, analytic=True)[0]
    clear_a = feasibility_oracle.input_feasibility(times, coeffs, DEFAULTS, 0.01, G)["margin"] > MARGIN_BOUND
    assert (analytic[clear_a] == FEASIBLE).sum() >= 100
    for mst in (0.01, 0.05, 0.10):
        rec = gpu_check(solver, times, coeffs, DEFAULTS, mst)[0]
        rows = (analytic == FEASIBLE) & clear_a & (exact(times, coeffs, DEFAULTS, mst)["margin"] > MARGIN_BOUND)
        assert np.all(np.isin(rec[rows], (FEASIBLE, INDET))), mst


@pytest.mark.gpu
def test_feasible_rows_keep_limits_on_dense_samples(solver):
    """GPU Feasible => thrust, |v|, |yaw'|, |yaw''| and Mueller's |p'''| / |p'' + g| within the limits on 1 ms samples
    (relative 1e-9)."""
    import torch
    times, coeffs = reference_distribution(solver, 512, 99)
    limits = dict(DEFAULTS, v_max=2.5)
    r = gpu_check(solver, times, coeffs, limits)[0]
    assert (r == FEASIBLE).sum() >= 20
    rows = np.nonzero(r == FEASIBLE)[0]
    t, c = _cuda(times[rows]), _cuda(coeffs[rows])
    n = int(np.ceil(times[rows].max() / 1e-3)) + 1
    samples = {k: solver.evaluate(t, c, k, 0.0, 1e-3, n) for k in (1, 2, 3)}
    torch.cuda.synchronize()
    v, a, j = (samples[k].cpu().numpy() for k in (1, 2, 3))
    valid = (np.arange(n)[None, :] * 1e-3) <= times[rows]
    tol = 1 + 1e-9
    speed = np.linalg.norm(v[:, :, :3], axis=2)
    thrust = np.linalg.norm(a[:, :, :3] + np.array([0, 0, G]), axis=2)
    jerk = np.linalg.norm(j[:, :, :3], axis=2)
    assert np.all(speed[valid] <= limits["v_max"] * tol)
    assert np.all(thrust[valid] <= limits["f_max"] * tol) and np.all(thrust[valid] >= limits["f_min"] / tol)
    assert np.all(np.abs(v[:, :, 3][valid]) <= limits["omega_z_max"] * tol)
    assert np.all(np.abs(a[:, :, 3][valid]) <= limits["omega_z_dot_max"] * tol)
    assert np.all(jerk[valid] / thrust[valid] <= limits["omega_xy_max"] * tol)


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 8, 12))
def test_quirk_rows(solver, N):
    cases = []  # (times, coeffs, limits, mst, result, segment)
    t, c = _seg(N, 3, {}, 0.04)
    cases.append((t, c, {}, 0.05, INDET, 0))  # T < min_section_time, no limit at all
    cases.append((t, c, {"v_max": 1.0}, 0.05, INDET, 0))
    cases.append((t, c, {}, 0.03, FEASIBLE, -1))
    t, c = _seg(N, 3, {2: {2: -G / 2}}, 1.0)  # free fall: f_min^2 <= 1e-6
    cases.append((t, c, {"omega_xy_max": 1e6}, 0.05, INDET, 0))
    t, c = _seg(N, 3, {2: {2: -0.3 * G, 3: 2.2 * G / 6}}, 1.0)  # ThrustLow wins over ThrustHigh
    cases.append((t, c, DEFAULTS, 0.05, THRUST_LOW, 0))
    t, c = _seg(N, 3, {2: {2: -0.3 * G}}, 1.0)  # omega_xy alone: thrust 0.4 g is no ThrustLow without f_min
    cases.append((t, c, {"omega_xy_max": 10.0}, 0.05, FEASIBLE, -1))
    t, c = _seg(N, 3, {0: {1: 3.5}}, 1.0)
    cases.append((t, c, DEFAULTS, 0.05, VELOCITY, 0))
    J = 1.0
    t, c = _seg(N, 3, {0: {3: J / 6}}, 2.0)  # constant jerk: the bound is J / g at t1 = 0
    cases.append((t, c, {"omega_xy_max": 1.02 * J / G}, 0.05, FEASIBLE, -1))
    cases.append((t, c, {"omega_xy_max": 0.98 * J / G}, 0.05, INDET, 0))
    t, c = _seg(N, 4, {3: {1: 2.0}}, 1.0)
    cases.append((t, c, DEFAULTS, 0.05, YAW_RATES, 0))
    t, c = _seg(N, 4, {3: {2: 3.5}}, 0.1)
    cases.append((t, c, DEFAULTS, 0.05, YAW_ACC, 0))
    t, c = _seg(N, 4, {3: {1: 2.0}, 2: {2: -0.3 * G}}, 1.0)  # the recursion's ThrustLow comes before the yaw checks
    cases.append((t, c, DEFAULTS, 0.05, THRUST_LOW, 0))
    if N >= 6:
        # one axis above v_max at an interior root of p_x'' only
        t, c = _seg(N, 3, {0: {1: 2.5, 2: 2.0, 3: -4.0 / 3.0}}, 1.0)
        cases.append((t, c, {"v_max": 3.0}, 0.05, VELOCITY, 0))
        cases.append((t, c, {"v_max": 3.6}, 0.05, FEASIBLE, -1))
    for D in (2, 5):
        t, c = _seg(N, D, {}, 1.0)
        cases.append((t, c, DEFAULTS, 0.05, INDET, 0))
    for T in (0.0, -0.0, -1.0, np.nan, np.inf, -np.inf):
        t, c = _seg(N, 3, {}, T)
        cases.append((t, c, DEFAULTS, 0.05, INDET, -1))
    for t, c, limits, mst, want_r, want_s in cases:
        r, s, st = gpu_check(solver, t, c, limits, mst)
        ex = exact(t, c, limits, mst)
        what = (N, limits, mst, t[0, 0])
        assert ex["result"][0] == want_r and ex["segment"][0] == want_s, what
        assert r[0] == want_r and s[0] == want_s, what
        bad_time = not (np.isfinite(t[0, 0]) and t[0, 0] > 0)
        assert st[0] == (STATUS_BAD_TIME if bad_time else 0), what


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 12))
def test_level_cap(solver, N):
    """Free fall splits every section: at a min_section_time below T / 2^64 the walk reaches its 64 levels and the
    row is Indeterminable with MTG_STATUS_FEAS_CAPACITY; the replay, without a cap, also ends Indeterminable."""
    t, c = _seg(N, 3, {2: {2: -G / 2}}, 1.0)
    r, s, st = gpu_check(solver, t, c, {"omega_xy_max": 1.0}, 1e-30)
    assert (r[0], s[0], st[0]) == (INDET, 0, STATUS_FEAS_CAPACITY)
    assert exact(t, c, {"omega_xy_max": 1.0}, 1e-30)["result"][0] == INDET
    r, s, st = gpu_check(solver, t, c, {"omega_xy_max": 1.0}, 1e-18)  # 2^-60 < 1e-18: 60 levels suffice
    assert (r[0], s[0], st[0]) == (INDET, 0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("N", (6, 10))
def test_row_equals_first_failing_segment(solver, N):
    """A K-segment row equals the first non-Feasible result of its segments run as K = 1 rows, bit for bit."""
    for D in (3, 4):
        K = 16
        times, coeffs = waypoint_fixtures(solver, N, K, D, 24, 60000 + N + D)
        times[3, 5] = np.nan
        for limits in limit_sets(0.7)[:6]:
            r, s, st = gpu_check(solver, times, coeffs, limits, 0.05)
            r1, s1, st1 = gpu_check(solver, times.reshape(-1, 1), coeffs.reshape(-1, 1, D, N), limits, 0.05)
            r1, st1 = r1.reshape(-1, K), st1.reshape(-1, K)
            for b in range(times.shape[0]):
                if st1[b].any():
                    assert r[b] == INDET and s[b] == -1 and st[b] == STATUS_BAD_TIME
                    continue
                fail = np.nonzero(r1[b] != FEASIBLE)[0]
                want = (r1[b, fail[0]], fail[0]) if fail.size else (FEASIBLE, -1)
                assert (r[b], s[b]) == want, (b, limits)


@pytest.mark.gpu
def test_host_twin_and_refusals(solver):
    import torch
    import mav_trajectory_generation_b200.capi as capi
    N, K, D, B = 10, 5, 4, 300
    times, coeffs = waypoint_fixtures(solver, N, K, D, B, 70000)
    times[7, 2] = 0.0
    lib = solver.lib
    for limits in (DEFAULTS, {"omega_xy_max": 2.0}, {}):
        r, s, st = gpu_check(solver, times, coeffs, limits)
        hr, hs, hst = (np.full(B, -7, dtype=np.int32) for _ in range(3))
        solver.check_input_feasibility_recursive_host(times, coeffs, limits, hr, hs, hst, 0.05, G)
        assert np.array_equal(hr, r) and np.array_equal(hs, s) and np.array_equal(hst, st)
        hr2 = np.full(B, -7, dtype=np.int32)
        solver.check_input_feasibility_recursive_host(times, coeffs, limits, hr2, None, None, 0.05, G)
        assert np.array_equal(hr2, r)
        dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        ic = capi.input_constraints(limits, 0.05, G)
        tt, cc = _cuda(times), _cuda(coeffs)
        assert lib.mtg_input_feasibility_recursive_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(),
                                                             C.byref(ic), dr.data_ptr(), None, None, None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(dr.cpu().numpy(), r)
    # every refusal of the analytic entry: MTG_ERR_BAD_ARG, no launch, outputs untouched
    bad = [dict(limits={"v_max": np.nan}), dict(limits={"f_min": -1.0}), dict(limits={"omega_xy_max": -0.5}),
           dict(limits=DEFAULTS, gravity=np.nan), dict(limits=DEFAULTS, gravity=np.inf),
           dict(limits=DEFAULTS, mst=0.0), dict(limits=DEFAULTS, mst=-0.05), dict(limits=DEFAULTS, mst=np.inf),
           dict(limits=DEFAULTS, mst=np.nan)]
    tt, cc = _cuda(times), _cuda(coeffs)
    ics = [capi.input_constraints(case["limits"], case.get("mst", 0.05), case.get("gravity", G)) for case in bad]
    extra = capi.input_constraints(DEFAULTS)
    extra.present |= 1 << 6
    ics.append(extra)
    shapes = [(N, K, D, B)] * len(ics) + [(n_bad, K, D, B) for n_bad in (2, 5, 14)] + [(N, 0, D, B), (N, K, 0, B)]
    ics += [capi.input_constraints(DEFAULTS)] * 5
    for (n, k, d, b), ic in zip(shapes, ics):
        for dev_entry, host_entry in (("mtg_input_feasibility_batch_f64", "mtg_input_feasibility_batch_host_f64"),
                                      ("mtg_input_feasibility_recursive_batch_f64",
                                       "mtg_input_feasibility_recursive_batch_host_f64")):
            before = solver.launch_count
            dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
            assert getattr(lib, dev_entry)(solver.h, n, k, d, b, tt.data_ptr(), cc.data_ptr(), C.byref(ic),
                                           dr.data_ptr(), None, None, None) == -1, (dev_entry, n, k, d)
            hr = np.full(B, -7, dtype=np.int32)
            assert getattr(lib, host_entry)(solver.h, n, k, d, b, times.ctypes.data, coeffs.ctypes.data, C.byref(ic),
                                            hr.ctypes.data, None, None) == -1, (host_entry, n, k, d)
            torch.cuda.synchronize()
            assert solver.launch_count == before and (dr.cpu().numpy() == -7).all() and (hr == -7).all()
    # +inf limits never fail
    r = gpu_check(solver, times, coeffs, {k: (0.0 if k == "f_min" else np.inf) for k in DEFAULTS})[0]
    assert np.all(r[np.arange(B) != 7] == FEASIBLE)


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    """BatchPolynomialOptimization<10>::checkInputFeasibilityRecursive against the host FeasibilityRecursive, both
    against the replay, on the rows whose margin is clear of rounding."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "batch.bin")
        out = subprocess.run([build_binary(), "batch", path], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
        raw = open(path, "rb").read()
    B, K, D, N = np.frombuffer(raw[:16], dtype=np.int32)
    o = 16
    times = np.frombuffer(raw[o:o + 8 * B * K], dtype=np.float64).reshape(B, K)
    o += 8 * B * K
    coeffs = np.frombuffer(raw[o:o + 8 * B * K * D * N], dtype=np.float64).reshape(B, K, D, N)
    o += 8 * B * K * D * N
    br, bs, hr, hs = np.frombuffer(raw[o:], dtype=np.int32).reshape(4, B)
    ex = exact(times, coeffs, DEFAULTS, 0.05)
    ok = ex["margin"] > MARGIN_BOUND
    assert ok.sum() >= 0.9 * B
    for name, r, s in (("batch", br, bs), ("host", hr, hs)):
        assert np.array_equal(r[ok], ex["result"][ok]), name
        assert np.array_equal(s[ok], ex["segment"][ok]), name
    assert np.array_equal(br[ok], hr[ok]) and np.array_equal(bs[ok], hs[ok])
