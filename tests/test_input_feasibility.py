"""Batched FeasibilityAnalytic::checkInputFeasibilityTrajectory (mtg_input_feasibility_batch_f64).

The exact reference is tests/feasibility_exact.cpp: binary128 roots and values, the roll/pitch walk in fp64 as the
reference runs it, and a per-row decision margin (the smallest relative gap of any comparison it made).  On the CPU it
is pinned to closed forms and to an mpmath replay; on the GPU the kernel must give the replay's result and segment on
every row whose margin (less the fp64 evaluation's forward error) exceeds the root-time tolerance; fewer than 1 % of
rows may fall under it, and they are reported."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import feasibility_oracle as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility")

G = 9.81
DEFAULTS = dict(f_min=0.5 * G, f_max=1.5 * G, v_max=3.0, omega_xy_max=np.pi / 2, omega_z_max=np.pi / 2,
                omega_z_dot_max=2 * np.pi)
FEASIBLE, INDET, THRUST_HIGH, THRUST_LOW, VELOCITY, ROLL_PITCH, YAW_RATES, YAW_ACC = range(8)


def limit_sets(scale=1.0):
    """The defaults, each limit alone, none at all, and tightened / loosened sets."""
    sets = [dict(DEFAULTS), {}]
    sets += [{k: v} for k, v in DEFAULTS.items()]
    sets.append({k: (v * scale if k != "f_min" else v / scale) for k, v in DEFAULTS.items()})
    sets.append(dict(f_min=0.9 * G, f_max=1.1 * G, v_max=1.5, omega_xy_max=4.0, omega_z_max=0.5, omega_z_dot_max=1.0))
    sets.append(dict(v_max=2.0, omega_z_max=1.0, omega_z_dot_max=2.0, omega_xy_max=20.0))
    return sets


def build_binary():
    """The C++ driver of the host FeasibilityAnalytic and the batch class (tests/cpp/test_input_feasibility.cpp)."""
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
    """FeasibilityAnalytic of the C++ host mirror on every row: (result [B], segment [B])."""
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
    return F.input_feasibility(times, coeffs, limits, mst, G)


# ---- CPU: the replay against closed forms and mpmath ---------------------------------------------------------------
@pytest.mark.parametrize("N", (4, 8, 12))
def test_replay_closed_forms(N):
    # hover: thrust g everywhere, nothing moves
    t, c = _seg(N, 3, {}, 2.0)
    assert exact(t, c, DEFAULTS)["result"][0] == FEASIBLE
    # constant z acceleration a: thrust |a + g|
    t, c = _seg(N, 3, {2: {2: -0.3 * G}}, 2.0)  # a = -0.6 g -> 0.4 g < 0.5 g
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_LOW
    t, c = _seg(N, 3, {2: {2: 0.3 * G}}, 2.0)  # 1.6 g > 1.5 g
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_HIGH
    # z acceleration ramps from -0.6 g to 1.6 g: ThrustLow is checked first
    t, c = _seg(N, 3, {2: {2: -0.3 * G, 3: 2.2 * G / 6}}, 1.0)
    assert exact(t, c, DEFAULTS)["result"][0] == THRUST_LOW
    assert exact(t, c, {"f_max": 1.5 * G})["result"][0] == THRUST_HIGH
    # constant speed 3.5 along x
    t, c = _seg(N, 3, {0: {1: 3.5}}, 1.0)
    r = exact(t, c, DEFAULTS)
    assert r["result"][0] == VELOCITY and r["segment"][0] == 0
    assert abs(r["margin"][0] - 0.5 / 3.0) < 1e-12  # the smallest gap: |v| against v_max, less rounding
    # yaw rate 2 rad/s, yaw acceleration 7 rad/s^2 (D = 4); D = 3 ignores dim 3 entirely
    t, c = _seg(N, 4, {3: {1: 2.0}}, 1.0)
    assert exact(t, c, DEFAULTS)["result"][0] == YAW_RATES
    t, c = _seg(N, 4, {3: {2: 3.5}}, 0.1)  # yaw' <= 0.7, yaw'' = 7 > 2 pi
    assert exact(t, c, DEFAULTS)["result"][0] == YAW_ACC
    t, c = _seg(N, 4, {3: {1: 2.0}}, 1.0)
    assert exact(t, c[:, :, :3].copy(), DEFAULTS)["result"][0] == FEASIBLE
    # constant jerk J along x: f_min = g at t = 0, j_max = J, bound sqrt(J / g)
    J = 1.0
    t, c = _seg(N, 3, {0: {3: J / 6}}, 2.0)
    assert exact(t, c, {"omega_xy_max": 0.5})["result"][0] == FEASIBLE  # sqrt(1 / 9.81) = 0.319
    r = exact(t, c, {"omega_xy_max": 0.3})  # never below: halved down to min_section_time
    assert r["result"][0] == INDET
    assert abs(r["margin"][0] - (np.sqrt(J / G) - 0.3) / 0.3) < 1e-12


def test_replay_quirks():
    N = 6
    # a segment shorter than min_section_time is Indeterminable as soon as omega_xy is present
    t, c = _seg(N, 3, {}, 0.04)
    assert exact(t, c, {"omega_xy_max": 1.0}, 0.05)["result"][0] == INDET
    assert exact(t, c, {"v_max": 1.0}, 0.05)["result"][0] == FEASIBLE
    # f_min <= 1e-6 (free fall everywhere): the bound is DBL_MAX, split down to min_section_time
    t, c = _seg(N, 3, {2: {2: -G / 2}, 0: {3: 1e-3}}, 1.0)
    assert exact(t, c, {"omega_xy_max": 1e6}, 0.05)["result"][0] == INDET
    # no jerk at all: bound 0, feasible at the root
    t, c = _seg(N, 3, {0: {2: 1.0}}, 1.0)
    assert exact(t, c, {"omega_xy_max": 1e-3}, 0.05)["result"][0] == FEASIBLE
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
    """An independent replay with mpmath.polyroots (50 digits) for one K = 1, D = 3 or 4 segment."""
    mp.mp.dps = 50
    N = c.shape[1]
    D = c.shape[0]

    def poly(d, k, lift=0.0):
        p = [mp.mpf(0)] * (N - k)
        for j in range(N - k):
            f = mp.mpf(1)
            for w in range(k):
                f *= j + k - w
            p[j] = f * mp.mpf(float(c[d, j + k]))
        p[0] += mp.mpf(lift)
        return p

    def ev(p, t):
        a = mp.mpf(0)
        for x in reversed(p):
            a = a * t + x
        return a

    def dp(p):
        return [j * p[j] for j in range(1, len(p))] or [mp.mpf(0)]

    def cands(ps):
        if len(ps) == 1:
            g = dp(ps[0])
        else:
            g = [mp.mpf(0)] * (2 * len(ps[0]))
            for p in ps:
                q = dp(p)
                for a in range(len(p)):
                    for j in range(len(q)):
                        g[a + j] += p[a] * q[j]
        while g and g[-1] == 0:
            g.pop()
        ts = [mp.mpf(0), mp.mpf(T)]
        if len(g) >= 2:
            for r in mp.polyroots(list(reversed(g)), maxsteps=400, extraprec=400):
                if abs(mp.im(r)) < mp.mpf(10) ** -30 and 0 <= mp.re(r) <= T:
                    ts.append(mp.re(r))
        return [(t, mp.sqrt(sum(ev(p, t) ** 2 for p in ps))) for t in ts]

    if D not in (3, 4):
        return INDET
    th = []
    if any(k in limits for k in ("f_min", "f_max", "omega_xy_max")):
        th = cands([poly(d, 2, G if d == 2 else 0.0) for d in range(3)])
        if "f_min" in limits and min(v for _, v in th) < limits["f_min"]:
            return THRUST_LOW
        if "f_max" in limits and max(v for _, v in th) > limits["f_max"]:
            return THRUST_HIGH
    if "v_max" in limits and max(v for _, v in cands([poly(d, 1) for d in range(3)])) > limits["v_max"]:
        return VELOCITY
    if D == 4:
        if "omega_z_max" in limits and max(v for _, v in cands([poly(3, 1)])) > limits["omega_z_max"]:
            return YAW_RATES
        if "omega_z_dot_max" in limits and max(v for _, v in cands([poly(3, 2)])) > limits["omega_z_dot_max"]:
            return YAW_ACC
    if "omega_xy_max" not in limits:
        return FEASIBLE
    jk = cands([poly(d, 3) for d in range(3)])
    lim = limits["omega_xy_max"]

    def walk(t1, t2):
        if t2 - t1 < mst:
            return INDET
        fs = [v for t, v in th if t1 <= t <= t2]
        js = [v for t, v in jk if t1 <= t <= t2]
        f_min = min(fs) if fs else mp.mpf(np.finfo(float).max)
        if not f_min > 1e-6:
            split = True
        elif not js:
            split = False
        else:
            split = mp.sqrt(max(js) / f_min) > lim
        if not split:
            return FEASIBLE
        h = (t1 + t2) / 2
        r = walk(t1, h)
        return r if r != FEASIBLE else walk(h, t2)

    return walk(0.0, float(T))


def test_replay_against_mpmath():
    mp = pytest.importorskip("mpmath")
    rng = np.random.default_rng(42)
    checked = 0
    for i in range(24):
        N = (6, 8, 10)[i % 3]
        D = 3 + i % 2
        T = float(rng.uniform(0.3, 2.0))
        c = rng.normal(size=(D, N)) / np.maximum(1.0, np.arange(N)) ** 2 * np.array([1, 1, 1, 0.5][:D])[:, None]
        limits = limit_sets(0.8)[i % 9]
        r = exact(np.array([[T]]), c[None, None], limits, 0.05)
        if r["margin"][0] < 1e-9:
            continue
        assert r["result"][0] == _mp_replay(c, T, limits, 0.05, mp), (i, limits)
        checked += 1
    assert checked >= 20


def test_host_mirror_matches_replay():
    """The single-object FeasibilityAnalytic (host roots, no GPU) against the replay on margin-clear rows."""
    import oracle_lib as O
    checked = 0
    for N, K, D in ((6, 3, 3), (10, 4, 4), (12, 2, 3)):
        pos, times = O.make_waypoint_batch(K, D, 48, base_seed=700 + N)
        coeffs, _ = O.solve_waypoint_batch(N, N // 2 - 1, pos, times)
        for i, limits in enumerate(limit_sets(0.7)):
            mst = (0.01, 0.05, 0.10)[i % 3]
            r, s = host_mirror(times, coeffs, limits, mst)
            ex = exact(times, coeffs, limits, mst)
            ok = ex["margin"] > MARGIN_BOUND
            assert np.array_equal(r[ok], ex["result"][ok]), (N, limits)
            assert np.array_equal(s[ok], ex["segment"][ok]), (N, limits)
            checked += int(ok.sum())
    t, c = _seg(6, 3, {}, 0.04)  # quirks: T < min_section_time, D = 5, bad time
    assert host_mirror(t, c, {"omega_xy_max": 1.0}, 0.05)[0][0] == INDET
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


def gpu_check(solver, times, coeffs, limits, mst=0.05):
    import torch
    r, s, st = solver.check_input_feasibility(_cuda(times), _cuda(coeffs), limits, mst, G)
    torch.cuda.synchronize()
    return r.cpu().numpy(), s.cpu().numpy(), st.cpu().numpy()


# The replay's margin already has the fp64 evaluation's forward error taken off every value comparison; what is left
# must also clear the root times, which the GPU finds to about 1e-15 T (a double root only to sqrt(u) ~ 1e-8 T, but its
# side of a boundary rarely matters).
MARGIN_BOUND = 1e-9


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


def waypoint_fixtures(solver, N, K, D, B, seed):
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=seed)
    prob = m.Problem(N, N // 2 - 1, K, D)
    coeffs = solver.solve_linear(prob, _cuda(times), _cuda(O.waypoint_d_fixed(N, pos)))
    torch.cuda.synchronize()
    return times, coeffs.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 6, 8, 10, 12))
def test_parity_with_binary128_replay(solver, N):
    under = total = 0
    counts = {}
    for D in (3, 4):
        for K in (1, 3, 16, 50):
            B = {1: 96, 3: 48, 16: 12, 50: 6}[K]
            times, coeffs = waypoint_fixtures(solver, N, K, D, B, 20000 + 100 * N + 10 * D + K)
            for i, limits in enumerate(limit_sets(0.7)):
                mst = (0.01, 0.05, 0.10)[i % 3]
                u, t = check_parity(solver, times, coeffs, limits, mst, f"N={N} D={D} K={K} set {i}", counts)
                under += u
                total += t
    print(f"N={N}: {under}/{total} rows within the margin bound; results {counts}")
    assert under <= 0.01 * total
    assert counts.get(ROLL_PITCH, 0) == 0


def reference_distribution(solver, B, seed):
    """tests/test_feasibility.cpp's segments: N = 12, K = 1, a 3-D snap solve between random points in [-5, 5] with
    random start and end velocities, plus a 1-D yaw solve in [-3 pi, 3 pi] (angular acceleration) as dim 3."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.default_rng(seed)
    N = 12
    p0, p1 = rng.uniform(-5, 5, (B, 3)), rng.uniform(-5, 5, (B, 3))

    def vel():
        d = rng.uniform(0.01, 1.0, (B, 3))
        return d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.0, 2.0, (B, 1))

    v0, v1 = vel(), vel()
    T = np.linalg.norm(p1 - p0, axis=1) / rng.uniform(0.5, 2.0, B)
    T = np.maximum(T, 1e-3)[:, None]
    mask_pos = np.array([[1, 1, 1, 1, 1, 0]] * 2, dtype=np.uint8)
    fixed = np.zeros((B, 3, 10))
    fixed[:, :, 0], fixed[:, :, 1], fixed[:, :, 5], fixed[:, :, 6] = p0, v0, p1, v1
    pos = solver.solve_linear(m.Problem(N, 4, 1, 3, mask_pos), _cuda(T), _cuda(fixed))
    mask_yaw = np.array([[1, 1, 0, 0, 0, 0]] * 2, dtype=np.uint8)
    fy = np.zeros((B, 1, 4))
    fy[:, 0, 0], fy[:, 0, 2] = rng.uniform(-3 * np.pi, 3 * np.pi, B), rng.uniform(-3 * np.pi, 3 * np.pi, B)
    yaw = solver.solve_linear(m.Problem(N, 2, 1, 1, mask_yaw), _cuda(T), _cuda(fy))
    torch.cuda.synchronize()
    return T, np.concatenate([pos.cpu().numpy(), yaw.cpu().numpy()], axis=2)


@pytest.mark.gpu
def test_reference_distribution_and_every_code(solver):
    times, coeffs = reference_distribution(solver, 8192, 1234567)
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
    for code in (FEASIBLE, INDET, THRUST_HIGH, THRUST_LOW, VELOCITY, YAW_RATES, YAW_ACC):
        assert counts.get(code, 0) >= 20, (code, counts)
    assert counts.get(ROLL_PITCH, 0) == 0
    # the reference test's property: Feasible at 0.01 => Feasible or Indeterminable at 0.05 and 0.10
    fine = gpu_check(solver, times, coeffs, DEFAULTS, 0.01)[0]
    for mst in (0.05, 0.10):
        coarse = gpu_check(solver, times, coeffs, DEFAULTS, mst)[0]
        assert np.all(np.isin(coarse[fine == FEASIBLE], (FEASIBLE, INDET))), mst


@pytest.mark.gpu
def test_feasible_rows_keep_limits_on_dense_samples(solver):
    """GPU Feasible => thrust, |v|, |yaw'| and |yaw''| within the limits on 1 ms samples (relative 1e-9)."""
    import torch
    times, coeffs = reference_distribution(solver, 512, 99)
    limits = dict(DEFAULTS, v_max=2.5)
    r = gpu_check(solver, times, coeffs, limits)[0]
    assert (r == FEASIBLE).sum() >= 20
    rows = np.nonzero(r == FEASIBLE)[0]
    t, c = _cuda(times[rows]), _cuda(coeffs[rows])
    n = int(np.ceil(times[rows].max() / 1e-3)) + 1
    samples = {}
    for k in (1, 2):
        samples[k] = solver.evaluate(t, c, k, 0.0, 1e-3, n)
    torch.cuda.synchronize()
    v, a = samples[1].cpu().numpy(), samples[2].cpu().numpy()
    valid = (np.arange(n)[None, :] * 1e-3) <= times[rows]
    tol = 1 + 1e-9
    speed = np.linalg.norm(v[:, :, :3], axis=2)
    thrust = np.linalg.norm(a[:, :, :3] + np.array([0, 0, G]), axis=2)
    assert np.all(speed[valid] <= limits["v_max"] * tol)
    assert np.all(thrust[valid] <= limits["f_max"] * tol) and np.all(thrust[valid] >= limits["f_min"] / tol)
    assert np.all(np.abs(v[:, :, 3][valid]) <= limits["omega_z_max"] * tol)
    assert np.all(np.abs(a[:, :, 3][valid]) <= limits["omega_z_dot_max"] * tol)


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 8, 12))
def test_quirk_rows(solver, N):
    cases = []  # (times, coeffs, limits, mst, result, segment)
    t, c = _seg(N, 3, {}, 0.04)
    cases.append((t, c, {"omega_xy_max": 1.0}, 0.05, INDET, 0))  # T < min_section_time
    cases.append((t, c, {"v_max": 1.0}, 0.05, FEASIBLE, -1))
    t, c = _seg(N, 3, {0: {2: 1.0}}, 1.0)
    cases.append((t, c, {"omega_xy_max": 1e-3}, 0.05, FEASIBLE, -1))  # no jerk: bound 0
    if N >= 6:
        # the walk splits down to interior sub-intervals, some without a thrust or a jerk candidate
        t, c = _seg(N, 3, {0: {3: 1.0 / 6, 4: -1.0 / 12}}, 1.0)
        cases.append((t, c, {"omega_xy_max": 0.2}, 0.05, None, None))
    t, c = _seg(N, 3, {2: {2: -G / 2}, 0: {3: 1e-3}}, 1.0)  # f_min <= 1e-6
    cases.append((t, c, {"omega_xy_max": 1e6}, 0.05, INDET, 0))
    t, c = _seg(N, 3, {2: {2: -0.3 * G, 3: 2.2 * G / 6}}, 1.0)  # ThrustLow wins over ThrustHigh
    cases.append((t, c, DEFAULTS, 0.05, THRUST_LOW, 0))
    t, c = _seg(N, 3, {2: {2: -0.3 * G}}, 1.0)  # omega_xy alone: thrust 0.4 g is no ThrustLow without f_min
    cases.append((t, c, {"omega_xy_max": 10.0}, 0.05, FEASIBLE, -1))
    # omega_xy alone still runs the thrust step: its f_min = g makes the bound sqrt(J / g) = 0.32 (without thrust
    # candidates the bound would be ~0 and the row Feasible at any limit)
    J = 1.0
    t, c = _seg(N, 3, {0: {3: J / 6}}, 2.0)
    cases.append((t, c, {"omega_xy_max": 0.5}, 0.05, FEASIBLE, -1))
    cases.append((t, c, {"omega_xy_max": 0.3}, 0.05, INDET, 0))
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
        if want_r is not None:
            assert ex["result"][0] == want_r and ex["segment"][0] == want_s, what
        assert r[0] == ex["result"][0] and s[0] == ex["segment"][0], what
        bad_time = not (np.isfinite(t[0, 0]) and t[0, 0] > 0)
        assert st[0] == (1 if bad_time else 0), what


@pytest.mark.gpu
@pytest.mark.parametrize("N", (6, 10))
def test_row_equals_first_failing_segment(solver, N):
    """A K-segment row equals the first non-Feasible result of its segments run as K = 1 rows, bit for bit."""
    for D in (3, 4):
        K = 16
        times, coeffs = waypoint_fixtures(solver, N, K, D, 24, 30000 + N + D)
        times[3, 5] = np.nan
        for limits in limit_sets(0.7)[:6]:
            r, s, st = gpu_check(solver, times, coeffs, limits, 0.05)
            r1, s1, st1 = gpu_check(solver, times.reshape(-1, 1), coeffs.reshape(-1, 1, D, N), limits, 0.05)
            r1, st1 = r1.reshape(-1, K), st1.reshape(-1, K)
            for b in range(times.shape[0]):
                if st1[b].any():
                    assert r[b] == INDET and s[b] == -1 and st[b] == 1
                    continue
                fail = np.nonzero(r1[b] != FEASIBLE)[0]
                want = (r1[b, fail[0]], fail[0]) if fail.size else (FEASIBLE, -1)
                assert (r[b], s[b]) == want, (b, limits)


@pytest.mark.gpu
def test_host_twin_and_refusals(solver):
    import torch
    import mav_trajectory_generation_b200.capi as capi
    N, K, D, B = 10, 5, 4, 300
    times, coeffs = waypoint_fixtures(solver, N, K, D, B, 40000)
    times[7, 2] = 0.0
    for limits in (DEFAULTS, {"omega_xy_max": 2.0}, {}):
        r, s, st = gpu_check(solver, times, coeffs, limits)
        hr, hs, hst = (np.full(B, -7, dtype=np.int32) for _ in range(3))
        solver.check_input_feasibility_host(times, coeffs, limits, hr, hs, hst, 0.05, G)
        assert np.array_equal(hr, r) and np.array_equal(hs, s) and np.array_equal(hst, st)
        hr2 = np.full(B, -7, dtype=np.int32)
        solver.check_input_feasibility_host(times, coeffs, limits, hr2, None, None, 0.05, G)
        assert np.array_equal(hr2, r)
        dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        lib = solver.lib
        ic = capi.input_constraints(limits, 0.05, G)
        tt, cc = _cuda(times), _cuda(coeffs)
        assert lib.mtg_input_feasibility_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(), C.byref(ic),
                                                   dr.data_ptr(), None, None, None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(dr.cpu().numpy(), r)
    # refusals: MTG_ERR_BAD_ARG, no launch, outputs untouched
    bad = [dict(limits={"v_max": np.nan}), dict(limits={"f_min": -1.0}), dict(limits={"omega_xy_max": -0.5}),
           dict(limits=DEFAULTS, gravity=np.nan), dict(limits=DEFAULTS, gravity=np.inf),
           dict(limits=DEFAULTS, mst=0.0), dict(limits=DEFAULTS, mst=-0.05), dict(limits=DEFAULTS, mst=np.inf),
           dict(limits=DEFAULTS, mst=np.nan)]
    tt, cc = _cuda(times), _cuda(coeffs)
    for case in bad:
        ic = capi.input_constraints(case["limits"], case.get("mst", 0.05), case.get("gravity", G))
        before = solver.launch_count
        dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        assert solver.lib.mtg_input_feasibility_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(),
                                                          C.byref(ic), dr.data_ptr(), None, None, None) == -1, case
        hr = np.full(B, -7, dtype=np.int32)
        assert solver.lib.mtg_input_feasibility_batch_host_f64(solver.h, N, K, D, B, times.ctypes.data,
                                                               coeffs.ctypes.data, C.byref(ic), hr.ctypes.data, None,
                                                               None) == -1, case
        torch.cuda.synchronize()
        assert solver.launch_count == before and (dr.cpu().numpy() == -7).all() and (hr == -7).all(), case
    ic = capi.input_constraints(DEFAULTS)
    ic.present |= 1 << 6
    assert solver.lib.mtg_input_feasibility_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(), C.byref(ic),
                                                      dr.data_ptr(), None, None, None) == -1
    for n_bad in (2, 5, 14):
        assert solver.lib.mtg_input_feasibility_batch_f64(solver.h, n_bad, K, D, B, tt.data_ptr(), cc.data_ptr(),
                                                          C.byref(capi.input_constraints(DEFAULTS)), dr.data_ptr(),
                                                          None, None, None) == -1
    # +inf limits never fail
    r = gpu_check(solver, times, coeffs, {k: (0.0 if k == "f_min" else np.inf) for k in DEFAULTS})[0]
    assert np.all(r[np.arange(B) != 7] == FEASIBLE)


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    """BatchPolynomialOptimization<10>::checkInputFeasibility against the host FeasibilityAnalytic, both against the
    replay, on the rows whose margin is clear of rounding."""
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
