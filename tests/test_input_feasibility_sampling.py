"""Batched FeasibilitySampling::checkInputFeasibilityTrajectory (mtg_input_feasibility_sampling_batch_f64).

The exact reference is tests/feasibility_sampling_exact.cpp: the reference's running fp64 sum of sample times, each
sample's full state in binary128, and a per-row decision margin (the smallest relative gap of any comparison made up to
the deciding one).  On the CPU it is pinned to closed forms, and the host mirror is checked against it; on the GPU the
kernel must give the replay's result and segment on every row whose margin exceeds MARGIN_BOUND; at most 1 % of rows
may fall under it, and they are reported."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import feasibility_oracle
import feasibility_recursive_oracle
import feasibility_sampling_oracle as F
from test_input_feasibility import limit_sets, reference_distribution, waypoint_fixtures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility_sampling.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_input_feasibility_sampling")

G = 9.81
DEFAULTS = dict(f_min=0.5 * G, f_max=1.5 * G, v_max=3.0, omega_xy_max=np.pi / 2, omega_z_max=np.pi / 2,
                omega_z_dot_max=2 * np.pi)
FEASIBLE, INDET, THRUST_HIGH, THRUST_LOW, VELOCITY, ROLL_PITCH, YAW_RATES, YAW_ACC = range(8)
STATUS_BAD_TIME, STATUS_FEAS_CAPACITY = 1, 4
# the analytic check's limit sets, and three that make RollPitchRates, YawRates and YawAcc common in the fixtures
PARITY_SETS = limit_sets(0.7) + [{"omega_xy_max": 0.05}, {"omega_z_max": 0.3},
                                 {"omega_z_dot_max": 0.2, "omega_xy_max": 3.0}]
DTS = (0.01, 0.05, 0.10)
# The device rounds every step of the state map in fp64 and its trigonometry is not correctly rounded: a few hundred
# units of rounding relative to the limit at most on these fixtures.  Rows whose margin is above this are decided
# identically by any faithful fp64 evaluation.
MARGIN_BOUND = 1e-9


def build_binary():
    """The C++ driver of the host FeasibilitySampling and the batch class
    (tests/cpp/test_input_feasibility_sampling.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


def host_mirror(times, coeffs, limits, dt, gravity=G):
    """FeasibilitySampling of the C++ host mirror on every row: (result [B], segment [B])."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    present = sum(1 << q for q, n in enumerate(F.LIMITS) if n in limits)
    lim = np.array([float(limits.get(n, 0.0)) for n in F.LIMITS])
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([B, K, D, N, present], dtype=np.int32).tobytes())
            f.write(np.concatenate([lim, [gravity, dt]]).tobytes())
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


def exact(times, coeffs, limits, dt=0.01):
    return F.input_feasibility_sampling(times, coeffs, limits, dt, G)


def closed_form_cases(N):
    """(times, coeffs, limits, dt, result, segment, status) rows whose decision follows from a closed form."""
    cases = []
    t, c = _seg(N, 3, {}, 2.0)  # hover: thrust g, nothing moves
    cases.append((t, c, DEFAULTS, 0.01, FEASIBLE, -1, 0))
    t, c = _seg(N, 3, {2: {2: -0.3 * G}}, 2.0)  # a_z = -0.6 g: thrust 0.4 g
    cases.append((t, c, DEFAULTS, 0.01, THRUST_LOW, 0, 0))
    cases.append((t, c, {"omega_xy_max": 10.0}, 0.01, FEASIBLE, -1, 0))  # thrust is not checked for omega_xy alone
    t, c = _seg(N, 3, {2: {2: 0.3 * G}}, 2.0)  # 1.6 g
    cases.append((t, c, DEFAULTS, 0.01, THRUST_HIGH, 0, 0))
    t, c = _seg(N, 3, {0: {1: 3.5}}, 1.0)  # constant speed 3.5: Velocity at the first sample
    cases.append((t, c, DEFAULTS, 0.01, VELOCITY, 0, 0))
    # v_x = 2.5 + A t (0.01 - t): 2.5 at both samples 0 and 0.01, 3.1 at t = 0.005 between them
    A = 0.6 / 0.005 ** 2
    t, c = _seg(N, 3, {0: {1: 2.5, 2: A * 0.01 / 2, 3: -A / 3}}, 0.01)
    cases.append((t, c, {"v_max": 3.0}, 0.01, FEASIBLE, -1, 0))
    # v_x = 10 t at dt = 0.1: the third running sum is 0.30000000000000004 > T = 0.3, so v(T) = 3 is never sampled
    t, c = _seg(N, 3, {0: {2: 5.0}}, 0.3)
    cases.append((t, c, {"v_max": 2.9}, 0.1, FEASIBLE, -1, 0))
    t, c = _seg(N, 3, {0: {2: 5.0}}, 0.31)
    cases.append((t, c, {"v_max": 2.9}, 0.1, VELOCITY, 0, 0))
    # constant jerk J along x at hover: omega_xy = J / g at t = 0, smaller later
    J = 1.0
    t, c = _seg(N, 3, {0: {3: J / 6}}, 2.0)
    cases.append((t, c, {"omega_xy_max": 0.99 * J / G}, 0.01, ROLL_PITCH, 0, 0))
    cases.append((t, c, {"omega_xy_max": 1.01 * J / G}, 0.01, FEASIBLE, -1, 0))
    # tilted hover (a_x = g, zb_z = 1 / sqrt 2) with yaw rate r: omega_z = r zb_z, so r = 1.2 passes omega_z_max = 1
    # while r = 1.5 does not
    t, c = _seg(N, 4, {0: {2: G / 2}, 3: {1: 1.2}}, 1.0)
    cases.append((t, c, {"omega_z_max": 1.0}, 0.01, FEASIBLE, -1, 0))
    t, c = _seg(N, 4, {0: {2: G / 2}, 3: {1: 1.5}}, 1.0)
    cases.append((t, c, {"omega_z_max": 1.0}, 0.01, YAW_RATES, 0, 0))
    t, c = _seg(N, 4, {3: {2: 3.5}}, 0.5)  # yaw acceleration 7 at hover
    cases.append((t, c, DEFAULTS, 0.01, YAW_ACC, 0, 0))
    # free fall: thrust exactly 0, a NaN state passes every comparison (the speed reaches 3 at t = 0.31)
    t, c = _seg(N, 3, {2: {2: -G / 2}}, 1.0)
    cases.append((t, c, {k: v for k, v in DEFAULTS.items() if k != "v_max"}, 0.01, FEASIBLE, -1, 0))
    for D in (2, 5):  # D not 3 or 4
        t, c = _seg(N, D, {}, 1.0)
        cases.append((t, c, DEFAULTS, 0.01, INDET, 0, 0))
    t, c = _seg(N, 3, {}, 2.0 ** 24 * 0.01 * 1.001)  # over the sample cap: not sampled
    cases.append((t, c, DEFAULTS, 0.01, INDET, 0, STATUS_FEAS_CAPACITY))
    for T in (0.0, -1.0, np.nan, np.inf):
        t, c = _seg(N, 3, {}, T)
        cases.append((t, c, DEFAULTS, 0.01, INDET, -1, STATUS_BAD_TIME))
    return cases


# ---- CPU: the replay against closed forms, the host mirror against the replay --------------------------------------
@pytest.mark.parametrize("N", (4, 8, 12))
def test_replay_closed_forms(N):
    for t, c, limits, dt, want_r, want_s, want_st in closed_form_cases(N):
        r = exact(t, c, limits, dt)
        assert (r["result"][0], r["segment"][0], r["status"][0]) == (want_r, want_s, want_st), (N, limits, dt, t)
    # the bump between two samples: the analytic check sees the exact maximum
    A = 0.6 / 0.005 ** 2
    t, c = _seg(N, 3, {0: {1: 2.5, 2: A * 0.01 / 2, 3: -A / 3}}, 0.01)
    assert feasibility_oracle.input_feasibility(t, c, {"v_max": 3.0}, 0.005, G)["result"][0] == VELOCITY
    # the margin is the relative gap of the deciding comparison here: |3.5 - 3| / 3
    t, c = _seg(N, 3, {0: {1: 3.5}}, 1.0)
    assert abs(exact(t, c, {"v_max": 3.0})["margin"][0] - 0.5 / 3.0) < 1e-15


@pytest.mark.parametrize("N", (4, 8, 12))
def test_host_mirror_closed_forms(N):
    for t, c, limits, dt, want_r, want_s, want_st in closed_form_cases(N):
        if want_st == STATUS_FEAS_CAPACITY:
            continue  # the single-object checker samples it all, as the reference
        if want_st == STATUS_BAD_TIME:  # the single-object checker has no bad-time rule (T = inf never ends)
            continue
        r, s = host_mirror(t, c, limits, dt)
        assert (r[0], s[0]) == (want_r, want_s), (N, limits, dt, t)


def test_host_mirror_matches_replay():
    """The single-object FeasibilitySampling (host, no GPU) against the replay on margin-clear rows."""
    import oracle_lib as O
    checked = 0
    for N, K, D in ((4, 3, 3), (8, 3, 4), (12, 2, 3), (12, 2, 4)):
        pos, times = O.make_waypoint_batch(K, D, 24, base_seed=950 + N + D)
        coeffs, _ = O.solve_waypoint_batch(N, N // 2 - 1, pos, times)
        for i, limits in enumerate(PARITY_SETS):
            dt = (0.05, 0.10)[i % 2]
            r, s = host_mirror(times, coeffs, limits, dt)
            ex = exact(times, coeffs, limits, dt)
            ok = ex["margin"] > MARGIN_BOUND
            assert np.array_equal(r[ok], ex["result"][ok]), (N, D, limits)
            assert np.array_equal(s[ok], ex["segment"][ok]), (N, D, limits)
            checked += int(ok.sum())
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


def gpu_check(solver, times, coeffs, limits, dt=0.01):
    import torch
    r, s, st = solver.check_input_feasibility_sampling(_cuda(times), _cuda(coeffs), limits, dt, G)
    torch.cuda.synchronize()
    return r.cpu().numpy(), s.cpu().numpy(), st.cpu().numpy()


def check_parity(solver, times, coeffs, limits, dt, what, counts=None):
    r, s, st = gpu_check(solver, times, coeffs, limits, dt)
    ex = exact(times, coeffs, limits, dt)
    ok = ex["margin"] > MARGIN_BOUND
    bad = np.nonzero(ok & ((r != ex["result"]) | (s != ex["segment"])))[0]
    assert bad.size == 0, (f"{what}: rows {bad[:8]} gpu {r[bad[:8]]}/{s[bad[:8]]} exact {ex['result'][bad[:8]]}/"
                           f"{ex['segment'][bad[:8]]} margin {ex['margin'][bad[:8]]}")
    assert np.array_equal(st, ex["status"]), what
    under = np.nonzero(~ok)[0]
    if under.size:
        print(f"{what}: {under.size}/{len(r)} rows within the margin bound: rows {under[:8]} gpu {r[under[:8]]} "
              f"exact {ex['result'][under[:8]]} margin {ex['margin'][under[:8]]}")
    if counts is not None:
        for code in range(8):
            counts[code] = counts.get(code, 0) + int((r == code).sum())
    return under.size, len(r)


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 6, 8, 10, 12))
def test_parity_with_binary128_replay(solver, N):
    under = total = 0
    counts = {}
    for D in (3, 4):
        for K in (1, 3, 16, 50):
            B = {1: 64, 3: 32, 16: 8, 50: 4}[K]
            times, coeffs = waypoint_fixtures(solver, N, K, D, B, 80000 + 100 * N + 10 * D + K)
            for i, limits in enumerate(PARITY_SETS):
                dt = DTS[(i + K) % 3]
                u, t = check_parity(solver, times, coeffs, limits, dt, f"N={N} D={D} K={K} set {i} dt {dt}", counts)
                under += u
                total += t
    print(f"N={N}: {under}/{total} rows within the margin bound; results {counts}")
    assert under <= 0.01 * total
    for code in (FEASIBLE, THRUST_HIGH, THRUST_LOW, VELOCITY, ROLL_PITCH, YAW_RATES, YAW_ACC):
        assert counts.get(code, 0) > 0, (N, code, counts)


@pytest.mark.gpu
def test_reference_test_property(solver):
    """The reference test's cross-check on its own segment distribution (N = 12, D = 4, K = 1), through the three GPU
    entries: analytic Feasible (min_section_time 0.01) => sampling Feasible at 0.01, 0.05 and 0.10 s, except for
    RollPitchRates on the few rows the analytic roll / pitch walk lets through; recursive Feasible at any of 0.01, 0.05, 0.10 => sampling
    Feasible at 0.01 s; on the rows every replay involved decides clear of rounding.  Each limit set also returns
    RollPitchRates on some row, and the sampling results match the replay."""
    times, coeffs = reference_distribution(solver, 4096, 24680)
    sets = [dict(DEFAULTS), dict(DEFAULTS, omega_xy_max=1.0), dict(DEFAULTS, f_max=3.0 * G, omega_xy_max=0.5)]
    for i, limits in enumerate(sets):
        counts = {}
        samp, clear_s = {}, {}
        for dt in DTS:
            check_parity(solver, times, coeffs, limits, dt, f"reference set {i} dt {dt}", counts)
            samp[dt] = gpu_check(solver, times, coeffs, limits, dt)[0]
            clear_s[dt] = exact(times, coeffs, limits, dt)["margin"] > MARGIN_BOUND
        print(f"reference set {i}: sampling results {counts}")
        assert counts.get(ROLL_PITCH, 0) >= 1, (i, counts)
        r, _, _ = solver.check_input_feasibility(_cuda(times), _cuda(coeffs), limits, 0.01, G)
        analytic = r.cpu().numpy()
        clear_a = feasibility_oracle.input_feasibility(times, coeffs, limits, 0.01, G)["margin"] > 1e-9
        for dt in DTS:
            rows = (analytic == FEASIBLE) & clear_a & clear_s[dt]
            # The analytic roll / pitch walk is not a sound bound: it takes sqrt(j_max / f_min), below j_max / f_min
            # wherever that exceeds 1 rad/s, and a section that holds no thrust or jerk candidate gets no bound and
            # passes.  So a row may pass the analytic check and show a sampled roll / pitch rate above the limit
            # (a few percent of the analytic-Feasible rows at most on these sets).  Every other result must be
            # Feasible.
            bad = np.nonzero(rows & (samp[dt] != FEASIBLE) & (samp[dt] != ROLL_PITCH))[0]
            assert bad.size == 0, (i, dt, bad[:8], samp[dt][bad[:8]])
            rp = int((rows & (samp[dt] == ROLL_PITCH)).sum())
            print(f"reference set {i} dt {dt}: {rp} analytic-Feasible rows sample RollPitchRates")
            assert rp <= 0.05 * rows.sum(), (i, dt, rp)
        rec_feasible = np.zeros(len(times), dtype=bool)
        for mst in DTS:
            r, _, _ = solver.check_input_feasibility_recursive(_cuda(times), _cuda(coeffs), limits, mst, G)
            clear_r = feasibility_recursive_oracle.input_feasibility_recursive(
                times, coeffs, limits, mst, G)["margin"] > 1e-9
            rec_feasible |= (r.cpu().numpy() == FEASIBLE) & clear_r
        bad = np.nonzero(rec_feasible & clear_s[0.01] & (samp[0.01] != FEASIBLE))[0]
        assert bad.size == 0, (i, bad[:8], samp[0.01][bad[:8]])
        assert ((analytic == FEASIBLE) & clear_a).sum() >= 20 and rec_feasible.sum() >= 20, i


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 8, 12))
def test_edge_rows(solver, N):
    """Closed-form rows, bad times, the sample cap (returned at once), free-fall NaN rows, and batch sizes that are
    not a multiple of the tile."""
    for t, c, limits, dt, want_r, want_s, want_st in closed_form_cases(N):
        r, s, st = gpu_check(solver, t, c, limits, dt)
        assert (r[0], s[0], st[0]) == (want_r, want_s, want_st), (N, limits, dt, t)
    # a capped segment after a passing one, and before a failing one
    t = np.array([[1.0, 1e9, 1.0]])
    c = np.zeros((1, 3, 3, N))
    c[0, 2, 0, 1] = 3.5
    r, s, st = gpu_check(solver, t, c, DEFAULTS, 0.01)
    assert (r[0], s[0], st[0]) == (INDET, 1, STATUS_FEAS_CAPACITY)
    # rows of every tile remainder: K = 3 tiles hold 42 rows, K = 16 tiles 8
    for K, B in ((3, 43), (3, 85), (16, 9), (16, 1), (1, 129)):
        times, coeffs = waypoint_fixtures(solver, N, K, 3, B, 90000 + N + K + B)
        times[B // 2, K - 1] = np.nan
        coeffs[B - 1, 0, :, 2:] = 0.0  # the last row's first segment falls freely: thrust 0, a NaN state
        coeffs[B - 1, 0, 2, 2] = -G / 2
        check_parity(solver, times, coeffs, DEFAULTS, 0.05, f"N={N} K={K} B={B}")


@pytest.mark.gpu
def test_host_twin_and_refusals(solver):
    import torch
    import mav_trajectory_generation_b200.capi as capi
    N, K, D, B = 10, 5, 4, 300
    times, coeffs = waypoint_fixtures(solver, N, K, D, B, 71000)
    times[7, 2] = 0.0
    lib = solver.lib
    for limits, dt in ((DEFAULTS, 0.01), ({"omega_xy_max": 0.5}, 0.05), ({}, 0.1)):
        r, s, st = gpu_check(solver, times, coeffs, limits, dt)
        hr, hs, hst = (np.full(B, -7, dtype=np.int32) for _ in range(3))
        solver.check_input_feasibility_sampling_host(times, coeffs, limits, hr, hs, hst, dt, G)
        assert np.array_equal(hr, r) and np.array_equal(hs, s) and np.array_equal(hst, st)
        hr2 = np.full(B, -7, dtype=np.int32)
        solver.check_input_feasibility_sampling_host(times, coeffs, limits, hr2, None, None, dt, G)
        assert np.array_equal(hr2, r)
        dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        ic = capi.input_constraints(limits, 0.05, G)
        ic.min_section_time = np.nan  # not read here
        tt, cc = _cuda(times), _cuda(coeffs)
        assert lib.mtg_input_feasibility_sampling_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(),
                                                            C.byref(ic), dt, dr.data_ptr(), None, None, None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(dr.cpu().numpy(), r)
    # refusals: MTG_ERR_BAD_ARG, no launch, outputs untouched
    bad_ic = [capi.input_constraints(lim, 0.05, g) for lim, g in
              (({"v_max": np.nan}, G), ({"f_min": -1.0}, G), ({"omega_xy_max": -0.5}, G), (DEFAULTS, np.nan),
               (DEFAULTS, np.inf))]
    extra = capi.input_constraints(DEFAULTS)
    extra.present |= 1 << 6
    bad_ic.append(extra)
    good = capi.input_constraints(DEFAULTS)
    cases = [(N, K, D, ic, 0.01) for ic in bad_ic]
    cases += [(N, K, D, good, dt) for dt in (0.0, -0.01, np.nan, np.inf, -np.inf)]
    cases += [(n_bad, K, D, good, 0.01) for n_bad in (2, 5, 14)] + [(N, 0, D, good, 0.01), (N, K, 0, good, 0.01)]
    tt, cc = _cuda(times), _cuda(coeffs)
    for n, k, d, ic, dt in cases:
        before = solver.launch_count
        dr = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        assert lib.mtg_input_feasibility_sampling_batch_f64(solver.h, n, k, d, B, tt.data_ptr(), cc.data_ptr(),
                                                            C.byref(ic), dt, dr.data_ptr(), None, None, None) == -1
        hr = np.full(B, -7, dtype=np.int32)
        assert lib.mtg_input_feasibility_sampling_batch_host_f64(solver.h, n, k, d, B, times.ctypes.data,
                                                                 coeffs.ctypes.data, C.byref(ic), dt, hr.ctypes.data,
                                                                 None, None) == -1
        torch.cuda.synchronize()
        assert solver.launch_count == before and (dr.cpu().numpy() == -7).all() and (hr == -7).all(), (n, k, d, dt)
    # +inf limits never fail
    r = gpu_check(solver, times, coeffs, {k: (0.0 if k == "f_min" else np.inf) for k in DEFAULTS})[0]
    assert np.all(r[np.arange(B) != 7] == FEASIBLE)


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    """BatchPolynomialOptimization<10>::checkInputFeasibilitySampling against the host FeasibilitySampling, both
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
