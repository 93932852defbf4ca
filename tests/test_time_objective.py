"""Batched computeMaximumOfMagnitude (mtg_max_magnitude_batch_f64) and the nonlinear optimiser's time objective with
soft velocity / acceleration constraints (mtg_time_objective_batch_f64).

The exact reference is tests/extrema_exact.cpp (binary128 critical polynomial, Taylor-bound root isolation); the CPU
tests pin it against mpmath and closed forms, the GPU tests hold the kernel to it."""
import math
import os
import subprocess

import numpy as np
import pytest

import extrema_oracle as X

EPS = np.finfo(np.float64).eps
NS = (2, 4, 6, 8, 10, 12)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_time_objective.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_time_objective")


def build_binary():
    """C++ check of the batch class against the single-object host mirror (tests/cpp/test_time_objective.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    out = subprocess.run([build_binary()], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert " 0 failures" in out.stdout


def random_segments(rng, B, K, D, N, t_lo=0.3, t_hi=3.0):
    """Coefficients scaled so that every power contributes O(1) over the segment."""
    times = rng.uniform(t_lo, t_hi, size=(B, K))
    scale = times[:, :, None, None] ** -np.arange(N)[None, None, None, :]
    coeffs = rng.standard_normal((B, K, D, N)) * scale
    return times, coeffs


def check_against_exact(value, time, segment, times, coeffs, k, what):
    ex = X.max_magnitude(times, coeffs, k)
    N = coeffs.shape[3]
    bound = 1e-13 * ex["value"] + 8 * max(N - 1 - k, 1) * EPS * ex["scale"]
    err = np.abs(value - ex["value"])
    bad = np.nonzero(~(err <= bound))[0]
    assert bad.size == 0, (f"{what} k={k}: {bad.size} values off, first b={bad[0]} gpu={value[bad[0]]!r} "
                           f"exact={ex['value'][bad[0]]!r} bound={bound[bad[0]]:.3e}")
    distinct = ex["runner_up"] <= ex["value"] * (1 - 1e-9)
    T = times[np.arange(times.shape[0]), ex["segment"]]
    # the maximiser's time is only determined to 1e-6 T where |p^(k)| drops measurably within that distance (a flat
    # maximum such as 1 - (t - c)^4 has the same fp64 value over 1e-4 T)
    for b in np.nonzero(distinct)[0]:
        seg = coeffs[b, ex["segment"][b]]
        pk = np.polynomial.polynomial.polyder(seg.T, k, axis=0)
        ts = np.clip(ex["time"][b] + np.array([-1e-6, 1e-6]) * T[b], 0.0, T[b])
        near = np.sqrt((np.atleast_2d(np.polynomial.polynomial.polyval(ts, pk)) ** 2).sum(axis=0)).max()
        if ex["value"][b] - near <= 4 * bound[b]:
            distinct[b] = False
    seg_ok = segment[distinct] == ex["segment"][distinct]
    assert seg_ok.all(), f"{what} k={k}: segment index differs at b={np.nonzero(distinct)[0][~seg_ok][:5]}"
    t_ok = np.abs(time - ex["time"])[distinct] <= 1e-6 * T[distinct]
    assert t_ok.all(), f"{what} k={k}: maximiser time differs at b={np.nonzero(distinct)[0][~t_ok][:5]}"
    return ex


# ---- CPU: the exact reference itself ----------------------------------------------------------------------------------
def _mp_max(c, T, k):
    """mpmath at 50 digits: candidates 0, T and the real roots of the critical polynomial, one segment c [D][N]."""
    import mpmath as mp
    mp.mp.dps = 50
    D, N = c.shape

    def deriv(row, m):
        return [mp.mpf(math.perm(j, m)) * mp.mpf(float(row[j])) for j in range(m, N)]

    pk = [deriv(c[d], k) for d in range(D)]
    if D == 1:
        g = deriv(c[0], k + 1)
    else:
        g = [mp.mpf(0)] * (2 * (N - k) - 2)
        for d in range(D):
            p1 = deriv(c[d], k + 1)
            for a in range(len(pk[d])):
                for j in range(len(p1)):
                    g[a + j] += pk[d][a] * p1[j]
    while g and g[-1] == 0:
        g.pop()
    cands = [mp.mpf(0), mp.mpf(float(T))]
    if len(g) >= 2:
        roots = mp.polyroots(g[::-1], maxsteps=400, extraprec=400, error=False)
        for r in roots:
            r = mp.mpc(r)
            if abs(r.imag) <= mp.mpf(10) ** -30 * (1 + abs(r.real)) and 0 <= r.real <= T:
                cands.append(r.real)

    def mag(t):
        return mp.sqrt(sum(mp.polyval(p[::-1], t) ** 2 for p in pk))

    return max(float(mag(t)) for t in cands)


def test_exact_matches_mpmath():
    rng = np.random.default_rng(7)
    cases = 0
    for it in range(240):
        N = int(rng.choice((4, 6, 8, 10)))
        D = int(rng.integers(1, 4))
        k = int(rng.integers(0, N - 1))
        times, coeffs = random_segments(rng, 1, 1, D, N)
        ex = X.max_magnitude(times, coeffs, k, n_threads=1)
        ref = _mp_max(coeffs[0, 0], times[0, 0], k)
        assert abs(ex["value"][0] - ref) <= 4 * EPS * ref, (it, N, D, k, ex["value"][0], ref)
        cases += 1
    assert cases == 240


def test_exact_closed_forms():
    # constant velocity (1 + 2t, 3t): |v| = sqrt(13) everywhere, the first candidate (t = 0) wins
    c = np.zeros((1, 1, 2, 4))
    c[0, 0, 0, :2] = (1, 2)
    c[0, 0, 1, 1] = 3
    ex = X.max_magnitude(np.array([[2.0]]), c, 1)
    assert ex["value"][0] == pytest.approx(math.sqrt(13), rel=1e-16) and ex["time"][0] == 0.0
    # single interior maximum: 4t(1-t) on [0, 1] -> 1 at 0.5
    c = np.zeros((1, 1, 1, 6))
    c[0, 0, 0, :3] = (0, 4, -4)
    ex = X.max_magnitude(np.array([[1.0]]), c, 0)
    assert ex["value"][0] == 1.0 and ex["time"][0] == 0.5
    # maximum at the segment end: t^2 on [0, 1.5], and at the start: 1 - t on [0, 0.5]
    c = np.zeros((2, 1, 1, 4))
    c[0, 0, 0, 2] = 1
    c[1, 0, 0, :2] = (1, -1)
    ex = X.max_magnitude(np.array([[1.5], [0.5]]), c, 0)
    assert ex["value"].tolist() == [2.25, 1.0] and ex["time"].tolist() == [1.5, 0.0]
    # all-zero derivative (second derivative of a line): Extremum() = (0, 0, 0)
    c = np.zeros((1, 2, 3, 4))
    c[0, :, :, :2] = 1.5
    ex = X.max_magnitude(np.array([[1.0, 2.0]]), c, 2)
    assert ex["value"][0] == 0.0 and ex["time"][0] == 0.0 and ex["segment"][0] == 0


def test_exact_bounds_dense_sampling():
    rng = np.random.default_rng(11)
    for N in (6, 10, 12):
        for D in (1, 3):
            times, coeffs = random_segments(rng, 40, 2, D, N)
            for k in (0, 1, N // 2):
                ex = X.max_magnitude(times, coeffs, k)
                for b in range(times.shape[0]):
                    s = 0.0
                    for i in range(2):
                        t = np.linspace(0, times[b, i], 4001)
                        pk = np.polynomial.polynomial.polyder(coeffs[b, i].T, k, axis=0)
                        vals = np.polynomial.polynomial.polyval(t, pk)
                        s = max(s, np.sqrt((np.atleast_2d(vals) ** 2).sum(axis=0)).max())
                    assert s <= ex["value"][b] * (1 + 1e-12) + 1e-300, (N, D, k, b, s, ex["value"][b])


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _run(solver, times, coeffs, derivs):
    import torch
    v, t, s, st = solver.max_magnitude(torch.from_numpy(times).cuda(), torch.from_numpy(np.ascontiguousarray(coeffs)).cuda(),
                                       derivs)
    torch.cuda.synchronize()
    return v.cpu().numpy(), t.cpu().numpy(), s.cpu().numpy(), st.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("D", (1, 2, 3, 4))
def test_max_magnitude_every_shape(solver, N, D):
    rng = np.random.default_rng(100 * N + D)
    times, coeffs = random_segments(rng, 48, 3, D, N)
    ks = list(range(N - 1))
    for c0 in range(0, len(ks), 8):  # at most 8 orders per call
        chunk = ks[c0:c0 + 8]
        v, t, s, st = _run(solver, times, coeffs, chunk)
        assert (st == 0).all()
        for q, k in enumerate(chunk):
            check_against_exact(v[:, q], t[:, q], s[:, q], times, coeffs, k, f"N={N} D={D}")


@pytest.mark.gpu
@pytest.mark.parametrize("K", (1, 16, 50))
def test_max_magnitude_solved_fixtures(solver, oracle, K):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, D, B = 10, 4, 3, 64
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=2000 + K)
    prob = m.Problem(N, r, K, D)
    coeffs = solver.solve_linear(prob, torch.from_numpy(times).cuda(),
                                 torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda()).cpu().numpy()
    ks = list(range(N - 1))
    for c0 in (0, 8):
        chunk = ks[c0:c0 + 8]
        v, t, s, st = _run(solver, times, coeffs, chunk)
        assert (st == 0).all()
        for q, k in enumerate(chunk):
            check_against_exact(v[:, q], t[:, q], s[:, q], times, coeffs, k, f"fixture K={K}")


def _poly_coeffs(roots_factor, N):
    """Increasing-power coefficients of a numpy poly1d, zero padded to N."""
    c = np.zeros(N)
    p = roots_factor.coeffs[::-1]
    c[:len(p)] = p
    return c


@pytest.mark.gpu
def test_max_magnitude_hard_cases(solver):
    N = 12
    P = np.poly1d
    segs = []  # (T, [D][N] coefficients)
    # near-tangent maxima: 1 - (t-c)^4 + e (t-c)^2 has maxima at c +- sqrt(e/2) and a minimum between (g has a
    # clustered / multiple root)
    for c0, e in ((0.5, 0.0), (0.37, 1e-8), (0.61, 1e-12), (0.5, 1e-4)):
        u = P([1, -c0])
        segs.append((1.0, [_poly_coeffs(1 - u ** 4 + e * u ** 2, N)]))
    # maximum exactly at t = 0 and at t = T
    segs.append((0.5, [_poly_coeffs(P([-1, 1]), N)]))
    segs.append((1.5, [_poly_coeffs(P([1, 0, 0]), N)]))
    # trailing zeros: the degree drops to 3 inside an N = 12 container
    segs.append((2.0, [_poly_coeffs(P([1, -3, 1, 2]), N)]))
    # long segment, T = 90 s
    rng = np.random.default_rng(5)
    segs.append((90.0, [rng.standard_normal(N) * 90.0 ** -np.arange(N)]))
    for D in (1, 3):
        times = np.array([[T] for T, _ in segs])
        coeffs = np.zeros((len(segs), 1, D, N))
        for b, (_, rows) in enumerate(segs):
            coeffs[b, 0, 0] = rows[0]
            for d in range(1, D):
                coeffs[b, 0, d, 0] = 0.25 * d  # constant components: same critical points, larger magnitude
        for ks in ([0, 1, 2], [3, 4, 5, 6, 7, 8, 9, 10]):
            v, t, s, st = _run(solver, times, coeffs, ks)
            assert (st == 0).all()
            for q, k in enumerate(ks):
                check_against_exact(v[:, q], t[:, q], s[:, q], times, coeffs, k, f"hard D={D}")
    # all-zero derivative -> Extremum() = (0, 0, 0)
    coeffs = np.zeros((2, 3, 2, 4))
    coeffs[0, :, :, :2] = 1.0
    v, t, s, st = _run(solver, np.ones((2, 3)), coeffs, [2])
    assert (v == 0).all() and (t == 0).all() and (s == 0).all() and (st == 0).all()
    v, t, s, st = _run(solver, np.ones((2, 3)), coeffs, [0])
    assert v[1, 0] == 0 and t[1, 0] == 0 and s[1, 0] == 0


@pytest.mark.gpu
def test_max_magnitude_bad_times_and_arguments(solver):
    import mav_trajectory_generation_b200 as m
    rng = np.random.default_rng(3)
    times, coeffs = random_segments(rng, 5, 4, 3, 10)
    times[1, 2] = 0.0
    times[2, 0] = -1.0
    times[3, 3] = np.nan
    times[4, 1] = np.inf
    v, t, s, st = _run(solver, times, coeffs, [1, 2])
    assert st[0] == 0 and (st[1:] == m.STATUS_BAD_TIME).all()
    assert np.isnan(v[1:]).all() and np.isfinite(v[0]).all()
    for derivs in ([-1], [9], [1] * 9):
        with pytest.raises(RuntimeError, match="rc=-1"):
            _run(solver, times, coeffs, derivs)
    with pytest.raises(RuntimeError, match="rc=-1"):  # odd N
        _run(solver, times, coeffs[:, :, :, :3], [0])


def _numpy_time_cost(times, richter, penalty):
    total = np.zeros(times.shape[0])
    for i in range(times.shape[1]):  # left to right, as computeTotalTrajectoryTime
        total = total + times[:, i]
    return total * penalty if richter else total * total * penalty


@pytest.mark.gpu
@pytest.mark.parametrize("with_free", (False, True))
@pytest.mark.parametrize("richter", (0, 1))
@pytest.mark.parametrize("constraints", ((), ((1, 2.0),), ((1, 2.5), (2, 3.0)), ((2, 1e-3), (1, 0.05))))
def test_time_objective(solver, oracle, with_free, richter, constraints):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 96
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=3000)
    prob = m.Problem(N, r, K, D)
    tt = torch.from_numpy(times).cuda()
    df = torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda()
    d_free = None
    if with_free:  # perturbed optimum, as the nonlinear optimiser's free-constraint iterate
        d_free = torch.empty((B, D, prob.n_free), dtype=torch.float64, device="cuda")
        solver.solve_linear(prob, tt, df, d_free=d_free)
        d_free = d_free + 0.05 * torch.randn(d_free.shape, dtype=torch.float64, device="cuda",
                                             generator=torch.Generator("cuda").manual_seed(1))
    weight, mcost, penalty = 100.0, 1e12, 500.0
    obj, terms, coeffs, status = solver.time_objective(prob, tt, df, d_free, constraints=constraints, time_cost=richter,
                                                       time_penalty=penalty, soft_constraint_weight=weight,
                                                       maximum_cost=mcost)
    if with_free:
        ref_coeffs = solver.coeffs_from_constraints(prob, tt, df, d_free)
    else:
        ref_coeffs = solver.solve_linear(prob, tt, df)
    ref_cost = solver.compute_cost(prob, tt, ref_coeffs)
    torch.cuda.synchronize()
    obj, terms, coeffs, status = (x.cpu().numpy() for x in (obj, terms, coeffs, status))
    assert (status == 0).all()
    assert np.array_equal(coeffs, ref_coeffs.cpu().numpy())
    assert np.array_equal(terms[:, 0], ref_cost.cpu().numpy())
    assert np.array_equal(terms[:, 1], _numpy_time_cost(times, richter, penalty))
    assert np.array_equal(obj, (terms[:, 0] + terms[:, 1]) + terms[:, 2])
    soft = np.zeros(B)
    tol = np.zeros(B)
    for k, mv in constraints:
        ex = X.max_magnitude(times, coeffs, k)
        dmax = 1e-13 * ex["value"] + 8 * (N - 1 - k) * EPS * ex["scale"]
        with np.errstate(over="ignore"):
            cur = np.minimum(mcost, np.exp((ex["value"] - mv) / mv * weight))
        soft += cur
        tol += np.where(cur < mcost, cur * weight * dmax / mv, 0.0) + 4 * EPS * cur
    assert (np.abs(terms[:, 2] - soft) <= tol).all(), np.max(np.abs(terms[:, 2] - soft) - tol)
    if constraints and constraints[0][1] == 1e-3:
        assert (terms[:, 2] >= mcost).all()  # exp overflowed: the clamp applies


@pytest.mark.gpu
def test_time_objective_not_spd_and_bad_time(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 4, 3, 8
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=4000)
    prob = m.Problem(N, r, K, D)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    times[3, 1] = -1.0
    times[5, 2] = np.inf  # the solve's factorisation meets a non-finite pivot: STATUS_NOT_SPD
    obj, terms, coeffs, status = solver.time_objective(prob, torch.from_numpy(times).cuda(),
                                                       torch.from_numpy(d_fixed).cuda(), constraints=((1, 3.0),))
    torch.cuda.synchronize()
    obj, status = obj.cpu().numpy(), status.cpu().numpy()
    assert status[3] & m.STATUS_BAD_TIME and status[5] & m.STATUS_NOT_SPD and status[5] & m.STATUS_BAD_TIME
    assert np.array_equal(np.isnan(obj), status != 0) and (status[[0, 1, 2, 4, 6, 7]] == 0).all()
    bad = m.time_objective_params(constraints=((1, 0.0),))
    with pytest.raises(RuntimeError, match="rc=-1"):
        solver._check(solver.lib.mtg_time_objective_batch_f64(
            solver.h, __import__("ctypes").byref(prob.c), B, torch.from_numpy(times).cuda().data_ptr(),
            torch.from_numpy(d_fixed).cuda().data_ptr(), None, __import__("ctypes").byref(bad),
            coeffs.data_ptr(), torch.empty(B, dtype=torch.float64, device="cuda").data_ptr(), None, None, None),
            "mtg_time_objective_batch_f64")


@pytest.mark.gpu
def test_host_variants_match_device(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 5, 3, 20011
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=5000)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    tt, df = torch.from_numpy(times).cuda(), torch.from_numpy(d_fixed).cuda()
    cons = ((1, 2.0), (2, 3.0))
    for with_free in (False, True):
        d_free = None
        if with_free:
            d_free = torch.empty((B, D, prob.n_free), dtype=torch.float64, device="cuda")
            solver.solve_linear(prob, tt, df, d_free=d_free)
            d_free = d_free * 1.01
        obj, terms, coeffs, status = solver.time_objective(prob, tt, df, d_free, constraints=cons)
        v, t, s, st = solver.max_magnitude(tt, coeffs, (1, 2))
        torch.cuda.synchronize()
        for pinned in (False, True):
            def buf(shape, dtype=np.float64):
                a = torch.empty(shape, dtype=torch.float64 if dtype == np.float64 else torch.int32)
                return a.pin_memory() if pinned else a.numpy()
            h_c, h_o, h_t, h_s = buf((B, K, D, N)), buf((B,)), buf((B, 3)), buf((B,), np.int32)
            solver.time_objective_host(prob, times, d_fixed, d_free.cpu().numpy() if with_free else None,
                                       m.time_objective_params(constraints=cons), h_c, h_o, h_t, h_s)
            for a, b in ((h_c, coeffs), (h_o, obj), (h_t, terms), (h_s, status)):
                assert np.array_equal(np.asarray(a), b.cpu().numpy(), equal_nan=True)
            hv, ht, hs, hst = buf((B, 2)), buf((B, 2)), buf((B, 2), np.int32), buf((B,), np.int32)
            solver.max_magnitude_host(times, np.asarray(h_c), (1, 2), hv, ht, hs, hst)
            for a, b in ((hv, v), (ht, t), (hs, s), (hst, st)):
                assert np.array_equal(np.asarray(a), b.cpu().numpy())
