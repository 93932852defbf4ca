"""The time-only nonlinear optimiser (mtg_optimize_time_batch_f64): PolynomialOptimizationNonLinear::optimize() with
kSquaredTime or kRichterTime, as the compass search that include/mtg_b200.h defines.

`replay` restates that search in NumPy over any objective provider.  On the CPU it runs over analytic objectives and
the fp64 oracle; on the GPU the entry must equal the replay whose every f comes from mtg_time_objective_batch_f64,
bit for bit, and must meet the assertions of the reference's UnconstrainedNonlinear test."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_optimize_time.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_optimize_time")

LOWER = 0.1
NOT_SPD = 2
FTOL, XTOL, MAXEVAL, FAILURE, INVALID_ARGS, ROUNDOFF = 3, 4, 5, -1, -2, -4
DEFAULTS = dict(f_abs=-1.0, f_rel=0.05, x_rel=-1.0, x_abs=-1.0, initial_stepsize_rel=0.1, max_iterations=3000)
# the UnconstrainedNonlinear test's NonlinearOptimizationParameters (reference test_polynomial_optimization.cpp:402-447)
REF_TEST_PARAMS = dict(max_iterations=3000, f_rel=0.05, x_rel=0.1, initial_stepsize_rel=0.1)


def replay(times, objective_fn, margin=None, **params):
    """The search of include/mtg_b200.h for B rows.  objective_fn(rows, X) -> (f [n], status [n]) at times X [n][K]
    of original rows `rows` [n], optionally with a third array: the scale of the rounding in f (default |f|).
    -> dict(x, f, evaluations, result, status).  margin [B] (optional output): per row, the smallest distance of a
    comparison between objective values that decided the row, relative to the larger scale of the two (candidates
    with the same times as what they are compared with are skipped: their values are equal under any objective)."""
    p = dict(DEFAULTS, **params)
    x = np.array(times, dtype=np.float64)
    B, K = x.shape
    NC = 2 * K
    if margin is not None:
        margin[:] = np.inf

    def near(rows, a, b, scale=None):
        if margin is not None:
            with np.errstate(divide="ignore", invalid="ignore"):
                d = np.abs(a - b) / (np.abs(b) if scale is None else scale)
            np.minimum.at(margin, rows, np.where(np.isnan(d), np.inf, d))

    def evaluate(rows, X):
        f_, st_, *sc = objective_fn(rows, X)
        return f_, st_, (sc[0] if sc else np.abs(f_))
    f = np.full(B, np.nan)
    fs = np.full(B, np.nan)  # the scale of f's rounding
    ev = np.zeros(B, dtype=np.int32)
    res = np.full(B, FAILURE, dtype=np.int32)
    st = np.zeros(B, dtype=np.int32)
    bad = (~(x > 0.0) | ~np.isfinite(x)).any(axis=1)
    low = ~bad & (x < LOWER).any(axis=1)
    rows = np.nonzero(~bad)[0]
    ev[rows] = 1
    if rows.size:
        f[rows], st0, fs[rows] = evaluate(rows, x[rows])
        st[rows] |= st0
        rows = rows[~low[rows] & ~(st0 & NOT_SPD).astype(bool)]
    rho = p["initial_stepsize_rel"] if p["initial_stepsize_rel"] > 0 else 0.1
    delta = rho * x
    maxit = p["max_iterations"]
    fits = (lambda e: maxit < 0 or e + NC <= maxit)
    if not fits(1):
        res[rows] = MAXEVAL
        rows = rows[:0]
    e = 1
    xtol_on = p["x_rel"] >= 0 or p["x_abs"] >= 0
    while rows.size:
        e += NC
        n = rows.size
        xr, dr, fr = x[rows], delta[rows], f[rows]
        cand = np.repeat(xr[:, None, :], NC, axis=1)
        for i in range(K):
            cand[:, 2 * i, i] = xr[:, i] + dr[:, i]
            v = xr[:, i] - dr[:, i]
            cand[:, 2 * i + 1, i] = np.where(v > LOWER, v, LOWER)
        fc, stc, sc = evaluate(np.repeat(rows, NC), cand.reshape(n * NC, K))
        fc, stc, sc = fc.reshape(n, NC), stc.reshape(n, NC), sc.reshape(n, NC)
        notspd = (stc & NOT_SPD).any(axis=1)
        with np.errstate(invalid="ignore"):
            below = fc < fr[:, None]
        acc = below.any(axis=1) & ~notspd
        best = np.argmin(np.where(below, fc, np.inf), axis=1)
        ar = np.arange(n)
        fn, xn, sn = fc[ar, best], cand[ar, best], sc[ar, best]
        same_x = (cand == xr[:, None, :]).all(axis=2)
        same_best = (cand == xn[:, None, :]).all(axis=2)
        sr = fs[rows]
        for j in range(NC):
            m = ~same_x[:, j]
            near(rows[m], fc[m, j], fr[m], np.maximum(sc[m, j], sr[m]))
            m = acc & ~same_best[:, j]
            near(rows[m], fc[m, j], fn[m], np.maximum(sc[m, j], sn[m]))
        df = np.abs(fn - fr)
        if p["f_rel"] >= 0:
            near(rows[acc], df[acc], p["f_rel"] * np.abs(fn[acc]))
        if p["f_abs"] > 0:
            near(rows[acc], df[acc], np.full(int(acc.sum()), p["f_abs"]))
        with np.errstate(invalid="ignore"):
            ftol = ((p["f_rel"] >= 0) & (df <= p["f_rel"] * np.abs(fn))) | ((p["f_abs"] >= 0) & (df <= p["f_abs"]))
        dx = np.abs(xn - xr)
        xtol_acc = xtol_on & (((p["x_rel"] >= 0) & (dx <= p["x_rel"] * np.abs(xn))) |
                              ((p["x_abs"] >= 0) & (dx <= p["x_abs"]))).all(axis=1)
        dh = dr * 0.5
        xtol_fail = xtol_on & (((p["x_rel"] >= 0) & (dh <= p["x_rel"] * np.abs(xr))) |
                               ((p["x_abs"] >= 0) & (dh <= p["x_abs"]))).all(axis=1)
        lo = xr - dh
        still = ((xr + dh == xr) & (np.where(lo > LOWER, lo, LOWER) == xr)).all(axis=1)
        r = np.zeros(n, dtype=np.int32)
        fail = ~acc & ~notspd
        r[acc & ftol] = FTOL
        r[acc & ~ftol & xtol_acc] = XTOL
        r[fail & xtol_fail] = XTOL
        r[fail & ~xtol_fail & still] = ROUNDOFF
        r[notspd] = FAILURE
        keep = (r == 0) & ~notspd
        if not fits(e):
            r[keep] = MAXEVAL
            keep[:] = False
        st[rows[notspd]] |= NOT_SPD
        x[rows[acc]] = xn[acc]
        f[rows[acc]] = fn[acc]
        fs[rows[acc]] = sn[acc]
        delta[rows[fail]] = dh[fail]
        done = rows[~keep]
        ev[done] = e
        res[done] = r[~keep]
        rows = rows[keep]
    return dict(x=x, f=f, evaluations=ev, result=res, status=st)


def build_binary():
    """C++ check of BatchPolynomialOptimization<10>::optimizeTime against the C-ABI entry
    (tests/cpp/test_optimize_time.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


# ---- CPU: the replay on analytic objectives -------------------------------------------------------------------------
def analytic(fn):
    """An objective provider from fn(X [n][K]) -> f [n]; every status 0."""
    def objective(rows, X):
        return fn(X), np.zeros(len(X), dtype=np.int32)
    return objective


def test_separable_convex_reaches_its_minimiser():
    target = np.array([0.7, 2.0, 1.3])
    out = replay(np.array([[1.0, 1.0, 1.0], [3.0, 0.5, 2.5]]), analytic(lambda X: ((X - target) ** 2).sum(axis=1)),
                 f_rel=-1.0, x_abs=1e-10, max_iterations=-1)
    assert (out["result"] == XTOL).all(), out["result"]
    assert np.abs(out["x"] - target).max() < 1e-8
    assert ((out["evaluations"] - 1) % 6 == 0).all() and (out["evaluations"] > 7).all()


def test_minimiser_below_the_bound_stops_on_the_bound():
    # no tolerance: an x tolerance would also stop the poll that moves x_0 from just above 0.1 onto it
    out = replay(np.array([[1.0, 2.0]]), analytic(lambda X: ((X - np.array([0.02, 1.5])) ** 2).sum(axis=1)),
                 f_rel=-1.0, max_iterations=-1)
    assert out["result"][0] == ROUNDOFF
    assert out["x"][0, 0] == LOWER and abs(out["x"][0, 1] - 1.5) < 1e-9


def test_flat_objective_ends_roundoff_limited():
    out = replay(np.array([[1.0, 3.0], [0.1, 7.5]]), analytic(lambda X: np.zeros(len(X))), f_rel=-1.0,
                 max_iterations=-1)
    assert (out["result"] == ROUNDOFF).all()
    assert np.array_equal(out["x"], [[1.0, 3.0], [0.1, 7.5]])
    # every poll fails: delta halves from 0.1 x down to where x +- delta rounds to x, about 55 times
    polls = (out["evaluations"] - 1) // 4
    assert (polls > 50).all() and (polls < 60).all(), polls


def test_every_stopping_rule():
    quad = analytic(lambda X: ((X - 2.0) ** 2).sum(axis=1) + 1.0)
    x0 = np.array([[1.0, 1.5, 3.0]])
    assert replay(x0, quad, f_rel=0.5)["result"][0] == FTOL
    assert replay(x0, quad, f_rel=-1.0, f_abs=10.0)["result"][0] == FTOL
    # x_rel stops an accepted poll whose one moved coordinate changed by <= x_rel |x|
    assert replay(x0, quad, f_rel=-1.0, x_rel=0.2)["result"][0] == XTOL
    assert replay(x0, quad, f_rel=-1.0, x_abs=1e-3, max_iterations=-1)["result"][0] == XTOL
    # max_iterations counts objective evaluations: the start, then 2K per poll
    K = x0.shape[1]
    for maxit, polls in ((0, 0), (1, 0), (1 + 2 * K - 1, 0), (1 + 2 * K, 1), (1 + 4 * K, 2)):
        out = replay(x0, quad, f_rel=-1.0, x_abs=-1.0, x_rel=-1.0, max_iterations=maxit)
        assert out["result"][0] == MAXEVAL and out["evaluations"][0] == 1 + 2 * K * polls, (maxit, out)


def test_edge_rows():
    quad = analytic(lambda X: ((X - 2.0) ** 2).sum(axis=1))
    x0 = np.array([[1.0, 0.0], [1.0, -1.0], [np.nan, 1.0], [1.0, np.inf], [0.05, 1.0], [1.0, 1.0]])
    out = replay(x0, quad)
    assert (out["result"][:5] == FAILURE).all() and out["result"][5] != FAILURE
    assert (out["evaluations"][:4] == 0).all() and out["evaluations"][4] == 1
    assert np.array_equal(out["x"][:5], x0[:5], equal_nan=True)

    def spd_fail(rows, X):  # the start of row 0 and every candidate of row 1 fail to solve
        st = np.zeros(len(X), dtype=np.int32)
        st[(rows == 0) | ((rows == 1) & (X[:, 0] != 1.0) | (rows == 1) & (X[:, 1] != 1.0))] = NOT_SPD
        return ((X - 2.0) ** 2).sum(axis=1), st
    out = replay(np.ones((2, 2)), spd_fail)
    assert (out["result"] == FAILURE).all() and (out["status"] & NOT_SPD).all()
    assert out["evaluations"].tolist() == [1, 5] and np.array_equal(out["x"], np.ones((2, 2)))


def test_rows_are_independent_of_their_batch():
    rng = np.random.default_rng(3)
    targets = rng.uniform(0.2, 3.0, size=(20, 4))

    def obj(rows, X):
        return ((X - targets[rows]) ** 2).sum(axis=1) + np.abs(X - targets[rows]).max(axis=1), np.zeros(len(X), "i4")
    x0 = rng.uniform(0.5, 2.0, size=(20, 4))
    full = replay(x0, obj, f_rel=-1.0, x_abs=1e-6)
    for b in (0, 7, 19):
        one = replay(x0[b:b + 1], lambda rows, X: obj(np.full(len(rows), b), X), f_rel=-1.0, x_abs=1e-6)
        for k in ("x", "f", "evaluations", "result"):
            assert np.array_equal(full[k][b:b + 1], one[k]), k


@pytest.mark.parametrize("D,r,K,seed,bounds,v_max,a_max",
                         [c for c in __import__("test_oracle").REF_PARAMS if c[2] <= 10])
def test_replay_over_the_oracle_descends(oracle, D, r, K, seed, bounds, v_max, a_max):
    """f never rises above its start (the non-smooth max-magnitude term included)."""
    pos = oracle.create_random_positions(K, D, -bounds, bounds, seed)[None]
    times = oracle.nfabian(pos[0], v_max, a_max)[None]
    obj = oracle_objective(oracle, 10, r, pos, ((1, v_max), (2, a_max)), 0)
    out = replay(times, obj, **REF_TEST_PARAMS)
    assert out["result"][0] in (FTOL, XTOL, MAXEVAL, ROUNDOFF)
    assert out["f"][0] <= obj(np.array([0]), times)[0][0]


def test_null_handle_is_refused_without_a_device():
    """A handle needs a device, so on the CPU only the null-handle refusal can run; refusals with a live handle, and
    that they launch nothing, are test_edge_rows_and_refusals."""
    import mav_trajectory_generation_b200 as m
    lib = m.load()
    p = m.Problem(10, 4, 3, 3)
    obj = m.time_objective_params(constraints=((1, 3.0),))
    prm = m.mellinger_params()
    for fn in (lib.mtg_optimize_time_batch_f64, lib.mtg_optimize_time_batch_host_f64):
        args = [None, C.byref(p.c), 1, None, None, C.byref(obj), C.byref(prm)] + [None] * 7
        if fn is lib.mtg_optimize_time_batch_f64:
            args.append(None)
        assert fn(*args) == -1  # MTG_ERR_BAD_ARG


# ---- the fp64 oracle's objective ------------------------------------------------------------------------------------
def oracle_objective(oracle, N, r, positions, constraints, time_cost, penalty=500.0, weight=100.0, max_cost=1e12):
    """objectiveFunctionTime over the fp64 oracle's solve and computeCost and the binary128 maxima of its
    coefficients, summed in the reference's order; the scale of its rounding leaves out soft terms clamped at
    max_cost, which are exact under any solve."""
    import extrema_oracle as X

    def objective(rows, T):
        n, K = T.shape
        D = positions.shape[2]
        coeffs, cost = np.zeros((n, K, D, N)), np.zeros(n)
        for q, b in enumerate(rows):
            mask, values = oracle.waypoint_problem(N, positions[b])
            s = oracle.solve(N, r, mask, values, T[q], want_cost=True)
            coeffs[q], cost[q] = s["coeffs"], s["cost"]
        total = np.zeros(n)
        for i in range(K):
            total = total + T[:, i]
        time_term = total * penalty if time_cost else total * total * penalty
        soft, unclamped = np.zeros(n), np.zeros(n)
        for k, mv in constraints:
            with np.errstate(over="ignore"):
                term = np.minimum(max_cost, np.exp((X.max_magnitude(T, coeffs, k)["value"] - mv) / mv * weight))
            soft = soft + term
            unclamped = unclamped + np.where(term < max_cost, term, 0.0)
        return (cost + time_term) + soft, np.zeros(n, dtype=np.int32), (cost + time_term) + unclamped
    return objective


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_objective(solver, prob, d_fixed, constraints, time_cost, **kw):
    """f and status from mtg_time_objective_batch_f64 at the materialised times."""
    import torch

    def objective(rows, X):
        obj, _, _, st = solver.time_objective(prob, _cuda(X), _cuda(d_fixed[rows]), constraints=constraints,
                                              time_cost=time_cost, **kw)
        torch.cuda.synchronize()
        return obj.cpu().numpy(), st.cpu().numpy()
    return objective


def run_entry(solver, prob, times, d_fixed, constraints, time_cost, **params):
    import torch
    import mav_trajectory_generation_b200 as m
    out = solver.optimize_time(prob, _cuda(times), _cuda(d_fixed), constraints=constraints, time_cost=time_cost,
                               params=m.mellinger_params(**params))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_against_replay(solver, prob, times, d_fixed, constraints, time_cost, what, **params):
    """The entry equals the replay over the objective entry, bit for bit; so do its coefficients, objective and terms
    against the objective entry at the returned times.  Returns the entry's outputs."""
    import torch
    out = run_entry(solver, prob, times, d_fixed, constraints, time_cost, **params)
    rep = replay(times, gpu_objective(solver, prob, d_fixed, constraints, time_cost), **params)
    assert np.array_equal(out["result"], rep["result"]), (what, np.unique(out["result"] - rep["result"],
                                                                          return_counts=True))
    assert np.array_equal(out["evaluations"], rep["evaluations"]), what
    assert np.array_equal(out["seg_times"], rep["x"], equal_nan=True), what
    assert np.array_equal(out["objective"], rep["f"], equal_nan=True), what
    obj, terms, coeffs, st = solver.time_objective(prob, _cuda(out["seg_times"]), _cuda(d_fixed),
                                                   constraints=constraints, time_cost=time_cost)
    torch.cuda.synchronize()
    assert np.array_equal(out["terms"], terms.cpu().numpy(), equal_nan=True), what
    assert np.array_equal(out["coeffs"], coeffs.cpu().numpy(), equal_nan=True), what
    assert np.array_equal(out["status"], st.cpu().numpy() | rep["status"]), what
    return out


WAYPOINT_SHAPES = [(6, 2), (8, 3), (10, 4), (12, 5)]
VA = ((1, 3.0), (2, 5.0))


@pytest.mark.gpu
@pytest.mark.parametrize("time_cost", (0, 1))
@pytest.mark.parametrize("constraints", ((), ((1, 3.0),), VA))
def test_entry_equals_the_replay_every_objective(solver, oracle, time_cost, constraints):
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 1024
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=41000 + 10 * time_cost + len(constraints))
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    out = check_against_replay(solver, m.Problem(N, r, K, D), times, d_fixed, constraints, time_cost,
                               f"cost={time_cost} constraints={constraints}", **REF_TEST_PARAMS)
    print(f"time_cost={time_cost} {constraints}: results {dict(zip(*np.unique(out['result'], return_counts=True)))}"
          f", evaluations mean {out['evaluations'].mean():.1f}")
    assert (out["result"] > 0).mean() > 0.9


@pytest.mark.gpu
@pytest.mark.parametrize("N,r", WAYPOINT_SHAPES)
@pytest.mark.parametrize("K", [1, 3, 16, 50])
def test_entry_equals_the_replay_every_shape(solver, oracle, N, r, K):
    import mav_trajectory_generation_b200 as m
    D = 3
    B = 256 if K == 50 else 1024
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=42000 + 100 * N + K)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    out = check_against_replay(solver, m.Problem(N, r, K, D), times, d_fixed, VA, 0, f"N={N} K={K}",
                               **REF_TEST_PARAMS)
    assert (out["evaluations"] > 1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("D", (1, 4))
def test_entry_equals_the_replay_every_dimension(solver, oracle, D):
    import mav_trajectory_generation_b200 as m
    N, r, K, B = 10, 4, 5, 1024
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=43000 + D)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    # without tolerances on f, so rows also stop on x and on rounding
    check_against_replay(solver, m.Problem(N, r, K, D), times, d_fixed, VA, 1, f"D={D}", f_rel=-1.0, x_rel=1e-6,
                         max_iterations=-1)


def chunk_rows(prob, n_fixed):
    """Rows per chunk of candidates in launch_optimize_time (its 512 MiB kTimeSearchBudget)."""
    K, D, N = prob.K, prob.D, prob.N
    per_x = (K + D * n_fixed + K * D * N + 1) * 8 + 4
    return max(8, (512 << 20) // (per_x * 2 * K) // 8 * 8)


@pytest.mark.gpu
@pytest.mark.parametrize("K,D,B,params", [
    (16, 3, 3757, REF_TEST_PARAMS),
    # 2K = 398 candidates per row: a tail chunk of 11 rows holds 4378, not a multiple of 16; no tolerance is met
    # within three polls, so max_iterations stops every row after exactly three
    (199, 1, 203, dict(f_rel=-1.0, x_rel=1e-3, max_iterations=1 + 2 * 199 * 3)),
])
def test_entry_spanning_several_chunks_equals_the_replay(solver, oracle, K, D, B, params):
    """Batches of several candidate chunks and a partial tail chunk, each poll: the per-chunk offsets, the reused
    candidate buffers and the count that accumulates over several decision launches."""
    import mav_trajectory_generation_b200 as m
    N, r = 10, 4
    prob = m.Problem(N, r, K, D)
    chunk = chunk_rows(prob, prob.n_fixed)
    assert B > chunk and B % chunk, (B, chunk)
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=45000 + K)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    out = check_against_replay(solver, prob, times, d_fixed, VA, 0, f"K={K} B={B}", **params)
    polls = (out["evaluations"] - 1) // (2 * K)
    print(f"K={K} B={B} chunk {chunk}: polls {dict(zip(*np.unique(polls, return_counts=True)))}")
    assert (polls >= 1).all()
    if K == 199:  # every row runs three polls, so each later poll spans several chunks too
        assert (polls == 3).all()


@pytest.mark.gpu
def test_not_spd_rows_equal_the_replay(solver, oracle):
    """Rows with valid times whose solve fails the factorisation (STATUS_NOT_SPD; the waypoint kernel at N = 12 with
    segment times three to four decades apart): one at its start times, one only at a candidate of its first poll."""
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 12, 5, 3, 1, 64
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=46000)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    start = [float.fromhex(v) for v in ("0x1.7354e5349fc49p+9", "0x1.3319c37f4d71dp-3", "0x1.537228c10abbfp+8")]
    cand = [float.fromhex(v) for v in ("0x1.17f746c9e591ep+7", "0x1.a1f99b2667699p-3", "0x1.2ba10b27a487ep+9")]
    times[5], times[40] = start, cand
    prob = m.Problem(N, r, K, D)
    out = check_against_replay(solver, prob, times, d_fixed, VA, 0, "NOT_SPD", **REF_TEST_PARAMS)
    for b, ev in ((5, 1), (40, 1 + 2 * K)):
        assert out["result"][b] == FAILURE and out["status"][b] & NOT_SPD and out["evaluations"][b] == ev, b
        assert np.array_equal(out["seg_times"][b], times[b]), b
    assert out["status"][40] == NOT_SPD  # the start itself solves
    others = np.setdiff1d(np.arange(B), [5, 40])
    assert (out["result"][others] != FAILURE).mean() > 0.9


@pytest.mark.gpu
def test_max_iterations_equals_the_replay(solver, oracle):
    """max_iterations counts objective evaluations: 0 and 2K stop every row after its start evaluation, 1 + 2K after
    one poll, 1 + 4K after at most two."""
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 5, 3, 256
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=47000)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    for maxit, most in ((0, 1), (2 * K, 1), (1 + 2 * K, 1 + 2 * K), (1 + 4 * K, 1 + 4 * K)):
        out = check_against_replay(solver, prob, times, d_fixed, VA, 0, f"max_iterations={maxit}", f_rel=-1.0,
                                   max_iterations=maxit)
        assert (out["result"] == MAXEVAL).all() and (out["evaluations"] == most).all(), maxit


@pytest.mark.gpu
def test_arbitrary_mask_equals_the_replay(solver):
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(5)
    K, N, D = 5, 8, 2
    h = N // 2
    mask = (rng.rand(K + 1, h) < 0.35).astype(np.uint8)
    mask[:, 0] = 1
    mask[0, :] = 1
    mask[-1, :] = 1
    prob = m.Problem(N, h - 1, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    times = rng.uniform(1.0, 3.0, size=(1024, K))
    d_fixed = rng.uniform(-3, 3, size=(1024, D, prob.n_fixed))
    out = check_against_replay(solver, prob, times, d_fixed, ((1, 2.0),), 0, "mask", f_rel=-1.0, x_rel=1e-6,
                               max_iterations=-1)
    assert (out["evaluations"] > 1 + 2 * K).mean() > 0.5


@pytest.mark.gpu
def test_rows_alone_equal_rows_in_a_shuffled_batch_and_host_equals_device(solver, oracle):
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 2000
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=4343)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    full = run_entry(solver, prob, times, d_fixed, VA, 0, **REF_TEST_PARAMS)
    perm = np.random.default_rng(1).permutation(B)
    shuf = run_entry(solver, prob, times[perm], d_fixed[perm], VA, 0, **REF_TEST_PARAMS)
    for k in full:
        assert np.array_equal(full[k][perm], shuf[k], equal_nan=True), k
    for b in (0, 7, B - 1):
        alone = run_entry(solver, prob, times[b:b + 1], d_fixed[b:b + 1], VA, 0, **REF_TEST_PARAMS)
        for k in full:
            assert np.array_equal(full[k][b:b + 1], alone[k], equal_nan=True), (b, k)
    host = solver.optimize_time_host(prob, times, d_fixed, constraints=VA, time_cost=0,
                                     params=m.mellinger_params(**REF_TEST_PARAMS))
    for k in full:
        assert np.array_equal(full[k], host[k], equal_nan=True), k


@pytest.mark.gpu
def test_edge_rows_and_refusals(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 4, 3, 12
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=99)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    times[1, 2] = 0.0
    times[2, 0] = -1.0
    times[3, 1] = np.nan
    times[4, 3] = np.inf
    times[5, 2] = 0.05
    times[6, 1] = 1e300  # finite, but T^N overflows: the objective is not finite, so no candidate ever wins
    t_in = _cuda(times)
    keep = t_in.clone()
    out = solver.optimize_time(prob, t_in, _cuda(d_fixed), constraints=VA)
    torch.cuda.synchronize()
    assert torch.equal(t_in.nan_to_num(), keep.nan_to_num())
    o = {k: v.cpu().numpy() for k, v in out.items()}
    for b in (1, 2, 3, 4):
        assert o["result"][b] == FAILURE and o["status"][b] & 1 and o["evaluations"][b] == 0
        assert np.array_equal(o["seg_times"][b], times[b], equal_nan=True) and np.isnan(o["objective"][b])
    assert o["result"][5] == FAILURE and o["status"][5] == 0 and o["evaluations"][5] == 1
    assert np.array_equal(o["seg_times"][5], times[5])
    f5, _, c5, _ = solver.time_objective(prob, _cuda(times[5:6]), _cuda(d_fixed[5:6]), constraints=VA)
    torch.cuda.synchronize()
    assert o["objective"][5] == f5.cpu().numpy()[0] and np.array_equal(o["coeffs"][5], c5.cpu().numpy()[0])
    assert o["result"][6] == ROUNDOFF and not np.isfinite(o["objective"][6])
    assert np.array_equal(o["seg_times"][6], times[6]) and (o["evaluations"][6] - 1) % (2 * K) == 0
    assert (o["result"][[0] + list(range(7, B))] != FAILURE).all()
    # K = 1: one coordinate, two candidates per poll
    pos1, t1 = oracle.make_waypoint_batch(1, D, 64, base_seed=98)
    check_against_replay(solver, m.Problem(N, r, 1, D), t1, oracle.waypoint_d_fixed(N, pos1), VA, 0, "K=1")
    # refusals: no launch
    lib, h = solver.lib, solver.h
    before = solver.launch_count
    none_stop = m.mellinger_params(f_rel=-1.0, max_iterations=-1)
    good_obj = m.time_objective_params(constraints=VA)
    dfc = _cuda(d_fixed)

    def call(prm, obj=good_obj, t=t_in.data_ptr(), coeffs=out["coeffs"].data_ptr()):
        return lib.mtg_optimize_time_batch_f64(h, C.byref(prob.c), B, t, dfc.data_ptr(), C.byref(obj) if obj else None,
                                               prm, coeffs, out["seg_times"].data_ptr(), *([None] * 6))
    assert call(C.byref(none_stop)) == -1
    assert call(None) == -1
    assert call(C.byref(m.mellinger_params()), obj=None) == -1
    assert call(C.byref(m.mellinger_params()), obj=m.time_objective_params(time_cost=2)) == -1
    assert call(C.byref(m.mellinger_params()), obj=m.time_objective_params(constraints=((1, 0.0),))) == -1
    assert call(C.byref(m.mellinger_params()), obj=m.time_objective_params(constraints=((N - 1, 1.0),))) == -1
    assert call(C.byref(m.mellinger_params()), t=None) == -1
    assert call(C.byref(m.mellinger_params()), coeffs=None) == -1
    assert solver.launch_count == before


def riemann_cost(times, coeffs, r, dt=1e-3):
    """checkCost's numeric integral (reference test_polynomial_optimization.cpp:176-197): sum over t = 0, dt, ... < T
    of |p^(r)(t)|^2 dt."""
    K, D, N = coeffs.shape
    total = 0.0
    for i in range(K):
        t = np.arange(0.0, times[i], dt)
        for d in range(D):
            dc = np.polynomial.polynomial.polyder(coeffs[i, d], r)
            total += (np.polynomial.polynomial.polyval(t, dc) ** 2).sum() * dt
    return total


@pytest.mark.gpu
@pytest.mark.parametrize("time_cost", (0, 1))
@pytest.mark.parametrize("D,r,K,seed,bounds,v_max,a_max", __import__("test_oracle").REF_PARAMS)
def test_reference_unconstrained_nonlinear_assertions(solver, oracle, time_cost, D, r, K, seed, bounds, v_max, a_max):
    """UnconstrainedNonlinear (reference test_polynomial_optimization.cpp:402-447) with kSquaredTime and with
    kRichterTime: Nfabian start, soft v / a limits, max_iterations 3000, f_rel 0.05, x_rel 0.1."""
    import torch
    import mav_trajectory_generation_b200 as m
    from test_oracle import check_path
    from test_time_scaling import exact_maxima
    N = 10
    pos = oracle.create_random_positions(K, D, -bounds, bounds, seed)
    prob = m.Problem(N, r, K, D)
    d_fixed = oracle.waypoint_d_fixed(N, pos[None])
    times = oracle.nfabian(pos, v_max, a_max)[None]
    cons = ((1, v_max), (2, a_max))
    out = run_entry(solver, prob, times, d_fixed, cons, time_cost, **REF_TEST_PARAMS)
    assert out["result"][0] not in (FAILURE, INVALID_ARGS), out["result"]

    def total_cost(t):  # getTotalCostWithSoftConstraints
        obj, _, _, _ = solver.time_objective(prob, _cuda(t), _cuda(d_fixed), constraints=cons, time_cost=time_cost,
                                             maximum_cost=1e9)
        torch.cuda.synchronize()
        return float(obj.cpu().numpy()[0])
    start, end = total_cost(times), total_cost(out["seg_times"])
    print(f"D={D} r={r} K={K} cost={time_cost}: result {out['result'][0]} after {out['evaluations'][0]} evaluations, "
          f"total cost {start:.6g} -> {end:.6g}")
    assert end <= 1.1 * start, (start, end)
    mask, values = oracle.waypoint_problem(N, pos)
    check_path(oracle, N, mask, values, out["seg_times"][0], out["coeffs"][0])
    ve, ae = exact_maxima(out["seg_times"], out["coeffs"])
    assert ve[0] <= 1.5 * v_max and ae[0] <= 1.5 * a_max, (ve, ae)
    cost = out["terms"][0, 0]
    numeric = riemann_cost(out["seg_times"][0], out["coeffs"][0], r)
    assert abs(cost - numeric) <= 0.1 * numeric, (cost, numeric)


@pytest.mark.gpu
@pytest.mark.parametrize("time_cost", (0, 1))
@pytest.mark.parametrize("K", (3, 6))
def test_decisions_agree_with_the_fp64_oracle(solver, oracle, time_cost, K):
    """The replay over the fp64 oracle's solve and cost and the binary128 maxima (an independent objective) against
    the entry: result and evaluations equal on every row whose deciding comparisons all lie more than 1e-10
    (relative) from equality; at least 90 % of rows must qualify."""
    import mav_trajectory_generation_b200 as m
    N, r, D, rows = 10, 4, 3, 40
    pos, times = oracle.make_waypoint_batch(K, D, rows, base_seed=44000 + K)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    out = run_entry(solver, m.Problem(N, r, K, D), times, d_fixed, VA, time_cost, **REF_TEST_PARAMS)
    margin = np.empty(rows)
    rep = replay(times, oracle_objective(oracle, N, r, pos, VA, time_cost), margin=margin, **REF_TEST_PARAMS)
    ok = margin > 1e-10
    print(f"K={K} cost={time_cost}: {int((~ok).sum())} of {rows} rows have a comparison within 1e-10")
    assert ok.mean() >= 0.9
    assert np.array_equal(out["result"][ok], rep["result"][ok])
    assert np.array_equal(out["evaluations"][ok], rep["evaluations"][ok])
    assert np.array_equal(out["seg_times"][ok], rep["x"][ok])


@pytest.mark.gpu
def test_batch_class_equals_the_entry():
    out = subprocess.run([build_binary()], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert " 0 failures" in out.stdout
