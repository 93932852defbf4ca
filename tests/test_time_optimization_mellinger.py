"""The Mellinger outer loop (mtg_optimize_time_mellinger_batch_f64): PolynomialOptimizationNonLinear::optimize() with
kMellingerOuterLoop, as the projected-gradient descent that include/mtg_b200.h defines, then
scaleSegmentTimesWithViolation.

`replay` restates that descent in NumPy over any (cost, gradient) and candidate-cost providers.  On the CPU it runs
over the fp64 oracle; on the GPU the entry must equal the replay whose every J and g come from
mtg_cost_gradient_mellinger_batch_f64, bit for bit, and must meet the reference TimeScaling test's assertions."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_mellinger_outer_loop.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_mellinger_outer_loop")

LOWER = 0.1
L_STEPS = 8
ARMIJO = 1e-4
SUCCESS, FTOL, XTOL, MAXEVAL, FAILURE, ROUNDOFF = 1, 3, 4, 5, -1, -4
DEFAULTS = dict(f_abs=-1.0, f_rel=0.05, x_rel=-1.0, x_abs=-1.0, initial_stepsize_rel=0.1, max_iterations=3000)


def candidates(x, g, alpha):
    """[rows][L][K] candidate times: max(l, fl(x - fl(a_j * g))) with a_j = alpha * 2^(1-j)."""
    steps = alpha[:, None] * (2.0 ** (1 - np.arange(L_STEPS)))[None, :]
    v = x[:, None, :] - steps[:, :, None] * g[:, None, :]
    return np.where(v > LOWER, v, LOWER), steps


def replay(times, grad_fn, cand_cost_fn, margin=None, drift=None, **params):
    """The descent of include/mtg_b200.h for B rows.  grad_fn(rows, x) -> (J [n], g [n][K]); cand_cost_fn(rows, xc)
    -> J [n][L] at candidate times xc [n][L][K].  -> (relative times, iterations, result).  margin [B] (optional
    output): per row, the smallest relative distance of an acceptance or stopping decision from its threshold.  When
    grad_fn also returns e [n][K], a bound on each gradient's error, drift [B][K] (optional output) sums step * e over
    the accepted steps: how far the times may move from that error alone."""
    p = dict(DEFAULTS, **params)
    if margin is not None:
        margin[:] = np.inf

    def near(b, value, threshold):
        if margin is not None:
            with np.errstate(divide="ignore", invalid="ignore"):
                margin[b] = min(margin[b], abs(value - threshold) / abs(threshold))
    x = np.array(times, dtype=np.float64)
    B, K = x.shape
    iters = np.zeros(B, dtype=np.int32)
    result = np.full(B, FAILURE, dtype=np.int32)
    bad = (~(x > 0.0) | ~np.isfinite(x)).any(axis=1)
    low = ~bad & (x < LOWER).any(axis=1)
    active = ~bad & ~low
    if p["max_iterations"] == 0:
        result[active] = MAXEVAL
        active[:] = False
    rows = np.nonzero(active)[0]
    alpha = None
    k = 0
    while rows.size:
        xr = x[rows]
        J, g, *gerr = grad_fn(rows, xr)
        if k == 0:
            rel = p["initial_stepsize_rel"] if p["initial_stepsize_rel"] > 0 else 0.1
            alpha = np.zeros(B)
            with np.errstate(divide="ignore", invalid="ignore"):  # a zero gradient stops its row below
                alpha[rows] = (rel * xr.max(axis=1)) / np.abs(g).max(axis=1)
        with np.errstate(invalid="ignore"):
            xc, steps = candidates(xr, g, alpha[rows])
        Jc = cand_cost_fn(rows, xc)
        zero = (g == 0.0).all(axis=1)
        acc = np.full(rows.size, -1)
        for j in range(L_STEPS):
            dec = np.zeros(rows.size)
            for i in range(K):
                dec = dec + g[:, i] * (xc[:, j, i] - xr[:, i])
            thr = J + ARMIJO * dec
            for q in np.nonzero((acc < 0) & ~zero)[0]:
                near(rows[q], Jc[q, j], thr[q])
            ok = (Jc[:, j] <= thr) & (acc < 0) & ~zero
            acc[ok] = j
        keep = np.zeros(rows.size, dtype=bool)
        for q, b in enumerate(rows):
            if zero[q]:
                iters[b], result[b] = k, SUCCESS
                continue
            if acc[q] < 0:
                iters[b], result[b] = k, ROUNDOFF
                continue
            xn = xc[q, acc[q]]
            Jn = Jc[q, acc[q]]
            iters[b] = k + 1
            dJ = abs(Jn - J[q])
            dx = np.abs(xn - xr[q])
            xtol_on = p["x_rel"] >= 0 or p["x_abs"] >= 0
            xtol = xtol_on and bool(np.all(((p["x_rel"] >= 0) & (dx <= p["x_rel"] * np.abs(xn))) |
                                           ((p["x_abs"] >= 0) & (dx <= p["x_abs"]))))
            x[b] = xn
            alpha[b] = steps[q, acc[q]]
            if drift is not None and gerr:
                drift[b] += steps[q, acc[q]] * gerr[0][q]
            if p["max_iterations"] >= 0 and k + 1 >= p["max_iterations"]:
                result[b] = MAXEVAL
                continue
            if p["f_rel"] > 0:
                near(b, dJ, p["f_rel"] * abs(Jn))
            if p["f_abs"] > 0:
                near(b, dJ, p["f_abs"])
            if (p["f_rel"] >= 0 and dJ <= p["f_rel"] * abs(Jn)) or (p["f_abs"] >= 0 and dJ <= p["f_abs"]):
                result[b] = FTOL
            elif xtol:
                result[b] = XTOL
            else:
                keep[q] = True
        rows = rows[keep]
        k += 1
    return x, iters, result


def build_binary():
    """C++ TimeScaling sequence through PolynomialOptimizationNonLinear<10> and the batch class
    (tests/cpp/test_mellinger_outer_loop.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


# ---- CPU: the replay over the fp64 oracle --------------------------------------------------------------------------
def oracle_providers(oracle, N, r, positions):
    def grad_fn(rows, x):
        out = [oracle.cost_gradient_mellinger(N, r, positions[b], x[q]) for q, b in enumerate(rows)]
        return np.array([o[0] for o in out]), np.array([o[1] for o in out])

    def cand_fn(rows, xc):
        return np.array([[oracle.cost_gradient_mellinger(N, r, positions[b], xc[q, j])[0] for j in range(L_STEPS)]
                         for q, b in enumerate(rows)])
    return grad_fn, cand_fn


def test_replay_equalises_a_mirror_symmetric_two_segment_problem(oracle):
    N, r = 10, 4
    pos = np.array([[[-2.0, 0.0, 0.0], [0.0, 0.0, 0.0], [2.0, 0.0, 0.0]]])
    g, c = oracle_providers(oracle, N, r, pos)
    x, it, res = replay(np.array([[1.0, 3.0]]), g, c, f_rel=-1.0, x_abs=1e-9, max_iterations=300)
    assert it[0] > 1 and res[0] in (XTOL, ROUNDOFF, MAXEVAL), (it, res)
    # equal to the resolution of the forward differences (0.1 s): from 2 s apart at the start
    assert abs(x[0, 0] - x[0, 1]) < 0.1, x


def test_replay_stops_one_segment_at_iteration_zero(oracle):
    N, r = 10, 4
    pos = oracle.create_random_positions(1, 3, -10, 10, 104)[None]
    g, c = oracle_providers(oracle, N, r, pos)
    x, it, res = replay(np.array([[2.5]]), g, c)
    assert it[0] == 0 and res[0] == SUCCESS and x[0, 0] == 2.5


@pytest.mark.parametrize("D,r,K,seed,bounds,v_max,a_max", __import__("test_oracle").REF_PARAMS)
def test_replay_never_raises_the_cost(oracle, D, r, K, seed, bounds, v_max, a_max):
    from test_time_scaling import velocity_ramp_times
    N = 10
    pos = oracle.create_random_positions(K, D, -bounds, bounds, seed)[None]
    times = velocity_ramp_times(pos[0], v_max, a_max)[None]
    g, c = oracle_providers(oracle, N, r, pos)
    x, it, res = replay(times, g, c)
    assert res[0] in (SUCCESS, FTOL, XTOL, MAXEVAL, ROUNDOFF)
    assert oracle.cost_gradient_mellinger(N, r, pos[0], x[0])[0] <= oracle.cost_gradient_mellinger(N, r, pos[0],
                                                                                                   times[0])[0]


def test_null_handle_is_refused_without_a_device():
    """A handle needs a device (mtg_create fails without one), so on the CPU only the null-handle refusal can run; the
    refusals of bad parameters with a live handle, and that they launch nothing, are test_edge_rows_and_refusals."""
    import mav_trajectory_generation_b200 as m
    lib = m.load()
    p = m.Problem(10, 4, 3, 3)
    prm = m.mellinger_params()
    for fn in (lib.mtg_optimize_time_mellinger_batch_f64, lib.mtg_optimize_time_mellinger_batch_host_f64):
        args = [None, C.byref(p.c), 1, None, None, C.byref(prm), 3.0, 5.0] + [None] * 9
        if fn is lib.mtg_optimize_time_mellinger_batch_f64:
            args.append(None)
        assert fn(*args) == -1  # MTG_ERR_BAD_ARG


def test_params_defaults_and_unknown_names():
    import mav_trajectory_generation_b200 as m
    prm = m.mellinger_params()
    assert (prm.f_abs, prm.f_rel, prm.x_rel, prm.x_abs, prm.initial_stepsize_rel, prm.max_iterations) == (
        -1.0, 0.05, -1.0, -1.0, 0.1, 3000)
    with pytest.raises(ValueError):
        m.mellinger_params(algorithm=1)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_providers(solver, prob, d_fixed):
    """J and g from mtg_cost_gradient_mellinger_batch_f64; a candidate's J from its `cost` output at the candidate."""
    import torch

    def grad_fn(rows, x):
        J, g = solver.cost_gradient_mellinger(prob, _cuda(x), _cuda(d_fixed[rows]))
        torch.cuda.synchronize()
        return J.cpu().numpy(), g.cpu().numpy()

    def cand_fn(rows, xc):
        n, L, K = xc.shape
        J, _ = solver.cost_gradient_mellinger(prob, _cuda(xc.reshape(n * L, K)),
                                              _cuda(np.repeat(d_fixed[rows], L, axis=0)))
        torch.cuda.synchronize()
        return J.cpu().numpy().reshape(n, L)
    return grad_fn, cand_fn


def run_entry(solver, prob, times, d_fixed, v_max, a_max, **params):
    import torch
    import mav_trajectory_generation_b200 as m
    out = solver.optimize_time_mellinger(prob, _cuda(times), _cuda(d_fixed), v_max, a_max,
                                         params=m.mellinger_params(**params))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_against_replay(solver, prob, times, d_fixed, v_max, a_max, what, **params):
    """The entry equals the replay over the Mellinger gradient entry, bit for bit, and the scaling of its relative
    times; returns the entry's outputs."""
    import torch
    out = run_entry(solver, prob, times, d_fixed, v_max, a_max, **params)
    g, c = gpu_providers(solver, prob, d_fixed)
    x, it, res = replay(times, g, c, **params)
    assert np.array_equal(out["result"], res), (what, np.unique(out["result"] - res, return_counts=True))
    assert np.array_equal(out["iterations"], it), what
    assert np.array_equal(out["relative_times"], x), what
    co, ts, w, mx, st = solver.scale_times_with_violation(prob, _cuda(x), _cuda(d_fixed), v_max, a_max)
    torch.cuda.synchronize()
    scaled = (res != FAILURE) | (out["status"] & 2).astype(bool)
    ts, co = ts.cpu().numpy(), co.cpu().numpy()
    assert np.array_equal(out["seg_times"][scaled], ts[scaled]), what
    assert np.array_equal(out["coeffs"][scaled], co[scaled]), what
    assert np.array_equal(out["within_range"][scaled], w.cpu().numpy()[scaled]), what
    cost = solver.compute_cost(prob, _cuda(out["seg_times"]), _cuda(out["coeffs"]))
    torch.cuda.synchronize()
    assert np.array_equal(out["cost"], cost.cpu().numpy()), what
    return out, x


WAYPOINT_SHAPES = [(6, 2), (8, 3), (10, 4), (12, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,r", WAYPOINT_SHAPES)
@pytest.mark.parametrize("K", [1, 3, 16, 50])
def test_entry_equals_the_replay(solver, oracle, N, r, K):
    import mav_trajectory_generation_b200 as m
    B, D = 8192, 3
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=31000 + 100 * N + K)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    out, x = check_against_replay(solver, prob, times, d_fixed, 3.0, 5.0, f"N={N} K={K}")
    res = out["result"]
    print(f"N={N} K={K}: results {dict(zip(*np.unique(res, return_counts=True)))}, "
          f"iterations max {out['iterations'].max()} mean {out['iterations'].mean():.2f}")
    if K == 1:
        assert (res == SUCCESS).all() and (out["iterations"] == 0).all()
    else:
        assert (out["iterations"] > 0).mean() > 0.5
    # no row's relative cost exceeds its starting cost
    J0, _ = gpu_providers(solver, prob, d_fixed)[0](np.arange(B), times)
    J1, _ = gpu_providers(solver, prob, d_fixed)[0](np.arange(B), x)
    assert (J1 <= J0).all()


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
    times = rng.uniform(1.0, 3.0, size=(2048, K))
    d_fixed = rng.uniform(-3, 3, size=(2048, D, prob.n_fixed))
    out, _ = check_against_replay(solver, prob, times, d_fixed, 2.0, 3.0, "mask")
    assert (out["iterations"] > 0).mean() > 0.5


@pytest.mark.gpu
def test_zero_iterations_is_the_scaling_entry(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 1024
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=777)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    out = run_entry(solver, prob, times, d_fixed, 3.0, 5.0, max_iterations=0)
    co, ts, w, mx, st = solver.scale_times_with_violation(prob, _cuda(times), _cuda(d_fixed), 3.0, 5.0)
    torch.cuda.synchronize()
    assert np.array_equal(out["seg_times"], ts.cpu().numpy()) and np.array_equal(out["coeffs"], co.cpu().numpy())
    assert np.array_equal(out["maxima"], mx.cpu().numpy()) and np.array_equal(out["status"], st.cpu().numpy())
    assert (out["result"] == MAXEVAL).all() and (out["iterations"] == 0).all()
    assert np.array_equal(out["relative_times"], times)


@pytest.mark.gpu
def test_rows_alone_equal_rows_in_a_shuffled_batch_and_host_equals_device(solver, oracle):
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 2000
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=4242)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    full = run_entry(solver, prob, times, d_fixed, 3.0, 5.0)
    perm = np.random.default_rng(1).permutation(B)
    shuf = run_entry(solver, prob, times[perm], d_fixed[perm], 3.0, 5.0)
    for k in full:
        assert np.array_equal(full[k][perm], shuf[k], equal_nan=True), k
    for b in (0, 7, B - 1):
        alone = run_entry(solver, prob, times[b:b + 1], d_fixed[b:b + 1], 3.0, 5.0)
        for k in full:
            assert np.array_equal(full[k][b:b + 1], alone[k], equal_nan=True), (b, k)
    host = solver.optimize_time_mellinger_host(prob, times, d_fixed, 3.0, 5.0)
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
    t_in = _cuda(times)
    keep = t_in.clone()
    out = solver.optimize_time_mellinger(prob, t_in, _cuda(d_fixed), 3.0, 5.0)
    torch.cuda.synchronize()
    assert torch.equal(t_in.nan_to_num(), keep.nan_to_num())
    o = {k: v.cpu().numpy() for k, v in out.items()}
    for b in (1, 2, 3, 4):
        assert o["result"][b] == FAILURE and o["status"][b] & 1 and o["iterations"][b] == 0
        assert np.array_equal(o["seg_times"][b], times[b], equal_nan=True)
        assert np.array_equal(o["relative_times"][b], times[b], equal_nan=True)
    assert o["result"][5] == FAILURE and o["status"][5] == 0 and o["iterations"][5] == 0
    assert np.array_equal(o["seg_times"][5], times[5]) and o["within_range"][5] == 0
    solved = solver.solve_linear(prob, _cuda(times[5:6]), _cuda(d_fixed[5:6]))
    torch.cuda.synchronize()
    assert np.array_equal(o["coeffs"][5], solved.cpu().numpy()[0])
    assert (o["result"][[0] + list(range(6, B))] != FAILURE).all()
    # refusals: no launch
    lib, h = solver.lib, solver.h
    before = solver.launch_count
    none_stop = m.mellinger_params(f_rel=-1.0, max_iterations=-1)
    args = lambda prm, v=3.0, a=5.0, t=t_in.data_ptr(): [h, C.byref(prob.c), B, t, _cuda(d_fixed).data_ptr(),  # noqa
                                                          prm, v, a, out["coeffs"].data_ptr(),
                                                          out["seg_times"].data_ptr()] + [None] * 7 + [None]
    assert lib.mtg_optimize_time_mellinger_batch_f64(*args(C.byref(none_stop))) == -1
    assert lib.mtg_optimize_time_mellinger_batch_f64(*args(None)) == -1
    assert lib.mtg_optimize_time_mellinger_batch_f64(*args(C.byref(m.mellinger_params()), v=0.0)) == -1
    assert lib.mtg_optimize_time_mellinger_batch_f64(*args(C.byref(m.mellinger_params()), t=None)) == -1
    assert solver.launch_count == before


@pytest.mark.gpu
@pytest.mark.parametrize("D,r,K,seed,bounds,v_max,a_max", __import__("test_oracle").REF_PARAMS)
def test_reference_time_scaling_assertions(solver, oracle, D, r, K, seed, bounds, v_max, a_max):
    """TimeScaling (reference test/test_polynomial_optimization.cpp:608-686): after optimize(), max |v| and max |a|
    are within 1e-3 of the limits and the cost is no higher than after scaleSegmentTimesWithViolation."""
    import torch
    import mav_trajectory_generation_b200 as m
    from test_time_scaling import exact_maxima, velocity_ramp_times
    N = 10
    pos = oracle.create_random_positions(K, D, -bounds, bounds, seed)
    prob = m.Problem(N, r, K, D)
    d_fixed = oracle.waypoint_d_fixed(N, pos[None])
    times = velocity_ramp_times(pos, v_max, a_max)[None]
    tt, df = _cuda(times), _cuda(d_fixed)
    co, t2, _, _, st2 = solver.scale_times_with_violation(prob, tt, df, v_max, a_max)
    scaled_cost = float(solver.compute_cost(prob, t2, co)[0])
    out = run_entry(solver, prob, t2.cpu().numpy(), d_fixed, v_max, a_max)
    torch.cuda.synchronize()
    assert out["status"][0] == 0 and out["result"][0] > 0, out["result"]
    ve, ae = exact_maxima(out["seg_times"], out["coeffs"])
    assert ve[0] <= (v_max + 1e-3) * (1 + 1e-9) and ae[0] <= (a_max + 1e-3) * (1 + 1e-9), (ve, ae)
    assert out["cost"][0] <= scaled_cost, (out["cost"][0], scaled_cost)


@pytest.mark.gpu
@pytest.mark.parametrize("N,r", WAYPOINT_SHAPES)
@pytest.mark.parametrize("K,rows", [(3, 256), (16, 256), (50, 48)])
def test_decisions_agree_with_the_fp64_oracle(solver, oracle, N, r, K, rows):
    """The replay over the fp64 oracle's costs and gradients (an independent solve) against the entry, on the first
    `rows` rows of the same batches as test_entry_equals_the_replay (rows are independent of their batch): result and
    iterations equal on every row whose acceptance and stopping decisions all lie more than 1e-10 (relative) from
    their thresholds (at least 90 % of rows must qualify), and relative times within 1e-9 of the replay's plus what
    the two gradients' difference can move them.  The Mellinger gradient is a forward difference of two costs over
    0.1 s: where the cost hardly changes, the two solves' rounding differences (1e-13..1e-10 relative at N = 12 and
    K = 50) are amplified in g, and the step carries them into the times.  The replay therefore also evaluates the
    GPU gradient at each of its iterates and allows 1e-9 |x| + 64 * sum(step * |g_oracle - g_gpu|) per time.  The
    sum is not a bound: the difference of one step moves the later iterates and so their gradients, which it does not
    see.  On an H100 80GB HBM3 the largest time difference was 24 times the sum (N = 12, K = 3) and 16 times (N = 12,
    K = 16); at N <= 10 it stayed below 8 times."""
    import mav_trajectory_generation_b200 as m
    B, D = 8192, 3
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=31000 + 100 * N + K)
    d_fixed = oracle.waypoint_d_fixed(N, pos)
    out = run_entry(solver, m.Problem(N, r, K, D), times, d_fixed, 3.0, 5.0)
    g_or, c = oracle_providers(oracle, N, r, pos[:rows])
    g_gpu = gpu_providers(solver, m.Problem(N, r, K, D), d_fixed[:rows])[0]

    def g(rows_, x_):
        J, gr = g_or(rows_, x_)
        return J, gr, np.abs(gr - g_gpu(rows_, x_)[1])
    margin, drift = np.empty(rows), np.zeros((rows, K))
    x, it, res = replay(times[:rows], g, c, margin=margin, drift=drift)
    ok = margin > 1e-10
    print(f"N={N} K={K}: {int((~ok).sum())} of {rows} rows have a decision within 1e-10 of its threshold")
    assert ok.mean() >= 0.9
    assert np.array_equal(out["result"][:rows][ok], res[ok])
    assert np.array_equal(out["iterations"][:rows][ok], it[ok])
    err = np.abs(out["relative_times"][:rows][ok] - x[ok])
    allowed = 1e-9 * np.abs(x[ok]) + 64.0 * drift[ok]
    print(f"  largest time difference {(err / np.abs(x[ok])).max():.2e} relative, "
          f"{(err / np.maximum(allowed, 1e-300)).max():.2f} of the allowance")
    assert (err <= allowed).all()


@pytest.mark.gpu
def test_nonlinear_mirror_runs_the_time_scaling_sequence():
    out = subprocess.run([build_binary()], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert " 0 failures" in out.stdout
