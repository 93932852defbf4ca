"""The rest of csrc/mtg_generic_kernel.cuh against exact references, and every host-pointer entry point against its
device-pointer call.

  1. exact references on the CPU (dyadic-integer arithmetic on the fp64 inputs), with self-tests on closed forms;
  2. setFreeConstraints (backsub_kernel, behind mtg_coeffs_from_constraints_batch_f64, every n_free == 0 solve and the
     time objective with d_free) at every even N, D in {1, 2, 3, 4, 7}, K in {1, 2, 5, 16, 50}, on the waypoint, the
     all-fixed and seeded random masks, and on bad segment times;
  3. evaluate (evaluate_kernel<N>, N = 1..12) on dyadic grids, where segment choice and local time are exact, and the
     sample-time contract t_s = fl(t_start + fl(s * dt)) on a grid where a fused multiply-add differs;
  4. evaluateRange (range_walk_kernel + range_eval_kernel<N>, N = 1..12) bit for bit against the reference-order
     oracle (compiled with -ffp-contract=off);
  5. the host-pointer entry points (pageable and pinned buffers) and refused host calls;
  6. the fused Nfabian entry into an output that is only 8-byte aligned (the pack fallback).

Error bounds are c * u * S with u = 2^-53 and S the same sum with every term replaced by its absolute value.
"""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle.gen_tables import tables as exact_tables
from test_gpu_parity import check_parity, global_rel_err
from test_large_k import _dyadic, _pinned, same_bits, solve
from test_masked_kernel import fixed_values, make_mask, segment_times, waypoint_mask
from test_resident_kernels import BAD_IDS, BAD_VALUES

U = 2.0 ** -53
ERR_BAD_ARG = -1  # MTG_ERR_BAD_ARG (include/mtg_b200.h)
NAN = float("nan")


# ---------------------------------------------------------------------------------------------------------------------
# 1. Exact references

def _scaled(m, e, den=1):
    """m * 2**e / den rounded once to fp64 (Python's int / int is correctly rounded)"""
    return (m << e) / den if e >= 0 else m / (den << -e)


_A1INV = {}


def a1inv_integers(N):
    """exact A(1)^-1 of oracle/gen_tables.py as (integer numerators [N][N], common denominator L)"""
    if N not in _A1INV:
        Ai = exact_tables(N, 0)[1]
        L = math.lcm(*(x.denominator for row in Ai for x in row))
        _A1INV[N] = ([[int(x * L) for x in row] for row in Ai], L)
    return _A1INV[N]


def backsub_bound(N):
    """Forward-error bound of back_substitute per coefficient, in units of u * S_j.  Coefficient j is
    T^-j * sum_s A1inv[j][s] * (T^(s mod h) * v_s): the rounded table entry (1 rounding), T^(s mod h) (<= h - 1), its
    product with v_s (1), the N-term fma chain (N), 1 / T and its j-th power (<= 2(N - 1)) and the final product (1)
    make at most 3.5 N roundings; 4N + 16 leaves room for the second-order terms."""
    return 4 * N + 16


def exact_backsub(N, T, v):
    """The N coefficients of the polynomial on [0, T] with derivative s at 0 equal to v[s] (s < h) and derivative s - h
    at T equal to v[s] (s >= h), over the rationals: c_j = T^-j sum_s A1inv[j][s] T^(s mod h) v_s, and the scale
    S_j = T^-j sum_s |A1inv[j][s]| T^(s mod h) |v_s|.  T > 0, v: fp64 -> (c [N], S [N]) rounded once to fp64."""
    h = N // 2
    num, L = a1inv_integers(N)
    tm, te = _dyadic(T)
    terms = []
    for s in range(N):
        vm, ve = _dyadic(v[s])
        p = s % h
        terms.append((tm ** p * vm, te * p + ve))
    e0 = min(e for _, e in terms)
    w = [m << (e - e0) for m, e in terms]
    c, S = np.empty(N), np.empty(N)
    for j in range(N):
        acc = sum(num[j][s] * w[s] for s in range(N))
        sc = sum(abs(num[j][s] * w[s]) for s in range(N))
        den = L * tm ** j
        c[j], S[j] = _scaled(acc, e0 - te * j, den), _scaled(sc, e0 - te * j, den)
    return c, S


def slot_values(prob, d_fixed, d_free):
    """v [B][K][D][N] with v[b][i][d][s] = d_all[b][d][slot_col[i*N+s]], d_all = [d_fixed | d_free]"""
    d_all = d_fixed if d_free is None else np.concatenate([d_fixed, d_free], axis=2)
    return d_all[:, :, prob.slot_col.reshape(prob.K, prob.N)].transpose(0, 2, 1, 3)


def exact_backsub_batch(prob, times, d_fixed, d_free):
    """exact_backsub of every (trajectory, segment, dimension) -> (coeffs, scale) [B][K][D][N]"""
    v = slot_values(prob, d_fixed, d_free)
    B, K, D, N = v.shape
    ref, scale = np.empty(v.shape), np.empty(v.shape)
    for b in range(B):
        for i in range(K):
            for d in range(D):
                ref[b, i, d], scale[b, i, d] = exact_backsub(N, float(times[b, i]), v[b, i, d])
    return ref, scale


def eval_bound(N):
    """Forward-error bound of the fused Horner evaluation in units of u * S: one rounding per B(k, j) * c_j product
    and one per fma step, <= 2N in all; 4N + 16 leaves room for second-order terms."""
    return 4 * N + 16


def exact_derivative(c, k, t):
    """p^(k)(t) of p(t) = sum_j c_j t^j over the rationals, with the scale sum_j |b_j c_j| |t|^(j-k), b_j = j!/(j-k)!
    c: fp64 [N], t: fp64 -> (value, scale) rounded once to fp64; (0, 0) for k >= N."""
    N = len(c)
    if k >= N:
        return 0.0, 0.0
    tm, te = _dyadic(t)
    if te > 0:
        tm, te = tm << te, 0
    sh = -te
    cm = [_dyadic(x) for x in c]
    e0 = min(cm[j][1] for j in range(k, N))
    acc = sacc = 0
    for j in range(N - 1, k - 1, -1):  # integer Horner on t * 2^sh, every term scaled by 2^(sh (N-1-k))
        m, e = cm[j]
        a = math.perm(j, k) * (m << (e - e0))
        wsh = sh * (N - 1 - j)
        acc = acc * tm + (a << wsh)
        sacc = sacc * abs(tm) + (abs(a) << wsh)
    ex = e0 - sh * (N - 1 - k)
    return _scaled(acc, ex), _scaled(sacc, ex)


def select_segment(times, t):
    """Segment index, local time and in-range flag of time t in Trajectory::evaluate's rules, in the kernel's fp64
    arithmetic: a time on a vertex belongs to the right segment, the total time to the last one, beyond it nothing,
    a negative time to segment 0."""
    K = len(times)
    start, i = 0.0, 0
    while i < K:
        if start + times[i] > t:
            break
        start += times[i]
        i += 1
    in_range = True
    if i == K:
        in_range = not (t > start)
        i = K - 1
        start -= times[i]
    return i, t - start, in_range


def exact_evaluate(times, coeffs, k, ts):
    """exact p^(k) at the sample times ts [S] for every trajectory: times [B][K], coeffs [B][K][D][N] ->
    (value, scale) [B][S][D]"""
    B, K, D, N = coeffs.shape
    val, scale = np.zeros((B, len(ts), D)), np.zeros((B, len(ts), D))
    for b in range(B):
        for s, t in enumerate(ts):
            i, tl, ok = select_segment([float(x) for x in times[b]], float(t))
            if ok:
                for d in range(D):
                    val[b, s, d], scale[b, s, d] = exact_derivative(coeffs[b, i, d], k, tl)
    return val, scale


def check_bound(got, ref, scale, c, label):
    err = np.abs(got - ref)
    bad = ~(err <= c * U * scale)
    assert not bad.any(), (f"{label}: {int(bad.sum())} values outside c*u*S; worst |got - exact| / (u S) = "
                           f"{np.max(np.where(scale > 0, err / (U * np.maximum(scale, 1e-300)), np.inf)):.3g} (c = {c})")


def test_exact_derivative_closed_forms():
    """c = t^r / r! has derivative r equal to r! * fl(1/r!) (within one ulp of 1) everywhere and derivative r + 1
    equal to 0; a Horner sum against Fraction arithmetic on random coefficients and times."""
    for N in range(1, 13):
        for r in range(N):
            c = np.zeros(N)
            c[r] = 1.0 / math.factorial(r)
            for t in (0.0, 0.3, -1.7, 2.0 ** -30, 13.0):
                v, s = exact_derivative(c, r, t)
                assert v == float(math.factorial(r) * Fraction(c[r])) and abs(v - 1.0) <= 2 * U and s == v
                assert exact_derivative(c, r + 1, t) == (0.0, 0.0)
    rng = np.random.RandomState(5)
    for trial in range(40):
        N = int(rng.randint(1, 13))
        k = int(rng.randint(0, N + 2))
        c = rng.uniform(-1, 1, N) * 10.0 ** rng.uniform(-3, 3, N)
        t = float(rng.uniform(-3, 5))
        want = sum((Fraction(math.perm(j, k)) * Fraction(c[j]) * Fraction(t) ** (j - k) for j in range(k, N)),
                   Fraction(0))
        v, s = exact_derivative(c, k, t)
        assert v == float(want) and s >= abs(v), (trial, N, k)


def test_exact_backsub_closed_forms(oracle):
    """A single segment whose end derivatives are those of a known polynomial (small integer coefficients, dyadic
    T, so every derivative value is exact in fp64) gives that polynomial back exactly; on random data the exact
    coefficients agree with the oracle's fp64 A(T)^-1 (reference invertMappingMatrix) to rounding."""
    rng = np.random.RandomState(6)
    for N in (2, 4, 6, 8, 10, 12):
        h = N // 2
        for T in (1.5, 0.25, 3.0):
            q = rng.randint(-8, 9, size=N).astype(np.float64)
            v = np.empty(N)
            for s in range(h):
                v[s] = math.factorial(s) * q[s]
                at_t = sum(Fraction(math.perm(j, s)) * Fraction(q[j]) * Fraction(T) ** (j - s) for j in range(s, N))
                assert at_t == Fraction(float(at_t))  # exact in fp64
                v[h + s] = float(at_t)
            c, S = exact_backsub(N, T, v)
            assert np.array_equal(c, q), (N, T, c, q)
            assert (S >= np.abs(c)).all()
        T = float(np.exp(rng.uniform(np.log(0.05), np.log(20.0))))
        v = rng.uniform(-2, 2, N)
        c, S = exact_backsub(N, T, v)
        fp = oracle.inverse_mapping_matrix(N, T) @ v
        assert (np.abs(fp - c) <= 1e-8 * S).all(), (N, T)


def contract_grid():
    """A non-dyadic (t_start, dt) and a sample index s at which fma(s, dt, t_start) -- what a contracted
    t_start + s * dt gives -- falls strictly below the twice-rounded fl(t_start + fl(s * dt)), searched with Fraction.
    -> (t_start, dt, s, twice-rounded time, fma time)"""
    for t_start, dt in ((0.1, 0.1), (0.3, 0.07), (1.1, 0.013)):
        for s in range(1, 2000):
            tr = t_start + s * dt
            tf = float(Fraction(s) * Fraction(dt) + Fraction(t_start))
            if tf < tr:
                return t_start, dt, s, tr, tf
    return None


def test_contract_grid_exists():
    g = contract_grid()
    assert g is not None, "no grid where the fused and the twice-rounded sample time differ"
    t_start, dt, s, tr, tf = g
    assert Fraction(t_start).denominator > 2 ** 20 and Fraction(dt).denominator > 2 ** 20  # not dyadic grids
    assert tf < tr and tr == t_start + s * dt


# ---------------------------------------------------------------------------------------------------------------------
# 2. setFreeConstraints / back-substitution

BACKSUB_NR = [(2, 0), (4, 1), (6, 2), (8, 3), (10, 4), (12, 5)]
BACKSUB_SIZES = [(1, 1), (2, 2), (5, 3), (16, 4), (50, 7)]  # (K, D)
MASK_KINDS = ["waypoint", "all_fixed", "random"]


def backsub_mask(kind, N, r, K, rng):
    if kind == "waypoint":
        return waypoint_mask(N, K)
    if kind == "all_fixed":
        return np.ones((K + 1, N // 2), dtype=np.uint8)
    mask = make_mask("random", N, r, K, rng)
    if not mask.any():  # at least one fixed constraint: the entry points take a non-null d_fixed
        mask[0, 0] = 1
    return mask


def coeffs_from_constraints(solver, prob, t_d, f_d, d_free, offset=0):
    """coeffs_from_constraints into a NaN-filled output starting `offset` doubles into its allocation -> numpy"""
    import torch
    B = t_d.shape[0]
    n = B * prob.K * prob.D * prob.N
    big = torch.full((n + offset,), NAN, dtype=torch.float64, device="cuda")
    out = big[offset:].view(B, prob.K, prob.D, prob.N)
    assert out.data_ptr() % 16 == 8 * offset
    solver.coeffs_from_constraints(prob, t_d, f_d, d_free, coeffs=out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", MASK_KINDS)
@pytest.mark.parametrize("N,r", BACKSUB_NR, ids=[f"N{n}r{r}" for n, r in BACKSUB_NR])
def test_coeffs_from_constraints_vs_exact(solver, oracle, N, r, kind):
    """For each (K, D): (a) coefficients from arbitrary d_free (not the optimum, which would hide errors in the free
    columns) within backsub_bound of the exact back-substitution, log-uniform times over [0.05, 20] s and non-zero
    end derivatives; (b) an 8-byte aligned output gives the same bits; (c) solve_linear's own d_free fed back
    reproduces solve_linear's coefficients under check_parity's rule, with solve_linear in the oracle's place."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(1000 * N + 10 * r + MASK_KINDS.index(kind))
    for K, D in BACKSUB_SIZES:
        B = min(64, max(2, 400 // (K * D)))
        mask = backsub_mask(kind, N, r, K, rng)
        prob = m.Problem(N, r, K, D, fixed_mask=mask)
        label = f"N={N} r={r} K={K} D={D} B={B} {kind}"
        assert (prob.n_free == 0) == (kind == "all_fixed" or kind == "waypoint" and (N == 2 or K == 1)), label
        if kind == "all_fixed":
            assert prob.kernel == m.KERNEL_NOFREE, label
        _, dfix = fixed_values(mask, B, D, rng)
        times = segment_times(B, K, "mixed", rng)
        dfree = rng.uniform(-2, 2, size=(B, D, prob.n_free)) if prob.n_free else None
        t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
        fr_d = torch.from_numpy(dfree).cuda() if prob.n_free else None

        out = coeffs_from_constraints(solver, prob, t_d, f_d, fr_d)
        ref, scale = exact_backsub_batch(prob, times, dfix, dfree)
        check_bound(out, ref, scale, backsub_bound(N), label)
        assert same_bits(coeffs_from_constraints(solver, prob, t_d, f_d, fr_d, offset=1), out), \
            f"{label}: 8-byte aligned output differs"

        if kind == "random":  # see RANDOM_MASK_ROUND_TRIP_TIMES
            times = segment_times(B, K, RANDOM_MASK_ROUND_TRIP_TIMES, rng)
            t_d = torch.from_numpy(times).cuda()
        sl, sl_free, status = solve(solver, prob, t_d, f_d)
        assert (status == 0).all() and np.isfinite(sl).all(), label
        own = torch.from_numpy(np.ascontiguousarray(sl_free[:, :, :prob.n_free])).cuda() if prob.n_free else None
        again = coeffs_from_constraints(solver, prob, t_d, f_d, own)
        if prob.n_free == 0:
            assert same_bits(again, sl), f"{label}: solve_linear without free constraints is not backsub_kernel"
        exact = oracle.exact_solve_batch(N, r, times, dfix, mask=mask)
        check_parity(again, sl, exact, label + " (d_free of solve_linear)")


# Random masks round-trip on segment times uniform in [0.5, 5] s (test_masked_kernel.py's fixture), not on the log-uniform
# [0.05, 20] s of the exact check.  There, at K = 1, the d_free that solve_linear (the masked kernel) returns is far less
# accurate than its coefficients, and back-substituting it loses what check_parity allows: 2.3e-10 from exact where
# solve_linear's coefficients are 9.2e-11 (N = 6), 1.9e-6 where they are 3.2e-8 (N = 8), 1.1e-4 where they are 3.5e-7
# (N = 12); and at N = 10, K = 16, D = 4 one row is not even SPD in fp64 (STATUS_NOT_SPD).  The back-substitution itself
# is held to its exact bound on those times above; this is the conditioning of the returned d_free.
RANDOM_MASK_ROUND_TRIP_TIMES = "uniform"


BAD_B = 70  # warps of 32, 32 and 6 trajectories
BAD_ROWS = [0, 5, 31, 32, 33, 50, 64, 69]


@pytest.mark.gpu
@pytest.mark.parametrize("value", BAD_VALUES, ids=BAD_IDS)
@pytest.mark.parametrize("N", [2, 4, 6, 8, 10, 12])
def test_bad_segment_time_all_fixed(solver, N, value):
    """All-fixed problems solve through backsub_kernel: a bad segment time in segment 0, in segment K-1 or in every
    segment sets STATUS_BAD_TIME in exactly those rows; every other row keeps the bits of the repaired batch, in
    solve_linear and in coeffs_from_constraints."""
    import torch
    import mav_trajectory_generation_b200 as m
    K, D = 5, 3
    rng = np.random.RandomState(77 + N)
    mask = np.ones((K + 1, N // 2), dtype=np.uint8)
    prob = m.Problem(N, N // 2 - 1, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_NOFREE
    _, dfix = fixed_values(mask, BAD_B, D, rng)
    times = segment_times(BAD_B, K, "mixed", rng)
    bad_times = times.copy()
    for n, b in enumerate(BAD_ROWS):
        bad_times[b, [[0], [K - 1], list(range(K))][n % 3]] = value
    f_d = torch.from_numpy(dfix).cuda()
    clean, _, clean_status = solve(solver, prob, torch.from_numpy(times).cuda(), f_d)
    out, _, status = solve(solver, prob, torch.from_numpy(bad_times).cuda(), f_d)
    assert (clean_status == 0).all()
    good = np.setdiff1d(np.arange(BAD_B), BAD_ROWS)
    assert (status[BAD_ROWS] == m.STATUS_BAD_TIME).all(), status[BAD_ROWS]
    assert (status[good] == 0).all()
    assert same_bits(out[good], clean[good])
    again = coeffs_from_constraints(solver, prob, torch.from_numpy(bad_times).cuda(), f_d, None)
    assert same_bits(again[good], clean[good])


@pytest.mark.gpu
@pytest.mark.parametrize("N,r", [(6, 2), (12, 5)])
def test_time_objective_with_free_equals_back_substitution(solver, N, r):
    """mtg_time_objective_batch_f64 with d_free on a non-waypoint mask writes the coefficients of
    coeffs_from_constraints, bit for bit."""
    import torch
    import mav_trajectory_generation_b200 as m
    K, D, B = 5, 3, 40
    rng = np.random.RandomState(90 + N)
    mask = make_mask("random", N, r, K, rng)
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.n_free > 0 and prob.kernel != m.KERNEL_WAYPOINT
    _, dfix = fixed_values(mask, B, D, rng)
    times = segment_times(B, K, "mixed", rng)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    fr_d = torch.from_numpy(rng.uniform(-2, 2, size=(B, D, prob.n_free))).cuda()
    _, _, coeffs, status = solver.time_objective(prob, t_d, f_d, fr_d, constraints=((1, 2.0),))
    want = coeffs_from_constraints(solver, prob, t_d, f_d, fr_d)
    assert (status.cpu().numpy() == 0).all()
    assert same_bits(coeffs.cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------------------------
# 3. evaluate

def evaluate(solver, t_d, c_d, der, t_start, dt, S):
    """solver.evaluate into a NaN-filled output -> numpy [B][S][D]"""
    import torch
    B, K, D, N = c_d.shape
    out = torch.full((B, S, D), NAN, dtype=torch.float64, device="cuda")
    solver.evaluate(t_d, c_d, der, t_start, dt, S, out=out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def dyadic_fixture(rng, B, K, D, N):
    """segment times that are multiples of 1/8 in [0.5, 2] s (so every vertex and every total time lies on the grid
    t_start = -3/8, dt = 1/8), random discontinuous coefficients -> (times, coeffs, t_start, dt, grid)"""
    times = rng.randint(4, 17, size=(B, K)) / 8.0
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    t_start, dt = -0.375, 0.125
    S = int((times.sum(axis=1).max() + 0.5 - t_start) / dt) + 1
    return times, coeffs, t_start, dt, t_start + np.arange(S) * dt


@pytest.mark.gpu
@pytest.mark.parametrize("N", range(1, 13))
def test_evaluate_every_order_dyadic_grid(solver, N):
    """Every derivative 0..N+1 at D in {1, 3, 4, 13} on a dyadic grid (every sum exact): every value within
    eval_bound of the exact value; orders >= N exactly zero; a sample on a vertex takes the right-hand segment (its
    position is exactly that segment's c_0); t = total time belongs to the last segment; beyond the end zeros;
    negative times extrapolate segment 0."""
    import torch
    rng = np.random.RandomState(700 + N)
    K, B = 3, 2
    for D in (1, 3, 4, 13):
        times, coeffs, t_start, dt, grid = dyadic_fixture(rng, B, K, D, N)
        S = len(grid)
        t_d, c_d = torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()
        for der in range(N + 2):
            got = evaluate(solver, t_d, c_d, der, t_start, dt, S)
            ref, scale = exact_evaluate(times, coeffs, der, grid)
            check_bound(got, ref, scale, eval_bound(N), f"evaluate N={N} D={D} derivative={der}")
            if der >= N:
                assert not got.any() and not np.signbit(got).any()
        # the fixture reaches every convention; the bound check above holds the values there
        got = evaluate(solver, t_d, c_d, 0, t_start, dt, S)
        assert (grid < 0).sum() == 3  # negative times: segment 0 extrapolated
        for b in range(B):
            ends = np.cumsum(times[b])
            for i in range(K - 1):  # interior vertex -> exactly the right segment's c_0 (local time 0)
                s = int(np.flatnonzero(grid == ends[i])[0])
                assert np.array_equal(got[b, s], coeffs[b, i + 1, :, 0]), (N, D, b, i)
            s_end = int(np.flatnonzero(grid == ends[-1])[0])  # the total time: the end of the last segment
            assert select_segment(list(times[b]), grid[s_end]) == (K - 1, times[b, -1], True)
            assert s_end + 1 < S and (got[b, s_end + 1:] == 0).all()  # beyond the end


@pytest.mark.gpu
@pytest.mark.parametrize("N", [5, 12])
def test_evaluate_wide_dimension_and_limit(solver, N):
    """D = 200: the host sizes the output tile to 32 threads and 51 200 bytes of dynamic shared memory (above the
    48 KB default); every value within the bound.  D = 641 needs more than the tile allows: MTG_ERR_BAD_ARG before
    any launch."""
    import torch
    rng = np.random.RandomState(800 + N)
    D, K, B = 200, 3, 2
    times, coeffs, t_start, dt, grid = dyadic_fixture(rng, B, K, D, N)
    grid = grid[::3]
    t_d, c_d = torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()
    for der in (0, 3):
        got = evaluate(solver, t_d, c_d, der, t_start, 3 * dt, len(grid))
        ref, scale = exact_evaluate(times, coeffs, der, grid)
        check_bound(got, ref, scale, eval_bound(N), f"evaluate N={N} D={D} derivative={der}")
    D = 641
    c_d = torch.zeros((1, 1, D, N), dtype=torch.float64, device="cuda")
    t_d = torch.ones((1, 1), dtype=torch.float64, device="cuda")
    out = torch.full((1, 2, D), NAN, dtype=torch.float64, device="cuda")
    launches = solver.launch_count
    rc = solver.lib.mtg_evaluate_batch_f64(solver.h, N, 1, D, 1, t_d.data_ptr(), c_d.data_ptr(), 0, 0.0, 0.5, 2,
                                           out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == ERR_BAD_ARG and solver.launch_count == launches
    assert torch.isnan(out).all()


@pytest.mark.gpu
def test_evaluate_grid_stride_wraps(solver):
    """B * S above sm_count * 32 * 256 (the grid's cap), with a ragged last tile: the tile loop wraps.  The batch
    repeats P base trajectories, so every row must equal its base row bit for bit; the base rows are checked against
    the exact values."""
    import torch
    N, K, D, P, S = 7, 2, 1, 29, 97
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = sm * 32 * 256 // S + 300
    while (B * S) % 256 == 0:
        B += 1
    assert B * S > sm * 32 * 256
    rng = np.random.RandomState(9)
    base_t = rng.randint(4, 17, size=(P, K)) / 8.0
    base_c = rng.uniform(-1, 1, size=(P, K, D, N))
    idx = np.arange(B) % P
    t_d = torch.from_numpy(base_t[idx]).cuda()
    c_d = torch.from_numpy(np.ascontiguousarray(base_c[idx])).cuda()
    t_start, dt = 0.0, 1.0 / 32
    got = evaluate(solver, t_d, c_d, 1, t_start, dt, S)
    ref, scale = exact_evaluate(base_t, base_c, 1, t_start + np.arange(S) * dt)
    check_bound(got[:P], ref, scale, eval_bound(N), "evaluate wrap base rows")
    assert same_bits(got, got[idx]), "a row differs from its base row"


@pytest.mark.gpu
def test_evaluate_sample_time_is_twice_rounded(solver):
    """On a non-dyadic grid where fma(s, dt, t_start) < fl(t_start + fl(s * dt)), segment 0 ends exactly at the
    twice-rounded time of sample s: that sample belongs to segment 1 (local time 0, position exactly c_0 of segment 1),
    as the documented grid and every host-side caller put it.  Every other sample is within the bound of the exact
    value at the twice-rounded time."""
    import torch
    g = contract_grid()
    assert g is not None
    t_start, dt, s, tr, tf = g
    N, K, D, B = 6, 2, 3, 4
    rng = np.random.RandomState(11)
    times = np.empty((B, K))
    times[:, 0] = tr
    times[:, 1] = rng.uniform(0.5, 1.5, size=B)
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    S = s + 20
    grid = np.array([t_start + q * dt for q in range(S)])
    assert grid[s] == tr and select_segment(list(times[0]), tf)[0] == 0 and select_segment(list(times[0]), tr)[0] == 1
    t_d, c_d = torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()
    got = evaluate(solver, t_d, c_d, 0, t_start, dt, S)
    assert np.array_equal(got[:, s], coeffs[:, 1, :, 0]), \
        f"sample {s} (t = {tr!r}) taken from segment 0, as at the fused time {tf!r}"
    for der in (0, 2):
        got = evaluate(solver, t_d, c_d, der, t_start, dt, S)
        val, scale = np.zeros((B, S, D)), np.zeros((B, S, D))
        for b in range(B):
            for q in range(S):
                i, tl, ok = select_segment(list(times[b]), grid[q])
                for d in range(D):
                    if ok:
                        val[b, q, d], scale[b, q, d] = exact_derivative(coeffs[b, i, d], der, tl)
        check_bound(got, val, scale, eval_bound(N), f"evaluate contract grid derivative={der}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. evaluateRange

def evaluate_range(solver, t_d, c_d, t_start, t_end, dt, derivs, max_samples, want_times):
    """mtg_evaluate_range_batch_f64 into NaN-filled outputs (sampling_times NULL unless want_times)
    -> (rc, out [B][max_samples][n_derivs][D], n_samples [B], sampling_times or None) as numpy"""
    import torch
    B, K, D, N = c_d.shape
    arr = (C.c_int32 * len(derivs))(*[int(x) for x in derivs])
    out = torch.full((B, max_samples, len(derivs), D), NAN, dtype=torch.float64, device="cuda")
    n = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    st = torch.full((B, max_samples), NAN, dtype=torch.float64, device="cuda") if want_times else None
    rc = solver.lib.mtg_evaluate_range_batch_f64(
        solver.h, N, K, D, B, t_d.data_ptr(), c_d.data_ptr(), float(t_start), float(t_end), float(dt), len(derivs),
        arr, int(max_samples), out.data_ptr() if max_samples else None, n.data_ptr(),
        st.data_ptr() if want_times else None, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, out.cpu().numpy(), n.cpu().numpy(), (st.cpu().numpy() if want_times else None)


def check_range(oracle, times, coeffs, case, out, n, st, label):
    """every row bit for bit against oracle.evaluate_range: count, stored samples, zero rows beyond the count,
    sampling times"""
    t_start, t_end, dt, derivs, S = case
    for b in range(times.shape[0]):
        for q, der in enumerate(derivs):
            n_ref, o_ref, st_ref = oracle.evaluate_range(times[b], coeffs[b], t_start, t_end, dt, der, S)
            assert n[b] == n_ref, (label, b, der, n[b], n_ref)
            k = min(max(n_ref, 0), S)
            assert same_bits(out[b, :k, q], o_ref[:k]), (label, b, der)
            assert (out[b, k:].view(np.uint64) == 0).all(), (label, b)
            if st is not None:
                assert same_bits(st[b, :k], st_ref[:k]), (label, b)


def walk_total(times_row):
    """the walk's running sum over all segments (left to right, fp64)"""
    acc = 0.0
    for x in times_row:
        acc += float(x)
    return acc


@pytest.mark.gpu
@pytest.mark.parametrize("N", range(1, 13))
def test_evaluate_range_every_order_bitwise(solver, oracle, N):
    """evaluateRange at every compiled order, bit for bit against the oracle, B = 70 (warps of 32, 32, 6), with
    derivative lists of 1 and 8 entries (orders >= N included), truncated buffers (n_samples still reports n),
    max_samples = 0, sampling_times NULL and not, and the edges: t_start on a vertex, at exactly the total time
    (n = 0), beyond it (n = -1), negative, t_end < t_start, and samples exactly on segment ends."""
    import torch
    D = (1, 3, 4, 13)[N % 4]
    K, B = 4, 70
    rng = np.random.RandomState(900 + N)
    d1 = [N // 2]
    d8 = [0, 1, 2, 3, 4, max(N - 1, 0), N, N + 1]
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    c_d = torch.from_numpy(coeffs).cuda()
    # per-row times, the first segment 0.75 s in every row (a common vertex)
    times = rng.uniform(0.3, 1.5, size=(B, K))
    times[:, 0] = 0.75
    full = lambda dt: int(times.sum(axis=1).max() / dt) + K + 8  # noqa: E731
    cases = [  # t_start, t_end, dt, derivs, max_samples, sampling times
        (0.0, float(times.sum(axis=1).min()), 0.05, d8, full(0.05), True),
        (0.75, 4.0, 0.07, d1, full(0.07), False),  # t_start on a vertex
        (-0.3, 2.0, 0.11, d8, 5, True),            # negative start; the buffer holds 5 of ~20 samples
        (1.3, 1e9, 0.09, d1, 0, False),            # counts only
        (2.0, 1.9, 0.01, d8, full(0.01), True),    # t_end < t_start: samples from the segment start up to t_end
        (3.0, 1e9, 0.1, d1, full(0.1), True),      # beyond the end of some rows (n = -1) but not others
    ]
    t_d = torch.from_numpy(times).cuda()
    for t0, t1, dt, derivs, S, want in cases:
        rc, out, n, st = evaluate_range(solver, t_d, c_d, t0, t1, dt, derivs, S, want)
        label = f"range N={N} D={D} t_start={t0} t_end={t1} dt={dt} {len(derivs)} derivs S={S}"
        assert rc == 0, label
        check_range(oracle, times, coeffs, (t0, t1, dt, derivs, S), out, n, st, label)
        if S == 5:
            assert (n > S).all(), label
        elif S > 0:
            assert (n <= S).all(), label
    assert (n == -1).any() and (n > 0).any()
    # one set of dyadic times shared by every row: samples land exactly on segment ends, and the total time is known
    base = rng.randint(4, 17, size=K) / 8.0
    times = np.ascontiguousarray(np.tile(base, (B, 1)))
    total = walk_total(base)
    t_d = torch.from_numpy(times).cuda()
    cases = [(0.0, 1e9, 1.0 / 16, d8, full(1.0 / 16), True), (float(base[0]), total, 0.125, d1, full(0.125), False),
             (total, total + 1.0, 0.1, d8, 8, True), (total + 0.25, total + 1.0, 0.1, d1, 8, False),
             (-0.5, 1.0, 0.125, d8, full(0.125), True)]
    for t0, t1, dt, derivs, S, want in cases:
        rc, out, n, st = evaluate_range(solver, t_d, c_d, t0, t1, dt, derivs, S, want)
        label = f"range N={N} D={D} dyadic t_start={t0} t_end={t1} dt={dt} {len(derivs)} derivs"
        assert rc == 0, label
        check_range(oracle, times, coeffs, (t0, t1, dt, derivs, S), out, n, st, label)
        if t0 == total:
            assert (n == 0).all(), label
        if t0 > total:
            assert (n == -1).all(), label


@pytest.mark.gpu
def test_evaluate_range_walk_grid_stride(solver, oracle):
    """B above sm_count * 16 * 128 (the walk's grid cap) with K = 1: the walk runs a second grid-stride round.  The
    batch repeats P base trajectories; every row must equal the oracle on its base row, bit for bit."""
    import torch
    N, K, D, P, S = 3, 1, 1, 61, 3
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = sm * 16 * 128 + 4099
    rng = np.random.RandomState(12)
    base_t = rng.uniform(1.31, 1.5, size=(P, K))  # samples at 0.1, 0.5, 0.9 (and 1.3): every row fills its S = 3
    base_c = rng.uniform(-1, 1, size=(P, K, D, N))
    idx = np.arange(B) % P
    t_d = torch.from_numpy(base_t[idx]).cuda()
    c_d = torch.from_numpy(np.ascontiguousarray(base_c[idx])).cuda()
    t0, t1, dt = 0.1, 1e9, 0.4
    rc, out, n, st = evaluate_range(solver, t_d, c_d, t0, t1, dt, [0], S, True)
    assert rc == 0
    ref_n = np.empty(P, dtype=np.int64)
    ref_o = np.zeros((P, S, 1, D))
    ref_st = np.zeros((P, S))
    for p in range(P):
        ref_n[p], ref_o[p, :, 0], ref_st[p] = oracle.evaluate_range(base_t[p], base_c[p], t0, t1, dt, 0, S)
    assert (ref_n >= S).all()
    assert np.array_equal(n, ref_n[idx])
    assert same_bits(out, ref_o[idx]) and same_bits(st, ref_st[idx])


@pytest.mark.gpu
def test_evaluate_range_tile_limit(solver):
    """8 derivative orders of 81 dimensions do not fit the output tile: MTG_ERR_BAD_ARG."""
    import torch
    N, K, D = 2, 1, 81
    t_d = torch.ones((2, K), dtype=torch.float64, device="cuda")
    c_d = torch.zeros((2, K, D, N), dtype=torch.float64, device="cuda")
    rc, out, _, _ = evaluate_range(solver, t_d, c_d, 0.0, 1.0, 0.5, list(range(8)), 2, False)
    assert rc == ERR_BAD_ARG
    assert np.isnan(out).all()
    assert b"tile" in solver.lib.mtg_last_error(solver.h)


# ---------------------------------------------------------------------------------------------------------------------
# 5. Host-pointer entry points

def _host_in(a, kind):
    return _pinned(a) if kind == "pinned" else np.ascontiguousarray(a)


def _host_out(shape, kind, dtype=np.float64, fill=NAN):
    import torch
    if kind == "pinned":
        tdt = torch.float64 if dtype == np.float64 else torch.int32
        return torch.full(shape, fill, dtype=tdt).pin_memory()
    return np.full(shape, fill, dtype=dtype)


def _np(a):
    return a.numpy() if hasattr(a, "numpy") else a


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pageable", "pinned"])
def test_host_entry_points_equal_device_calls(solver, oracle, kind):
    """compute_cost_host, cost_gradient_mellinger_host and evaluate_range_host (sampling times NULL and not) at a
    ragged B equal their device-pointer calls bit for bit."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(13)
    # computeCost
    N, r, K, D, B = 10, 4, 5, 3, 1001
    prob = m.Problem(N, r, K, D)
    times = segment_times(B, K, "mixed", rng)
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    dev = solver.compute_cost(prob, torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()).cpu().numpy()
    host = _host_out((B,), kind)
    solver.compute_cost_host(prob, _host_in(times, kind), _host_in(coeffs, kind), host)
    assert same_bits(_np(host), dev)
    # getCostAndGradientMellinger
    K, B = 5, 37
    prob = m.Problem(N, r, K, D)
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=14000)
    dfix = oracle.waypoint_d_fixed(N, pos)
    cost, grad = solver.cost_gradient_mellinger(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda())
    torch.cuda.synchronize()
    h_cost, h_grad = _host_out((B,), kind), _host_out((B, K), kind)
    solver.cost_gradient_mellinger_host(prob, _host_in(times, kind), _host_in(dfix, kind), h_cost, h_grad)
    assert same_bits(_np(h_cost), cost.cpu().numpy()) and same_bits(_np(h_grad), grad.cpu().numpy())
    # evaluateRange
    N, K, D, B, S = 8, 4, 3, 101, 40
    times = rng.uniform(0.3, 1.5, size=(B, K))
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    derivs = (0, 2, 5)
    t_d, c_d = torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()
    rc, out, n, st = evaluate_range(solver, t_d, c_d, 0.4, 3.5, 0.09, derivs, S, True)
    assert rc == 0
    for want_times in (True, False):
        h_out, h_n = _host_out((B, S, len(derivs), D), kind), _host_out((B,), kind, np.int32, -7)
        h_st = _host_out((B, S), kind) if want_times else None
        solver.evaluate_range_host(_host_in(times, kind), _host_in(coeffs, kind), 0.4, 3.5, 0.09, derivs, h_out, h_n,
                                   sampling_times=h_st)
        assert same_bits(_np(h_out), out) and same_bits(_np(h_n), n)
        if want_times:
            k = min(int(n.min()), S)
            assert same_bits(_np(h_st)[:, :k], st[:, :k])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pageable", "pinned"])
@pytest.mark.parametrize("with_free", [True, False], ids=["free", "all_fixed"])
def test_coeffs_from_constraints_host_pipeline(solver, kind, with_free):
    """coeffs_from_constraints_host at B = 9001 (three pipeline chunks on three streams) equals the device call bit for
    bit, with free constraints and without (no d_free is needed or read); a problem with free constraints and no
    d_free is refused."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 8, 3, 5, 3, 9001
    rng = np.random.RandomState(15 + with_free)
    mask = waypoint_mask(N, K) if with_free else np.ones((K + 1, N // 2), dtype=np.uint8)
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert (prob.n_free > 0) == with_free
    _, dfix = fixed_values(mask, B, D, rng)
    times = segment_times(B, K, "mixed", rng)
    dfree = rng.uniform(-2, 2, size=(B, D, prob.n_free)) if with_free else None
    dev = coeffs_from_constraints(solver, prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda(),
                                  torch.from_numpy(dfree).cuda() if with_free else None)
    host = _host_out((B, K, D, N), kind)
    solver.coeffs_from_constraints_host(prob, _host_in(times, kind), _host_in(dfix, kind),
                                        _host_in(dfree, kind) if with_free else None, host)
    assert same_bits(_np(host), dev)
    if with_free:
        with pytest.raises(RuntimeError, match="d_free is required"):
            solver.coeffs_from_constraints_host(prob, _host_in(times, kind), _host_in(dfix, kind), None, host)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pageable", "pinned"])
def test_refused_host_calls(solver, kind):
    """A host call the device entry refuses (computeCost with K * D too large for shared memory; evaluateRange with
    n_derivs * D too large for the output tile) returns the error, launches no cost kernel, and leaves the handle's
    pipeline usable: the next host calls equal their device calls bit for bit."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(16)
    N, r, K, D, B = 2, 0, 10000, 3, 2
    prob = m.Problem(N, r, K, D)
    times = rng.uniform(0.5, 1.5, size=(B, K))
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    cost = _host_out((B,), kind)
    launches = solver.launch_count
    with pytest.raises(RuntimeError, match="K \\* D too large"):
        solver.compute_cost_host(prob, _host_in(times, kind), _host_in(coeffs, kind), cost)
    assert solver.launch_count == launches and np.isnan(_np(cost)).all()
    N, K, D, B, S = 2, 1, 81, 3, 2
    out, n = _host_out((B, S, 8, D), kind), _host_out((B,), kind, np.int32, -7)
    with pytest.raises(RuntimeError, match="tile"):
        solver.evaluate_range_host(_host_in(np.ones((B, K)), kind), _host_in(np.zeros((B, K, D, N)), kind), 0.0, 1.0,
                                   0.5, range(8), out, n)
    assert np.isnan(_np(out)).all()
    N, r, K, D, B = 6, 2, 4, 2, 33
    prob = m.Problem(N, r, K, D)
    times = segment_times(B, K, "mixed", rng)
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N))
    dev = solver.compute_cost(prob, torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda()).cpu().numpy()
    cost = _host_out((B,), kind)
    solver.compute_cost_host(prob, _host_in(times, kind), _host_in(coeffs, kind), cost)
    assert same_bits(_np(cost), dev)


# ---------------------------------------------------------------------------------------------------------------------
# 6. The fused Nfabian entry into an 8-byte aligned output

@pytest.mark.gpu
def test_fused_nfabian_unaligned_output(solver, oracle):
    """plan_waypoint declines a coefficient output that is not 16-byte aligned, so the fused entry packs and solves
    through the fallback.  seg_times_out and status equal the aligned (fused kernel) call bit for bit; the
    coefficients equal solve_linear into an 8-byte aligned output (the banded generic kernel) on those times and the
    packed constraints bit for bit, and are within 1e-10 of the binary128 solve, as the fused kernel's are.  The two
    kernels round differently, so the aligned and unaligned coefficients agree to rounding only."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 50
    pos, _ = oracle.make_waypoint_batch(K, D, B, base_seed=17000)
    p_d = torch.from_numpy(pos).cuda()

    def run(offset):
        big = torch.full((B * K * D * N + offset,), NAN, dtype=torch.float64, device="cuda")
        coeffs = big[offset:].view(B, K, D, N)
        assert coeffs.data_ptr() % 16 == 8 * offset
        t_out = torch.full((B, K), NAN, dtype=torch.float64, device="cuda")
        status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        solver.solve_waypoints_nfabian(N, r, p_d, 3.0, 5.0, 6.5, coeffs=coeffs, seg_times_out=t_out, status=status)
        torch.cuda.synchronize()
        return coeffs.cpu().numpy(), t_out.cpu().numpy(), status.cpu().numpy()

    aligned, odd = run(0), run(1)
    assert (aligned[2] == 0).all() and np.isfinite(aligned[0]).all()
    assert same_bits(odd[1], aligned[1]), "8-byte aligned output: seg_times_out differ"
    assert same_bits(odd[2], aligned[2]), "8-byte aligned output: status differs"
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    big = torch.full((B * K * D * N + 1,), NAN, dtype=torch.float64, device="cuda")
    banded = big[1:].view(B, K, D, N)
    solver.solve_linear(prob, torch.from_numpy(odd[1]).cuda(), torch.from_numpy(dfix).cuda(), coeffs=banded)
    torch.cuda.synchronize()
    assert same_bits(odd[0], banded.cpu().numpy()), "fallback differs from solve_linear on its own inputs"
    exact = oracle.exact_solve_batch(N, r, odd[1], dfix)
    e_odd, e_al = global_rel_err(odd[0], exact), global_rel_err(aligned[0], exact)
    print(f"fused unaligned: vs exact {e_odd.max():.2e} (aligned {e_al.max():.2e}), "
          f"vs aligned {global_rel_err(odd[0], aligned[0]).max():.2e}")
    assert e_odd.max() <= 1e-10 and e_al.max() <= 1e-10
