"""The masked block kernel K4 (masked_block_kernel<N, DG>, csrc/mtg_masked_block_kernel.cuh) against binary128.

K4 is the default for every constraint mask that is not the waypoint topology, and for the waypoint topology at every
(N, r, D) outside kWaypointKernels.  This file runs it

  1. on masks that are well posed by construction (CPU: the mask generator, the binary128 checker on those masks and
     the routing of every GPU case);
  2. at every compiled (N, dimension group) and every H(1;r) table, next to the banded generic kernel;
  3. on dimension groups (D > 4), large K, the benchmark's mask and many tiles per warp;
  4. on bad and infinite segment times (status bits).

Every GPU case also runs the banded generic kernel (OPT_GENERIC_VARIANT = 1), the second, independent implementation
of the same solve, under the same rules.
"""
import numpy as np
import pytest

from test_gpu_parity import check_parity, global_rel_err
from test_large_k import WAYPOINT_SHAPES, rel_err_free, same_bits, solve

FAMILIES = ("random", "free_position", "bench", "free_end", "free_vertex", "fixed_vertex", "one_free", "waypoint")


# ---------------------------------------------------------------------------------------------------------------------
# 1. Masks that are well posed by construction

def well_posed(mask, r):
    """The cost integral((p^(r))^2) vanishes over all slots exactly on the global polynomials of degree < r (every
    vertex shares its h slots between its two segments and r <= h - 1), so R_pp is SPD when no nonzero such polynomial
    vanishes on every fixed (vertex, derivative).  Sufficient: vertex 0 fixes derivatives 0..r-1 (Taylor), positions
    are fixed at >= r vertices (Lagrange), or r = 0."""
    return r == 0 or bool(mask[0, :r].all()) or int(mask[:, 0].sum()) >= r


def waypoint_mask(N, K):
    """createRandomVertices: positions everywhere, both ends fully fixed"""
    mask = np.zeros((K + 1, N // 2), dtype=np.uint8)
    mask[:, 0] = 1
    mask[0, :] = 1
    mask[-1, :] = 1
    return mask


def family_exists(family, N, r, D, K):
    """Whether the family has a mask with at least one free slot that K4 runs at this shape."""
    h = N // 2
    if family in ("random", "one_free"):
        return True
    if family == "free_vertex":
        return K >= 2
    if family in ("free_position", "free_end"):
        return h >= 2 and K >= 2
    if family == "fixed_vertex":
        return h >= 2 and K >= 3
    if family == "bench":
        return h >= 3 and K >= 2
    return h >= 2 and K >= 2 and (N, r, D) not in WAYPOINT_SHAPES  # waypoint: no registry entry


def make_mask(family, N, r, K, rng):
    """A [K+1][h] mask of the family with n_free >= 1 that meets well_posed (asserted)."""
    h = N // 2
    if family == "random":  # each slot fixed with probability 0.35, then repaired
        mask = (rng.rand(K + 1, h) < 0.35).astype(np.uint8)
        if not well_posed(mask, r):
            if K + 1 >= r:
                for v in rng.permutation(K + 1):  # Lagrange: positions at r vertices
                    mask[v, 0] = 1
                    if well_posed(mask, r):
                        break
            else:
                mask[0, :r] = 1  # Taylor
        if mask.all():
            for i in rng.permutation(mask.size):
                mask.flat[i] = 0
                if well_posed(mask, r):
                    break
                mask.flat[i] = 1
    elif family == "one_free":
        mask = np.ones((K + 1, h), dtype=np.uint8)
        for i in rng.permutation(mask.size):
            mask.flat[i] = 0
            if well_posed(mask, r):
                break
            mask.flat[i] = 1
    elif family == "bench":  # bench.py's generic mask: positions and velocities everywhere, both ends fully fixed
        mask = waypoint_mask(N, K)
        mask[:, 1] = 1
    else:
        mask = waypoint_mask(N, K)
        interior = rng.permutation(np.arange(1, K))
        if family == "free_position":  # velocity instead of position at some interior vertices
            for v in interior[:max(1, len(interior) // 2)]:
                mask[v, 0], mask[v, 1] = 0, 1
        elif family == "free_end":
            mask[-1, 1:] = 0
        elif family == "free_vertex":
            mask[interior[0], :] = 0
        elif family == "fixed_vertex":
            mask[interior[0], :] = 1
    assert well_posed(mask, r) and not mask.all(), (family, N, r, K, mask)
    if family != "waypoint":
        assert not np.array_equal(mask, waypoint_mask(N, K)), (family, N, r, K)
    return mask


def fixed_values(mask, B, D, rng, dim_scale=False):
    """values [B][K+1][h][D]: positions uniform in [-10, 10], derivatives in [-2, 2], zero at free slots; with dim_scale
    dimension d is scaled by d + 1, so that data read from a wrong dimension cannot pass.  -> (values, d_fixed
    [B][D][n_fixed] in the compact order: (vertex, derivative) row-major over the fixed slots)"""
    K1, h = mask.shape
    values = rng.uniform(-2, 2, size=(B, K1, h, D))
    values[:, :, 0, :] = rng.uniform(-10, 10, size=(B, K1, D))
    if dim_scale:
        values *= np.arange(1, D + 1)
    values *= mask[None, :, :, None]
    dfix = np.ascontiguousarray(np.transpose(values[:, mask.astype(bool), :], (0, 2, 1)))
    return values, dfix


def segment_times(B, K, kind, rng):
    """uniform in [0.5, 5] s, or log-uniform over [0.05, 20] s ("mixed", as waypoint_fixture)"""
    if kind == "mixed":
        return np.exp(rng.uniform(np.log(0.05), np.log(20.0), size=(B, K)))
    return rng.uniform(0.5, 5.0, size=(B, K))


def references(oracle, N, r, mask, values, times, dfix):
    """(exact coeffs, exact d_free) from the binary128 solve; (coeffs, d_free) of the reference-order fp64 solve"""
    B, K = times.shape
    D = dfix.shape[1]
    exact, exact_free, _ = oracle.exact_solve_batch(N, r, times, dfix, mask=mask, want_free=True)
    n_free = exact_free.shape[2]
    ref, ref_free = np.zeros((B, K, D, N)), np.zeros((B, D, n_free))
    for b in range(B):
        res = oracle.solve(N, r, mask, values[b], times[b])
        assert b > 0 or np.array_equal(res["d_fixed"], dfix[b])  # the compact order of fixed_values
        ref[b], ref_free[b] = res["coeffs"], res["d_free"]
    return exact, exact_free, ref, ref_free


def check_solution(label, out, dfree, ref, ref_free, exact, exact_free, free_floor):
    """check_parity on the coefficients; d_free within max(free_floor, 2 * the oracle's own d_free error) of exact
    (the rule test_large_k documents)"""
    assert np.isfinite(out).all() and np.isfinite(dfree).all(), label
    e_ge, _, _ = check_parity(out, ref, exact, label)
    e_f, e_of = rel_err_free(dfree, exact_free), rel_err_free(ref_free, exact_free)
    bad = e_f > np.maximum(free_floor, 2.0 * e_of)
    assert not bad.any(), f"{label}: d_free vs exact {e_f[bad].max():.3e} (oracle vs exact {e_of[bad].max():.3e})"
    return e_ge


# Parametrisations where a few trajectories miss check_parity, for K4 and the banded generic kernel alike.  On these
# fixtures (random masks with free positions over log-uniform times, N = 12 at r = 5, and single rows at N = 10) both
# kernels land 1e-10 .. 2e-3 from exact on the same trajectories, within 3.5x of each other, while the exact solution
# moves by at most 1e-14 under one-ulp changes of the times and fixed values: the digits are lost by fp64 Cholesky
# elimination of R_pp, which both kernels share as a method but not as code (the worst: N=10 r=3 D=4 trajectory 1,
# K4 1.9e-7 / banded 2.0e-7 / oracle 2.5e-8 from exact; the host-pipeline row misses rule 2 only: K4 8.4e-11 and the
# oracle 7.4e-11 from exact on opposite sides).  There each kernel is held, per trajectory, to
#     err(kernel, exact) <= max(2e-10, 2 * err(oracle, exact), 4 * err(other kernel, exact))
# on the coefficients and, with the case's floor for 2e-10, on d_free.  A defect of one kernel breaks it.
MASKED_LOSS_CASES = {"every N6r2D4", "every N10r3D4", "every N12r5D1", "every N12r5D2", "host pipeline",
                     "large K N12r5D1 K50", "many tiles D4"}


def check_pair(case, label, k4, banded, ref, ref_free, exact, exact_free, free_floor):
    """check_solution on K4 and on the banded kernel ((coeffs, d_free) each), or on a MASKED_LOSS_CASES case the rule
    described there.  -> K4's per-trajectory error vs exact"""
    if case not in MASKED_LOSS_CASES:
        e_ge = check_solution(label, *k4, ref, ref_free, exact, exact_free, free_floor)
        check_solution(label + " banded", *banded, ref, ref_free, exact, exact_free, free_floor)
        return e_ge
    assert all(np.isfinite(a).all() for a in k4 + banded), label
    e_k = (global_rel_err(k4[0], exact), rel_err_free(k4[1], exact_free))
    e_b = (global_rel_err(banded[0], exact), rel_err_free(banded[1], exact_free))
    e_o = (global_rel_err(ref, exact), rel_err_free(ref_free, exact_free))
    for what, i, floor in (("coefficients", 0, 2e-10), ("d_free", 1, max(2e-10, free_floor))):
        for name, mine, other in (("K4", e_k[i], e_b[i]), ("banded", e_b[i], e_k[i])):
            bound = np.maximum(floor, np.maximum(2.0 * e_o[i], 4.0 * other))
            bad = mine > bound
            j = int(np.argmax(bad))
            assert not bad.any(), (f"{label}: {name} {what} vs exact {mine[j]:.3e} on trajectory {j} "
                                   f"(oracle {e_o[i][j]:.3e}, other kernel {other[j]:.3e})")
    return e_k[0]


def _truth():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import truth
    return truth


CHECKER_CASES = [(f, N, r) for N in (2, 6, 12) for r in sorted({0, N // 2 - 1}) for f in FAMILIES
                 if family_exists(f, N, r, 1, 4)]


@pytest.mark.parametrize("family,N,r", CHECKER_CASES, ids=["{}-N{}r{}".format(*c) for c in CHECKER_CASES])
def test_binary128_checker_on_mask_families(oracle, family, N, r):
    """Every mask family: the binary128 solve (oracle/exact.cpp) == the 60-digit solve (oracle/truth.py) to fp64
    rounding, coefficients and d_free; the generator's masks are SPD in both."""
    truth = _truth()
    rng = np.random.RandomState(100 * N + 10 * r + FAMILIES.index(family))
    K, D = 4, 2
    mask = make_mask(family, N, r, K, rng)
    values, dfix = fixed_values(mask, 1, D, rng)
    times = segment_times(1, K, "uniform", rng)
    ex, ex_free, _ = oracle.exact_solve_batch(N, r, times, dfix, mask=mask, n_threads=1, want_free=True)
    tru, tru_free = truth.solve(N, r, mask, values[0], times[0])
    assert np.abs(ex[0] - tru).max() <= 2.3e-16 * np.abs(tru).max(), (family, N, r)
    assert np.abs(ex_free[0] - tru_free).max() <= 2.3e-16 * np.abs(tru_free).max(), (family, N, r)


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases (enumerated on the host, so that the CPU test below can check their routing)

# every (N, r) with r <= h - 1 -- all 21 H(1;r) tables -- crossed with D = 1..4: all 24 masked_block_kernel<N, DG>
EVERY_CASES = []
for _i, (_N, _r, _D) in enumerate([(N, r, D) for N in range(2, 13, 2) for r in range(N // 2) for D in (1, 2, 3, 4)]):
    _rng = np.random.RandomState(7000 + _i)
    _K = int(_rng.randint(3, 10))
    _fams = [f for f in FAMILIES if family_exists(f, _N, _r, _D, _K)]
    EVERY_CASES.append(dict(N=_N, r=_r, D=_D, K=_K, B=1 if (_r == 0 and _D == 2) else 37, seed=7000 + _i,
                            times="mixed" if _i % 4 == 3 else "uniform",
                            families=(_fams[_i % len(_fams)], _fams[(_i + 1) % len(_fams)])))

DG_SHAPES = [(10, 4), (8, 2)]
DG_DIMS = [5, 6, 7, 9]  # groups 3+2, 4+2, 4+3, 4+3+2
LARGE_K_SHAPES = [(10, 4, 3), (12, 5, 1), (8, 3, 4)]


def case_masks(case):
    rng = np.random.RandomState(case["seed"])
    return [(f, make_mask(f, case["N"], case["r"], case["K"], rng)) for f in case["families"]]


def gpu_problems():
    """(label, N, r, K, D, mask) of every K4 solve the GPU tests run"""
    out = []
    for c in EVERY_CASES:
        for f, mask in case_masks(c):
            out.append((f"every {f}", c["N"], c["r"], c["K"], c["D"], mask))
    for N, r in DG_SHAPES:
        for D in DG_DIMS:
            for f in ("random", "free_position"):
                out.append((f"dg {f}", N, r, 6, D, make_mask(f, N, r, 6, np.random.RandomState(N * 100 + D))))
    out.append(("host pipeline", 10, 4, 6, 7, make_mask("random", 10, 4, 6, np.random.RandomState(77))))
    out.append(("bench", 10, 4, 16, 3, make_mask("bench", 10, 4, 16, None)))
    for K in (50, 100):
        for N, r, D in LARGE_K_SHAPES:
            for f in ("random", "free_position"):
                out.append((f"large K {f}", N, r, K, D, make_mask(f, N, r, K, np.random.RandomState(K + N))))
    for D in (4, 7):
        out.append(("many tiles", 10, 4, 8, D, make_mask("free_position", 10, 4, 8, np.random.RandomState(D))))
    for D in (3, 7):
        out.append(("bad times", 10, 4, 6, D, make_mask("random", 10, 4, 6, np.random.RandomState(30 + D))))
    for r, f in INF_CASES:
        out.append((f"inf {f}", 10, r, 6, 3, inf_mask(f, r)))
    return out


def inf_mask(family, r):
    """fixed_vertex here fixes vertex 1 fully: segment 0 lies between two fully fixed vertices, so no pivot sees
    its time"""
    if family == "fixed_vertex":
        mask = waypoint_mask(10, 6)
        mask[1, :] = 1
        return mask
    return make_mask(family, 10, r, 6, np.random.RandomState(50 + r))


INF_CASES = [(1, "random"), (4, "bench"), (4, "fixed_vertex"), (1, "fixed_vertex"), (0, "random")]


def test_every_gpu_case_routes_to_the_masked_kernel():
    """Host-only: every (N, r, K, D, mask) the GPU part of this file runs is routed to the generic kernel (K4), so the
    suite cannot drift onto the waypoint kernels unnoticed; and every mask meets well_posed."""
    import mav_trajectory_generation_b200 as m
    probs = gpu_problems()
    assert len(probs) >= 84 * 2
    for label, N, r, K, D, mask in probs:
        assert well_posed(mask, r), (label, N, r, K, D)
        prob = m.Problem(N, r, K, D, fixed_mask=mask)
        assert prob.n_free >= 1, (label, N, r, K, D)
        assert prob.kernel == m.KERNEL_GENERIC, (label, N, r, K, D, mask)
    every = {f"every N{c['N']}r{c['r']}D{c['D']}" for c in EVERY_CASES}
    large = {f"large K N{N}r{r}D{D} K{K}" for N, r, D in LARGE_K_SHAPES for K in (50, 100)}
    assert MASKED_LOSS_CASES <= every | large | {"host pipeline", "many tiles D4", "many tiles D7"}
    # all 24 instantiations and all 21 tables
    assert {(c["N"], min(c["D"], 4)) for c in EVERY_CASES} == {(N, dg) for N in range(2, 13, 2) for dg in (1, 2, 3, 4)}
    assert len({(c["N"], c["r"]) for c in EVERY_CASES}) == 21
    # every family at every N where it exists, and a B = 1 case per N
    for N in range(2, 13, 2):
        cases = [c for c in EVERY_CASES if c["N"] == N]
        ran = {f for c in cases for f in c["families"]}
        assert ran == {f for c in cases for f in FAMILIES if family_exists(f, N, c["r"], c["D"], c["K"])}, N
        assert any(c["B"] == 1 for c in cases), N


# ---------------------------------------------------------------------------------------------------------------------
# 2. Every instantiation and every table

def run_case(solver, oracle, case, label, N, r, K, D, B, mask, times_kind, rng, dim_scale=False, free_floor=None):
    """K4 and the banded generic kernel (OPT_GENERIC_VARIANT = 1) on the same inputs, both against the binary128
    solve and the reference-order oracle (check_pair).  -> K4's per-trajectory error vs exact"""
    import torch
    import mav_trajectory_generation_b200 as m
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    values, dfix = fixed_values(mask, B, D, rng, dim_scale=dim_scale)
    times = segment_times(B, K, times_kind, rng)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    if free_floor is None:
        free_floor = 1e-9 if times_kind == "mixed" else 1e-10
    exact, exact_free, ref, ref_free = references(oracle, N, r, mask, values, times, dfix)
    out, dfree, status = solve(solver, prob, t_d, f_d)
    assert (status == 0).all(), (label, status)
    o1, f1, s1 = solve(solver, prob, t_d, f_d, GENERIC_VARIANT=1)
    assert (s1 == 0).all(), (label + " banded", s1)
    return check_pair(case, label, (out, dfree), (o1, f1), ref, ref_free, exact, exact_free, free_floor)


@pytest.mark.gpu
@pytest.mark.parametrize("case", EVERY_CASES, ids=["N{N}r{r}D{D}".format(**c) for c in EVERY_CASES])
def test_every_instantiation_and_table(solver, oracle, case):
    """K4 at every (N, r) and D = 1..4, two mask families per case, K in 3..9, ragged B (37: a full warp tile and a
    5-row tile; B = 1 once per N), uniform or log-uniform times: status 0, coefficients under check_parity, d_free
    within max(1e-10, 2 * the oracle's d_free error) of exact (1e-9 floor on log-uniform times); the banded generic
    kernel on the same inputs meets the same rules."""
    N, r, K, D, B = case["N"], case["r"], case["K"], case["D"], case["B"]
    rng = np.random.RandomState(case["seed"] + 1)
    for family, mask in case_masks(case):
        label = f"K4 {family} N={N} r={r} K={K} D={D} B={B} {case['times']}"
        run_case(solver, oracle, f"every N{N}r{r}D{D}", label, N, r, K, D, B, mask, case["times"], rng)


# ---------------------------------------------------------------------------------------------------------------------
# 3. Dimension groups, large K, the benchmark's mask, persistent reuse

@pytest.mark.gpu
@pytest.mark.parametrize("D", DG_DIMS)
@pytest.mark.parametrize("N,r", DG_SHAPES, ids=["N{}r{}".format(*s) for s in DG_SHAPES])
def test_dimension_groups(solver, oracle, N, r, D):
    """D > 4 runs one launch per dimension group, each offsetting the fixed values, the d_free index and the TMA column
    by d0.  Each dimension is scaled differently, so that a wrong offset cannot cancel out."""
    for family, mask in [(f, make_mask(f, N, r, 6, np.random.RandomState(N * 100 + D))) for f in ("random", "free_position")]:
        run_case(solver, oracle, "dg", f"K4 {family} N={N} r={r} K=6 D={D}", N, r, 6, D, 37, mask, "uniform",
                 np.random.RandomState(N * 1000 + D), dim_scale=True)


def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


@pytest.mark.gpu
def test_dimension_groups_host_pipeline(solver, oracle):
    """solve_linear_host with pinned buffers, B > one pipeline chunk, D = 7 (groups 4 + 3): three streams each run
    both group launches with their factor LIFO in their own scratch slot.  Bitwise equal to the device path."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 7, 5003
    mask = make_mask("random", N, r, K, np.random.RandomState(77))
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    rng = np.random.RandomState(78)
    values, dfix = fixed_values(mask, B, D, rng, dim_scale=True)
    times = segment_times(B, K, "uniform", rng)
    dev, dev_free, dev_status = solve(solver, prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda())
    assert (dev_status == 0).all()
    host = torch.full((B, K, D, N), float("nan"), dtype=torch.float64).pin_memory()
    host_free = torch.full((B, D, prob.n_free), float("nan"), dtype=torch.float64).pin_memory()
    host_status = torch.full((B,), -1, dtype=torch.int32).pin_memory()
    solver.solve_linear_host(prob, _pinned(times), _pinned(dfix), host, d_free=host_free, status=host_status)
    assert same_bits(host.numpy(), dev), "host pipeline differs from the device path"
    assert same_bits(host_free.numpy(), dev_free)
    assert same_bits(host_status.numpy(), dev_status)
    sub = rng.choice(B, size=32, replace=False)
    check_rows(solver, oracle, "host pipeline", "host pipeline N=10 K=6 D=7", prob, mask, values, times, dfix, sub,
               dev, dev_free)


def check_rows(solver, oracle, case, label, prob, mask, values, times, dfix, sub, out, dfree):
    """check_pair on the rows `sub` of a batch, the banded generic kernel solving those rows alone"""
    import torch
    t_s, f_s = np.ascontiguousarray(times[sub]), np.ascontiguousarray(dfix[sub])
    o1, f1, s1 = solve(solver, prob, torch.from_numpy(t_s).cuda(), torch.from_numpy(f_s).cuda(), GENERIC_VARIANT=1)
    assert (s1 == 0).all(), label
    exact, exact_free, ref, ref_free = references(oracle, prob.N, prob.r, mask, values[sub], t_s, f_s)
    check_pair(case, label, (out[sub], dfree[sub]), (o1, f1), ref, ref_free, exact, exact_free, 1e-10)


@pytest.mark.gpu
def test_benchmark_mask_every_row(solver, oracle):
    """The mask bench.py measures (C3 shape, velocity fixed at every vertex), 4096 trajectories, every row under
    check_parity and d_free against exact."""
    N, r, K, D, B = 10, 4, 16, 3, 4096
    mask = make_mask("bench", N, r, K, None)
    e_ge = run_case(solver, oracle, "bench", "K4 bench mask", N, r, K, D, B, mask, "uniform", np.random.RandomState(16))
    print(f"bench mask N=10 K=16 D=3 B=4096: CUDA-exact median {np.median(e_ge):.2e}  "
          f"p99 {np.quantile(e_ge, 0.99):.2e}  max {e_ge.max():.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [50, 100])
@pytest.mark.parametrize("N,r,D", LARGE_K_SHAPES, ids=["N{}r{}D{}".format(*s) for s in LARGE_K_SHAPES])
def test_large_k_vs_exact(solver, oracle, N, r, D, K):
    """K = 50 and 100: the factor LIFO is (K+1) * slots deep.  random and free_position masks, B = 5."""
    for f in ("random", "free_position"):
        mask = make_mask(f, N, r, K, np.random.RandomState(K + N))
        run_case(solver, oracle, f"large K N{N}r{r}D{D} K{K}", f"K4 {f} N={N} r={r} K={K} D={D}", N, r, K, D, 5, mask,
                 "uniform",
                 np.random.RandomState(K * 10 + N))


def resident_warp_bound():
    """Warps per SM K4 can keep resident: 128-thread CTAs, >= 128 registers per thread at N = 10 (ptxas: 243 at
    DG = 4, 212 at DG = 3), so at most four CTAs = 16 warps."""
    return 16


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 7])
def test_many_tiles_per_warp(solver, oracle, D):
    """Every resident warp runs >= 3 warp tiles, reusing its LIFO column: rows solved alone and a batch split off a
    warp boundary are bitwise equal to the batch; 256 sampled rows under check_parity; on every row the fixed values
    are reproduced and derivatives 0..h-1 are continuous at interior vertices (evaluated with torch)."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K = 10, 4, 8
    h = N // 2
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = sms * resident_warp_bound() * 32 * 3 + 21
    mask = make_mask("free_position", N, r, K, np.random.RandomState(D))
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    rng = np.random.RandomState(90 + D)
    values, dfix = fixed_values(mask, B, D, rng, dim_scale=True)
    times = segment_times(B, K, "uniform", rng)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    out, dfree, status = solve(solver, prob, t_d, f_d)
    assert (status == 0).all()
    label = f"many tiles D={D} B={B}"

    for b in rng.choice(B, size=64, replace=False):
        o1, f1, s1 = solve(solver, prob, t_d[b:b + 1], f_d[b:b + 1])
        assert same_bits(o1, out[b:b + 1]) and same_bits(f1, dfree[b:b + 1]) and same_bits(s1, status[b:b + 1]), \
            f"{label}: row {b} alone differs from the batch"
    cut = 32 * 1000 + 13
    oa, fa, sa = solve(solver, prob, t_d[:cut], f_d[:cut])
    ob, fb, sb = solve(solver, prob, t_d[cut:], f_d[cut:])
    assert same_bits(np.concatenate([oa, ob]), out), f"{label}: split at {cut} differs"
    assert same_bits(np.concatenate([fa, fb]), dfree) and same_bits(np.concatenate([sa, sb]), status)

    sub = np.sort(rng.choice(B, size=256, replace=False))
    check_rows(solver, oracle, f"many tiles D{D}", label, prob, mask, values, times, dfix, sub, out, dfree)

    # every row: derivative k at both ends of every segment, from the coefficients, with torch
    c = torch.from_numpy(out).cuda()
    T = t_d[:, :, None, None]
    powers = torch.arange(N, device="cuda", dtype=torch.float64)
    fixed = torch.from_numpy(mask.astype(bool)).cuda()
    vals = torch.from_numpy(values).cuda()
    for k in range(h):
        fall = torch.ones(N, device="cuda", dtype=torch.float64)
        for q in range(k):
            fall = fall * (powers - q).clamp_min(0)
        at0 = c[..., k] * fall[k]                                            # [B][K][D], t = 0
        atT = (c * fall * T ** (powers - k).clamp_min(0)).sum(dim=-1)        # t = T
        vert = torch.cat([at0, atT[:, -1:]], dim=1)                          # [B][K+1][D]
        tol = 1e-9 * max(1.0, float(vert.abs().max()))
        err_fix = (vert[:, fixed[:, k]] - vals[:, fixed[:, k], k]).abs().max()
        err_cont = (atT[:, :-1] - at0[:, 1:]).abs().max()
        assert err_fix <= tol, f"{label}: derivative {k} misses its fixed values by {float(err_fix):.3e}"
        assert err_cont <= tol, f"{label}: derivative {k} jumps by {float(err_cont):.3e} at an interior vertex"


# ---------------------------------------------------------------------------------------------------------------------
# 4. Status bits

BAD_ROWS = [2, 7, 13, 31, 32, 40, 50, 63, 68]  # B = 70: warp tiles of 32, 32 and 6 rows


def _bad_time_batch(D, mask, seed):
    rng = np.random.RandomState(seed)
    K, B = mask.shape[0] - 1, 70
    values, dfix = fixed_values(mask, B, D, rng)
    times = segment_times(B, K, "uniform", rng)
    return times, dfix


def _rest_equal(solver, prob, times, dfix, bad, out, dfree, status, label):
    """the rows outside `bad` are bitwise equal to the same batch solved without the bad rows"""
    import torch
    good = np.setdiff1d(np.arange(times.shape[0]), bad)
    o2, f2, s2 = solve(solver, prob, torch.from_numpy(np.ascontiguousarray(times[good])).cuda(),
                       torch.from_numpy(np.ascontiguousarray(dfix[good])).cuda())
    assert (s2 == 0).all(), label
    assert same_bits(out[good], o2), f"{label}: good rows differ from the clean batch"
    assert same_bits(dfree[good], f2) and same_bits(status[good], s2), f"{label}: good d_free / status differ"


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 7])
def test_bad_times_set_status(solver, D):
    """Time 0, a negative time and NaN in the first, a middle and the last segment of rows spread over the warp
    tiles: STATUS_BAD_TIME on those rows (written by the d0 = 0 launch), every other row bitwise unaffected."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K = 10, 4, 6
    mask = make_mask("random", N, r, K, np.random.RandomState(30 + D))
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    times, dfix = _bad_time_batch(D, mask, 31 + D)
    for i, b in enumerate(BAD_ROWS):
        times[b, (0, K // 2, K - 1)[i % 3]] = (0.0, -1.0, float("nan"))[i // 3]
    out, dfree, status = solve(solver, prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda())
    assert all(status[b] & m.STATUS_BAD_TIME for b in BAD_ROWS), status[BAD_ROWS]
    _rest_equal(solver, prob, times, dfix, BAD_ROWS, out, dfree, status, f"bad times D={D}")


@pytest.mark.gpu
@pytest.mark.parametrize("r,family", INF_CASES, ids=["r{}-{}".format(*c) for c in INF_CASES])
def test_infinite_time_sets_status(solver, r, family):
    """A segment time of +inf in the first, a middle and the last segment sets STATUS_BAD_TIME.  The fixed_vertex mask
    puts segment 0 between two fully fixed vertices, where no pivot sees the time: before the time check caught +inf,
    those rows came back with status 0 and non-finite coefficients."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, K, D = 10, 6, 3
    mask = inf_mask(family, r)
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    times, dfix = _bad_time_batch(D, mask, 60 + r)
    bad = BAD_ROWS[:3]
    for i, b in enumerate(bad):
        times[b, (0, K // 2, K - 1)[i]] = float("inf")
    out, dfree, status = solve(solver, prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda())
    finite = [bool(np.isfinite(out[b]).all()) for b in bad]
    assert all(status[b] & m.STATUS_BAD_TIME for b in bad), (f"r={r} {family}: status {status[bad]} on +inf rows "
                                                             f"(coefficients finite: {finite})")
    _rest_equal(solver, prob, times, dfix, bad, out, dfree, status, f"inf r={r} {family}")
