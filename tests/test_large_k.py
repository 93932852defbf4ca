"""Large-K paths against high-precision references.

  1. the chunked checkpoint-and-recompute waypoint kernel (K3, MTG_OPT_WAYPOINT_VARIANT = 5) at every compiled
     (N, r, D) of the waypoint registry, with non-zero start / end derivatives and every chunk-boundary case;
  2. default routing at the reference's own sizes (K = 50, 100), the fused Nfabian entry's pack fallback and the
     host pipeline on a K3 shape;
  3. the Mellinger gradient where it leaves the fused cost-only kernel (large K, shapes without a cost-only kernel,
     K * D > 256) and where the perturbed times hit the 0.1 s lower bound;
  4. computeCost() at every cost_kernel specialisation and the generic fallback, against the exact rational value.
"""
import contextlib
import math
from fractions import Fraction

import numpy as np
import pytest

from test_gpu_parity import check_parity, global_rel_err

# every (N, r, D) of kWaypointKernels (csrc/mtg_capi.cu); each has its own K3 instantiation
WAYPOINT_SHAPES = [(10, 4, 3), (10, 4, 1), (10, 4, 2), (10, 4, 4), (10, 3, 3), (10, 3, 1), (10, 2, 3), (10, 2, 1),
                   (8, 3, 3), (8, 3, 1), (8, 3, 2), (8, 3, 4), (12, 5, 3), (12, 5, 1), (12, 5, 4), (6, 2, 3), (6, 2, 1)]
# shapes of kV4Kernels: the persistent kernel v4 runs the same fold-carry arithmetic as K3
V4_SHAPES = {(10, 4, 3), (8, 3, 3), (10, 4, 1), (10, 3, 3), (10, 2, 3), (12, 5, 3)}
# Mellinger: reference increment_time (nonlinear_impl.h:310) and kOptimizationTimeLowerBound
MEL_INC, MEL_LOWER = 0.1, 0.1


def _shape_id(shape):
    return "N{}r{}D{}".format(*shape)


@contextlib.contextmanager
def options(solver, **opts):
    """Set MTG_OPT_<name> options for the block; every one goes back to 0 (its default) afterwards."""
    import mav_trajectory_generation_b200 as m
    try:
        for name, value in opts.items():
            solver.set_option(getattr(m.capi, "OPT_" + name), value)
        yield
    finally:
        for name in opts:
            solver.set_option(getattr(m.capi, "OPT_" + name), 0)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def rel_err_free(got, exact):
    """per-trajectory max |got - exact| / max |exact| of d_free [B][D][n_free]"""
    B = exact.shape[0]
    return np.abs(got - exact).reshape(B, -1).max(axis=1) / np.abs(exact).reshape(B, -1).max(axis=1)


def solve(solver, prob, t_d, f_d, **opts):
    """solve_linear with the given options -> (coeffs, d_free, status) as numpy.  Outputs start as NaN / -1 so that
    an entry the kernel never writes cannot pass a comparison."""
    import torch
    B = t_d.shape[0]
    coeffs = torch.full((B, prob.K, prob.D, prob.N), float("nan"), dtype=torch.float64, device="cuda")
    dfree = torch.full((B, prob.D, max(prob.n_free, 1)), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    with options(solver, **opts):
        solver.solve_linear(prob, t_d, f_d, coeffs=coeffs, d_free=dfree, status=status)
        torch.cuda.synchronize()
    return coeffs.cpu().numpy(), dfree.cpu().numpy(), status.cpu().numpy()


def waypoint_fixture(oracle, N, K, D, B, times_kind, seed):
    """createRandomVertices positions; segment times from the Nfabian fixture ("nfabian") or log-uniform over
    [0.05, 20] s within each trajectory ("mixed"); even trajectories get start / end derivatives uniform in [-1, 1],
    odd ones keep them zero.  -> positions [B][K+1][D], times [B][K], start / end derivatives [B][h-1][D]"""
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    rng = np.random.RandomState(seed)
    if times_kind == "mixed":
        times = np.exp(rng.uniform(np.log(0.05), np.log(20.0), size=(B, K)))
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    sd[1::2] = 0.0
    ed[1::2] = 0.0
    return pos, np.ascontiguousarray(times), sd, ed


def oracle_solve(oracle, N, r, pos, times, sd, ed):
    """The reference-order fp64 solve of every trajectory, end derivatives included -> (coeffs, d_free)."""
    B, K = times.shape
    D = pos.shape[2]
    coeffs = np.zeros((B, K, D, N))
    dfree = np.zeros((B, D, (K - 1) * (N // 2 - 1)))
    for b in range(B):
        mask, values = oracle.waypoint_problem(N, pos[b])
        values[0, 1:, :] = sd[b]
        values[-1, 1:, :] = ed[b]
        res = oracle.solve(N, r, mask, values, times[b])
        coeffs[b], dfree[b] = res["coeffs"], res["d_free"]
    return coeffs, dfree


# ---------------------------------------------------------------------------------------------------------------------
# 1. K3 at every compiled specialisation

K3_CASES = [  # K, forced chunk (0 = auto), B, segment times
    pytest.param(2, 0, 1, "nfabian", id="K2-B1"),             # one interior vertex: no sweep step before the middle one
    pytest.param(7, 1, 5, "mixed", id="K7-chunk1-B5"),        # odd K: unbalanced halves, one block per chunk
    pytest.param(16, 3, 33, "nfabian", id="K16-chunk3-B33"),  # 7 own vertices in chunks of 3: partial outer chunk
    pytest.param(50, 0, 17, "mixed", id="K50-auto-B17"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("K,chunk,B,times_kind", K3_CASES)
@pytest.mark.parametrize("N,r,D", WAYPOINT_SHAPES, ids=[_shape_id(s) for s in WAYPOINT_SHAPES])
def test_chunked_kernel_every_specialisation(solver, oracle, N, r, D, K, chunk, B, times_kind):
    """K3 forced at every registry shape, half the trajectories with non-zero end derivatives:
    (a) against the binary128 solve under check_parity, d_free against the exact d_free;
    (b) coefficients, d_free and status bitwise equal for forced chunks 1, 2 and auto (the recompute replays the
        same arithmetic);
    (c) bitwise equal to the persistent kernel v4 where it exists (K <= 8): both fold the fixed end derivatives into
        the first step's carry and compute the outward coupling before the activity test."""
    import torch
    import mav_trajectory_generation_b200 as m
    pos, times, sd, ed = waypoint_fixture(oracle, N, K, D, B, times_kind, seed=1000 * N + 100 * r + 10 * D + K)
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_WAYPOINT
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    label = f"K3 N={N} r={r} D={D} K={K} chunk={chunk} B={B} {times_kind}"
    out, dfree, status = solve(solver, prob, t_d, f_d, WAYPOINT_VARIANT=5, CHUNK_BLOCKS=chunk)
    assert (status == 0).all(), (label, status)
    assert np.isfinite(out).all() and np.isfinite(dfree).all(), label

    # (a) binary128 solve; the reference-order side handles the non-zero end derivatives
    exact, exact_free, _ = oracle.exact_solve_batch(N, r, times, dfix, want_free=True)
    ref, ref_free = oracle_solve(oracle, N, r, pos, times, sd, ed)
    check_parity(out, ref, exact, label)
    # d_free: a flat 1e-9 from exact on the Nfabian fixture at N <= 10 (as test_large_k_chunked_kernel).  On log-uniform
    # times and at N = 12 the sweep's d_free lands up to ~6e-3 from exact (N = 12, K = 7), where the reference-order
    # arithmetic is ~1e-1 off -- the same loss check_parity admits for the coefficients -- so there d_free is held to
    # check_parity's first rule instead: within max(1e-9, 2 * the oracle's own d_free error).
    e_f, e_of = rel_err_free(dfree, exact_free), rel_err_free(ref_free, exact_free)
    flat = times_kind == "nfabian" and N <= 10
    bad = e_f > (1e-9 if flat else np.maximum(1e-9, 2.0 * e_of))
    assert not bad.any(), f"{label}: d_free vs exact {e_f[bad].max():.3e} (oracle vs exact {e_of[bad].max():.3e})"

    # (b) chunk invariance
    for c in (1, 2, 0):
        if c == chunk:
            continue
        o2, f2, s2 = solve(solver, prob, t_d, f_d, WAYPOINT_VARIANT=5, CHUNK_BLOCKS=c)
        assert same_bits(o2, out), f"{label}: coefficients differ with chunk {c}"
        assert same_bits(f2, dfree), f"{label}: d_free differs with chunk {c}"
        assert same_bits(s2, status), f"{label}: status differs with chunk {c}"

    # (c) the persistent kernel v4: identical arithmetic
    if K <= 8 and (N, r, D) in V4_SHAPES:
        o4, f4, s4 = solve(solver, prob, t_d, f_d, WAYPOINT_VARIANT=4)
        assert same_bits(o4, out), f"{label}: K3 differs from v4"
        assert same_bits(f4, dfree), f"{label}: K3 d_free differs from v4"
        assert same_bits(s4, status), f"{label}: K3 status differs from v4"


# ---------------------------------------------------------------------------------------------------------------------
# 2. Default routing at the reference's sizes

def banded_solve(solver, prob, t_d, f_d):
    """The same solve through the banded generic kernel, which shares no code with the waypoint sweep: an output that
    is only 8-byte aligned takes it (launch_solve)."""
    import torch
    B = t_d.shape[0]
    n = B * prob.K * prob.D * prob.N
    big = torch.full((n + 1,), float("nan"), dtype=torch.float64, device="cuda")
    out = big[1:].view(B, prob.K, prob.D, prob.N)
    assert out.data_ptr() % 16 == 8
    solver.solve_linear(prob, t_d, f_d, coeffs=out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


# Parametrisations where check_parity does not hold for the waypoint sweep.  On these 1-D fixtures a few trajectories
# land further from exact than check_parity allows: (10,4,1) at K = 50 / 100 up to 7.1e-11 from exact where the oracle
# is at 8.5e-11, so CUDA vs oracle exceeds 1e-10 (rule 2); (12,5,1) at K = 50 1.9e-8 where the oracle is at 4.4e-9, and
# the Nfabian entry at (10,4,1), K = 100 1.1e-10 where the oracle is at 2.4e-11 (rule 1).  The exact solutions move by
# ~1e-15 under one-ulp input perturbations, so these are digits lost by fp64 elimination: the banded generic kernel,
# which shares no code with the sweep, is 2e-8 from exact on the (12,5,1) fixture and 4e-11 on the (10,4,1) ones, and
# the sweep's results are bit-identical to those of the kernels before the sweep arithmetic was factored into
# mtg_sweep.cuh.  There each trajectory is held to
#     err(CUDA, exact) <= max(2e-10, 2 * err(oracle, exact), 4 * err(banded generic kernel, exact)),
# which the measured errors meet with a margin of 1.3x or more (and which a real defect of the sweep would not).
SWEEP_LOSS_CASES = {("default", 10, 4, 1, 50), ("default", 10, 4, 1, 100), ("default", 12, 5, 1, 50),
                    ("nfabian", 10, 4, 1, 100)}


def check_parity_or_sweep_loss(case, out, ref, exact, banded, label):
    """check_parity, or on a SWEEP_LOSS_CASES parametrisation the bounded rule described there (`banded`: a thunk
    returning the banded generic kernel's result on the same inputs)."""
    if case not in SWEEP_LOSS_CASES:
        check_parity(out, ref, exact, label)
        return
    gen = banded()
    assert np.isfinite(gen).all(), label
    e_ge, e_oe, e_be = global_rel_err(out, exact), global_rel_err(ref, exact), global_rel_err(gen, exact)
    bound = np.maximum(2e-10, np.maximum(2.0 * e_oe, 4.0 * e_be))
    bad = e_ge > bound
    assert not bad.any(), (f"{label}: CUDA vs exact {e_ge[bad].max():.3e} on trajectory {int(np.argmax(bad))} "
                           f"(oracle {e_oe[np.argmax(bad)]:.3e}, banded generic kernel {e_be[np.argmax(bad)]:.3e})")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [50, 100])  # polynomial_timing_evaluation.cpp:114-129, test_polynomial_optimization.cpp
@pytest.mark.parametrize("N,r,D", WAYPOINT_SHAPES, ids=[_shape_id(s) for s in WAYPOINT_SHAPES])
def test_default_routing_large_k(solver, oracle, N, r, D, K):
    """Default routing at K = 50 and 100 on the Nfabian fixture (zero end derivatives, where v3, v4, v5 and K3 agree
    bitwise wherever they overlap): equal to forced K3 at auto chunk, and within the parity contract."""
    import torch
    import mav_trajectory_generation_b200 as m
    B = 48
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=20000 + 100 * N + 10 * r + D)
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_WAYPOINT
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    label = f"default N={N} r={r} D={D} K={K}"
    out, dfree, status = solve(solver, prob, t_d, f_d)
    k3, k3_free, k3_status = solve(solver, prob, t_d, f_d, WAYPOINT_VARIANT=5)
    assert (status == 0).all() and (k3_status == 0).all(), label
    assert np.isfinite(out).all(), label
    assert same_bits(out, k3), f"{label}: default differs from K3"
    assert same_bits(dfree, k3_free) and same_bits(status, k3_status), f"{label}: default d_free / status differ from K3"
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, times, n_threads=oracle.hardware_threads())
    exact = oracle.exact_solve_batch(N, r, times, dfix)
    check_parity_or_sweep_loss(("default", N, r, D, K), out, ref, exact, lambda: banded_solve(solver, prob, t_d, f_d),
                               label)


NFABIAN_FALLBACK_SHAPES = [(8, 3, 3), (12, 5, 3), (10, 4, 1)]  # the fused kernel does not fit at large K


@pytest.mark.gpu
@pytest.mark.parametrize("K", [50, 100])
@pytest.mark.parametrize("N,r,D", NFABIAN_FALLBACK_SHAPES, ids=[_shape_id(s) for s in NFABIAN_FALLBACK_SHAPES])
def test_fused_nfabian_large_k_fallback(solver, oracle, N, r, D, K):
    """solve_waypoints_nfabian where the fused kernel does not fit: the pack fallback must give exactly what
    solve_linear gives on the kernel's own segment times and the packed constraints, and pass the parity contract."""
    import torch
    import mav_trajectory_generation_b200 as m
    B = 48
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=30000 + 100 * N + 10 * r + D)  # v_max 3, a_max 5
    t_out = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    out = solver.solve_waypoints_nfabian(N, r, torch.from_numpy(pos).cuda(), 3.0, 5.0, 6.5, seg_times_out=t_out,
                                         status=status)
    torch.cuda.synchronize()
    assert (status.cpu().numpy() == 0).all()
    np.testing.assert_allclose(t_out.cpu().numpy(), times, rtol=4e-16, atol=0)  # device exp() vs glibc exp()
    seg_times = t_out.cpu().numpy()
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    f_d = torch.from_numpy(dfix).cuda()
    again = solver.solve_linear(prob, t_out, f_d)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    assert np.isfinite(out).all()
    assert np.array_equal(out, again.cpu().numpy()), "fused entry differs from solve_linear on its own inputs"
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, seg_times, n_threads=oracle.hardware_threads())
    exact = oracle.exact_solve_batch(N, r, seg_times, dfix)
    check_parity_or_sweep_loss(("nfabian", N, r, D, K), out, ref, exact, lambda: banded_solve(solver, prob, t_out, f_d),
                               f"nfabian N={N} r={r} D={D} K={K}")


def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


@pytest.mark.gpu
def test_host_pipeline_chunked_kernel_bitwise(solver, oracle):
    """The host-pointer pipeline at a non-headline K3 shape, B > one pipeline chunk, pinned buffers: three streams run
    K3 concurrently, each with its checkpoints in its own scratch slot.  Bitwise equal to one device-pointer launch."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 12, 5, 40, 4, 5003
    rng = np.random.RandomState(40)
    pos = rng.uniform(-10, 10, size=(B, K + 1, D))
    dist = np.maximum(np.linalg.norm(np.diff(pos, axis=1), axis=2), 0.2)
    times = np.ascontiguousarray(dist / 3.0 * 2 * (1.0 + 6.5 * 3.0 / 5.0 * np.exp(-dist / 3.0 * 2)))
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    sd[1::2] = 0.0
    ed[1::2] = 0.0
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    dev, dev_free, dev_status = solve(solver, prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda(),
                                      WAYPOINT_VARIANT=5)
    assert (dev_status == 0).all()
    host = torch.full((B, K, D, N), float("nan"), dtype=torch.float64).pin_memory()
    host_free = torch.full((B, D, prob.n_free), float("nan"), dtype=torch.float64).pin_memory()
    host_status = torch.full((B,), -1, dtype=torch.int32).pin_memory()
    with options(solver, WAYPOINT_VARIANT=5):
        solver.solve_linear_host(prob, _pinned(times), _pinned(dfix), host, d_free=host_free, status=host_status)
    assert same_bits(host.numpy(), dev), "host pipeline differs from the device path"
    assert same_bits(host_free.numpy(), dev_free)
    assert same_bits(host_status.numpy(), dev_status)
    sub = rng.choice(B, size=32, replace=False)
    exact = oracle.exact_solve_batch(N, r, times[sub], dfix[sub])
    ref, _ = oracle_solve(oracle, N, r, pos[sub], times[sub], sd[sub], ed[sub])
    check_parity(dev[sub], ref, exact, "host pipeline N=12 K=40 D=4")


# ---------------------------------------------------------------------------------------------------------------------
# 3. Mellinger gradient at large K, and the time clamp

def mellinger_times(times):
    """[B][K] -> [B][K+1][K]: the unperturbed times, then for each segment n the reference's perturbation (+0.1 on n,
    -0.1/(K-1) on the others, then max(0.1, t)) in the reference's fp64 arithmetic."""
    B, K = times.shape
    out = np.empty((B, K + 1, K))
    out[:, 0] = times
    corr = MEL_INC / (K - 1.0)
    for n in range(K):
        t = times - corr
        t[:, n] = times[:, n] + MEL_INC
        out[:, n + 1] = np.maximum(MEL_LOWER, t)
    return out


def mellinger_reference(oracle, N, r, times, dfix):
    """(cost [B], gradient [B][K]): binary128 costs of the K+1 time vectors, forward differences in fp64."""
    B, K = times.shape
    tx = mellinger_times(times).reshape(B * (K + 1), K)
    _, _, J = oracle.exact_solve_batch(N, r, tx, np.repeat(dfix, K + 1, axis=0), want_cost=True)
    J = J.reshape(B, K + 1)
    return J[:, 0], (J[:, 1:] - J[:, :1]) / MEL_INC


MELLINGER_CASES = [  # N, r, K, D, B, segment times
    pytest.param(10, 4, 50, 3, 4, "nfabian", id="N10r4K50D3"),  # cost-only kernel does not fit: expand + solve + cost
    pytest.param(12, 5, 20, 3, 4, "nfabian", id="N12r5K20D3"),
    pytest.param(10, 4, 12, 2, 6, "nfabian", id="N10r4K12D2"),  # no cost-only kernel for the shape
    pytest.param(8, 3, 12, 4, 6, "nfabian", id="N8r3K12D4"),
    pytest.param(10, 4, 90, 3, 2, "nfabian", id="N10r4K90D3"),  # K * D = 270 > 256: one trajectory per cost block
    pytest.param(10, 4, 2, 3, 5, "clamp", id="N10r4K2D3-clamp"),  # 0.12 s segments: t - 0.1 / (K-1) < 0.1
    pytest.param(10, 4, 5, 3, 5, "clamp", id="N10r4K5D3-clamp"),
    pytest.param(8, 3, 5, 4, 5, "clamp", id="N8r3K5D4-clamp"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("N,r,K,D,B,times_kind", MELLINGER_CASES)
def test_mellinger_gradient_large_k_and_clamp(solver, oracle, N, r, K, D, B, times_kind):
    """cost_gradient_mellinger against the binary128 reference on the same expanded time vectors: cost within 1e-8
    relative, gradient within 1e-6 * max(|J|, |grad|) (the tolerances of test_batched_mellinger_gradient), on the
    default path and on the unfused path (expand + solve + cost kernels); the two paths agree as in that test."""
    import torch
    import mav_trajectory_generation_b200 as m
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=40000 + 100 * N + 10 * K + D)
    if times_kind == "clamp":
        times[:, ::2] = 0.12
        assert (mellinger_times(times)[:, 1:] == MEL_LOWER).any()  # the fixture reaches the clamp
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    c_ref, g_ref = mellinger_reference(oracle, N, r, times, dfix)
    results = {}
    for unfused in (0, 1):
        with options(solver, MELLINGER_UNFUSED=unfused):
            cost, grad = solver.cost_gradient_mellinger(prob, t_d, f_d)
            torch.cuda.synchronize()
        cost, grad = cost.cpu().numpy(), grad.cpu().numpy()
        results[unfused] = cost, grad
        e_c = np.abs(cost - c_ref) / np.abs(c_ref)
        e_g = np.abs(grad - g_ref).max(axis=1) / np.maximum(np.abs(c_ref), np.abs(g_ref).max(axis=1))
        label = f"Mellinger N={N} r={r} K={K} D={D} {times_kind} unfused={unfused}"
        print(f"{label}: cost vs exact {e_c.max():.2e}, gradient vs exact {e_g.max():.2e}")
        assert (e_c <= 1e-8).all(), f"{label}: cost vs exact {e_c.max():.3e}"
        assert (e_g <= 1e-6).all(), f"{label}: gradient vs exact {e_g.max():.3e}"
    (cost, grad), (cost_u, grad_u) = results[0], results[1]
    assert np.abs(cost_u - cost).max() <= 1e-8 * np.abs(cost).max()
    assert np.abs(grad_u - grad).max() <= 1e-6 * max(np.abs(cost).max(), np.abs(grad).max())


# ---------------------------------------------------------------------------------------------------------------------
# 4. computeCost() against the exact quadratic form

_LCM = math.lcm(*range(1, 24))  # every denominator a + b - 2r + 1 of Q (N <= 12)


def _dyadic(x):
    """float -> (m, e) with x == m * 2**e exactly"""
    num, den = float(x).as_integer_ratio()
    return num, 1 - den.bit_length()


def _dyadic_sum(terms):
    """exact sum of (m, e) terms (value m * 2**e) -> Fraction"""
    e0 = min(e for _, e in terms)
    total = sum(mm << (e - e0) for mm, e in terms)
    return Fraction(total) * Fraction(2) ** e0


def exact_cost(N, r, times, coeffs):
    """computeCost() over the rationals, evaluated on the given fp64 inputs: per trajectory
    J = 0.5 * sum_{segment, dimension} c^T Q(T) c  with  Q[a][b] = 2 B(r,a) B(r,b) T^(a+b-2r+1) / (a+b-2r+1)
    (reference linear_impl.h:567-583), and S = the same sum with |q_a| |q_b| for q_a q_b, q_a = B(r,a) c_a T^(a-r).
    times [B][K], coeffs [B][K][D][N] -> (J, S): lists of Fractions."""
    B, K, D, _ = coeffs.shape
    bc = [math.perm(a, r) for a in range(N)]  # B(r, a) = a! / (a-r)!
    J, S = [], []
    for b in range(B):
        terms_j, terms_s = [], []  # each: (numerator over _LCM, binary exponent)
        for i in range(K):
            tm, te = _dyadic(times[b, i])
            for d in range(D):
                q = []
                for a in range(r, N):
                    cm, ce = _dyadic(coeffs[b, i, d, a])
                    q.append((bc[a] * cm * tm ** (a - r), ce + te * (a - r)))
                e0 = min(e for _, e in q)
                qi = [mm << (e - e0) for mm, e in q]
                nj = ns = 0
                for ia, qa in enumerate(qi):
                    for ib, qb in enumerate(qi):
                        w = qa * qb * (_LCM // (ia + ib + 1))
                        nj += w
                        ns += abs(w)
                # 0.5 * 2 * T * sum q_a q_b / (a+b-2r+1)
                terms_j.append((tm * nj, 2 * e0 + te))
                terms_s.append((tm * ns, 2 * e0 + te))
        J.append(_dyadic_sum(terms_j) / _LCM)
        S.append(_dyadic_sum(terms_s) / _LCM)
    return J, S


def cost_bound(N, r, K, D):
    """forward-error bound of cost_kernel in units of S: the (N-r)^2-term fma sum of rounded q_a q_b / k products, the
    K*D-term accumulation, and the powers of T"""
    return (4 * (N - r) ** 2 + 2 * K * D + 64) * 2.0 ** -53


def test_exact_cost_helper_vs_cost_matrix(oracle):
    """The rational computeCost() helper against the oracle's fp64 cost matrix (reference
    computeQuadraticCostJacobian) on random single segments, and on one closed form."""
    rng = np.random.RandomState(12)
    for trial in range(12):
        N = int(rng.choice([2, 4, 6, 8, 10, 12]))
        r = int(rng.randint(0, N // 2))
        T = float(np.exp(rng.uniform(np.log(0.05), np.log(20.0))))
        c = rng.uniform(-1, 1, size=N) * 10.0 ** rng.uniform(-2, 2, size=N)
        J, S = exact_cost(N, r, np.array([[T]]), c.reshape(1, 1, 1, N))
        Q = oracle.cost_matrix(N, r, T)
        want = 0.5 * float(c @ Q @ c)
        assert abs(want - float(J[0])) <= (4 * N * N + 64) * 2.0 ** -53 * float(S[0]), (trial, N, r, T)
        assert float(S[0]) >= abs(float(J[0]))
    # c = t^r / r! on a segment of length T: the r-th derivative is 1, so the cost is 0.5 * 2 * T / 1 * (r!)^2 / (r!)^2
    for N, r in ((10, 4), (2, 0), (12, 5)):
        c = np.zeros((1, 1, 1, N))
        c[0, 0, 0, r] = 1.0 / math.factorial(r)
        J, _ = exact_cost(N, r, np.array([[1.5]]), c)
        assert J[0] == Fraction(3, 2) * Fraction(c[0, 0, 0, r]) ** 2 * math.factorial(r) ** 2


COST_SHAPES = [  # the eight cost_kernel<N, r> specialisations, then shapes of the generic cost_kernel<0, 0>
    (10, 4), (10, 3), (10, 2), (8, 3), (12, 5), (12, 4), (6, 2), (4, 1),
    (12, 3), (8, 1), (2, 0)]
COST_SIZES = [  # K, D, B: K*D below 256 (17 trajectories per block pass, B not a multiple) and above (one per block)
    pytest.param(5, 3, 40, id="K5D3-B40"),
    pytest.param(86, 3, 3, id="K86D3-B3"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("K,D,B", COST_SIZES)
@pytest.mark.parametrize("N,r", COST_SHAPES, ids=["N{}r{}".format(*s) for s in COST_SHAPES])
def test_compute_cost_vs_exact_rational(solver, N, r, K, D, B):
    """compute_cost on seeded random coefficients and log-uniform segment times: within a forward-error bound of the
    exact value (any O(1) slip in the formula -- an index of 1/k, a factor of T, B(r, a) -- fails it)."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(100 * N + 10 * r + K)
    times = np.exp(rng.uniform(np.log(0.05), np.log(20.0), size=(B, K)))
    coeffs = rng.uniform(-1, 1, size=(B, K, D, N)) * 10.0 ** rng.uniform(-2, 2, size=(B, K, D, N))
    prob = m.Problem(N, r, K, D)
    cost = solver.compute_cost(prob, torch.from_numpy(times).cuda(), torch.from_numpy(coeffs).cuda())
    torch.cuda.synchronize()
    cost = cost.cpu().numpy()
    J, S = exact_cost(N, r, times, coeffs)
    exact = np.array([float(x) for x in J])
    scale = np.array([float(x) for x in S])
    err = np.abs(cost - exact)
    bound = cost_bound(N, r, K, D) * scale
    assert (err <= bound).all(), (f"N={N} r={r} K={K} D={D}: |cost - exact| / S = {(err / scale).max():.3e} "
                                  f"> {cost_bound(N, r, K, D):.3e}")
