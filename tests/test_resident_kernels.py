"""The resident waypoint kernels against binary128, each case proving by name which instantiation ran.

  1. v3 (twisted_tmem_kernel<N, R, D>) at all 17 registry shapes, plain and fused Nfabian;
  2. v4 (twisted_tmem_v4_kernel) and v5 (twisted_tmem_v5_kernel: double buffered, single buffered with and without
     the EARLY refill) at their 6 shapes, plain and fused, bitwise equal to each other and to the chunked kernel K3;
  3. the cost-only twisted_tmem_kernel<N, R, D, false, true> behind cost_gradient_mellinger at its 7 shapes;
  4. rows solved alone and split batches bitwise equal to the whole batch, with every warp running >= 3 tiles;
  5. bad segment times (0, -0, -1, NaN, +inf, -inf) in every waypoint kernel family, the banded kernel,
     backsub_kernel and the fused entry.

launch_solve falls back silently when a forced kernel is not eligible (B % 16, alignment, resident CTAs), so every
case lists the CUDA kernels the call launched, as recorded by torch.profiler (CUPTI traces the library's launches
too), and asserts that exactly the intended instantiation ran and no fallback.
"""
import contextlib
import re
import time

import numpy as np
import pytest

from test_gpu_parity import check_parity, global_rel_err
from test_large_k import (WAYPOINT_SHAPES, banded_solve, mellinger_reference, mellinger_times, oracle_solve,
                          rel_err_free, same_bits, waypoint_fixture)

# The real default of every option (mtg_handle in csrc/mtg_capi.cu): TMA_INPUTS is 2, and 0 turns v5 off.
DEFAULT_OPTIONS = dict(WAYPOINT_VARIANT=0, CTAS_PER_SM=0, DYNAMIC_TILES=0, CHUNK_BLOCKS=0, GENERIC_VARIANT=0,
                       MELLINGER_UNFUSED=0, TMA_INPUTS=2, EARLY_REFILL=0, CHUNK_WARPS=0, L2_HINTS=0)

V45_SHAPES = [(10, 4, 3), (8, 3, 3), (10, 4, 1), (10, 3, 3), (10, 2, 3), (12, 5, 3)]  # kV4Kernels / kV5Kernels
MINB = {(8, 3, 3): 3}  # __launch_bounds__ min blocks of the v4 / v5 instantiations (2 elsewhere)
COST_SHAPES = [(10, 4, 3), (10, 4, 1), (10, 4, 4), (10, 3, 3), (10, 2, 3), (8, 3, 3), (12, 5, 3)]  # kCostKernels

# K values chosen by stepping K = 2, 3, ... on an H100 80GB HBM3 (132 SMs) and reading the profiler (which kernel each
# launch ran).  The largest K <= 8 at which a forced v3 still launches v3, plain and fused (beyond it two CTAs per SM
# no longer fit: the plain entry runs K3, the fused one the pack fallback):
V3_KMAX = {(10, 4, 3): 6, (10, 4, 1): 8, (10, 4, 2): 8, (10, 4, 4): 6, (10, 3, 3): 6, (10, 3, 1): 8, (10, 2, 3): 6,
           (10, 2, 1): 8, (8, 3, 3): 8, (8, 3, 1): 8, (8, 3, 2): 8, (8, 3, 4): 8, (12, 5, 3): 6, (12, 5, 1): 8,
           (12, 5, 4): 4, (6, 2, 3): 8, (6, 2, 1): 8}
# The largest K at which a forced v4 still fits one CTA per SM, plain and fused (K3 / the pack fallback beyond):
V4_KBIG = {(10, 4, 3): 14, (8, 3, 3): 20, (10, 4, 1): 28, (10, 3, 3): 14, (10, 2, 3): 14, (12, 5, 3): 12}
# The largest K at which default routing with TMA_INPUTS = 1 takes v5 (two tile buffers), plain and fused; at K = 5
# five of the six shapes already take one buffer:
V5_DOUBLE_KMAX = {(10, 4, 3): 4, (8, 3, 3): 3, (10, 4, 1): 6, (10, 3, 3): 4, (10, 2, 3): 4, (12, 5, 3): 3}
# K values at which a forced v5 (variant 6) takes one tile buffer and the EARLY refill.  The EARLY instantiation runs
# only where one buffer admits more resident CTAs than two, so the plain and the fused entry (whose tiles hold
# positions) reach it at different K: (10, 4, 3) plain at K = 13, 14 only, fused at K = 15, 16 only.
V5_EARLY_PLAIN_K = {(10, 4, 3): [13, 14], (8, 3, 3): [9, 17, 21], (10, 4, 1): [7, 13, 28], (10, 3, 3): [13, 14],
                    (10, 2, 3): [13, 14], (12, 5, 3): [10, 11, 12]}
V5_EARLY_FUSED_K = {(10, 4, 3): [15, 16], (8, 3, 3): [9, 10, 22], (10, 4, 1): [13, 14, 28], (10, 3, 3): [15, 16],
                    (10, 2, 3): [15, 16], (12, 5, 3): [11, 12]}
# The largest K at which cost_gradient_mellinger still takes the fused cost-only kernel:
COST_KMAX = {(10, 4, 3): 6, (10, 4, 1): 14, (10, 4, 4): 6, (10, 3, 3): 6, (10, 2, 3): 6, (8, 3, 3): 10, (12, 5, 3): 6}


def _sid(shape):
    return "N{}r{}D{}".format(*shape)


# ---------------------------------------------------------------------------------------------------------------------
# Which kernels ran

_NAME = re.compile(r"mtg::(\w+<[^<>]*>|\w+)")


def kernel_id(base, *args):
    """'base<a,b,...>' as the demangled name shows it with the whitespace removed (bools as true / false)"""
    return base + "<" + ",".join(str(a).lower() if isinstance(a, bool) else str(a) for a in args) + ">"


def v3_id(N, r, D, fused=False, cost=False):
    return kernel_id("twisted_tmem_kernel", N, r, D, fused, cost)


def v4_id(N, r, D, fused=False):
    return kernel_id("twisted_tmem_v4_kernel", N, r, D, fused, 3, MINB.get((N, r, D), 2))


def v5_id(N, r, D, fused=False, early=0):
    return kernel_id("twisted_tmem_v5_kernel", N, r, D, MINB.get((N, r, D), 2), fused, early)


def k3_id(N, r, D):
    return kernel_id("twisted_chunked_kernel", N, r, D, 3, 1)  # ring depth 3, one warp per CTA (auto)


# Host time kept between the start of a profiler session and the call, and between the call and the end.  The trace
# keeps only device activity inside the session's window, which is measured on the host clock: a short kernel right at
# an edge of the window can fall outside it.
PROFILE_PAD_S = 0.01
_last_events = []


def _profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(PROFILE_PAD_S)
        result = fn()
        torch.cuda.synchronize()
        time.sleep(PROFILE_PAD_S)
    ids = []
    _last_events[:] = [re.sub(r"\s+", "", ev.name)[:80] for ev in prof.events()]
    for name in _last_events:
        found = _NAME.search(name)
        if found:
            ids.append(found.group(1))
    return result, ids


def _matches(ids, want, helpers):
    solves = [k for k in ids if k not in helpers]
    return want(solves) if callable(want) else solves == [want]


# Attempts per profiled call.  Now and then a profiler session came back without the kernel record of its call (in 2 to
# 3 of about 1300 sessions per run on the H100, before the padding above), so a call whose list does not show `want` is
# run again.  Every call profiled here is idempotent -- the same inputs, options and output buffers give the same
# bits -- and the route is a deterministic function of shapes, alignment and options: a real fallback fails every
# attempt.
PROFILE_ATTEMPTS = 3


def launched_kernels(fn, want=None, helpers=()):
    """Run fn() under the CUDA profiler -> (fn's result, ids of the project's kernels it launched, in order).  With
    `want` (a kernel id, or a predicate on the ids outside `helpers`) the call is repeated while the list does not
    match, PROFILE_ATTEMPTS times in all."""
    for _ in range(PROFILE_ATTEMPTS):
        result, ids = _profile(fn)
        if want is None or _matches(ids, want, helpers):
            break
    return result, ids


def assert_ran(ids, want, label, helpers=()):
    """exactly one launch, of `want` (or one that the predicate `want` accepts), besides the named helper kernels: no
    fallback kernel ran"""
    assert _matches(ids, want, helpers), f"{label}: launched {ids}, expected {want} (trace: {_last_events})"


@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (no CPU fallback exists)")
    import mav_trajectory_generation_b200 as m
    s = m.Solver(0)
    for name, value in DEFAULT_OPTIONS.items():
        s.set_option(getattr(m.capi, "OPT_" + name), value)
    yield s
    s.close()


@pytest.fixture(scope="module")
def kernels(solver, oracle):
    """launched_kernels, checked once: a forced K3 launch (variant 5 has no fallback) must show up by name."""
    import torch
    import mav_trajectory_generation_b200 as m
    pos, times = oracle.make_waypoint_batch(4, 3, 5, base_seed=7)
    prob = m.Problem(10, 4, 4, 3)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(oracle.waypoint_d_fixed(10, pos)).cuda()
    with options(solver, WAYPOINT_VARIANT=5):
        _, ids = launched_kernels(lambda: solver.solve_linear(prob, t_d, f_d), want=k3_id(10, 4, 3))
    assert ids == [k3_id(10, 4, 3)], f"the profiler does not list the library's kernels: {ids}"
    return launched_kernels


@contextlib.contextmanager
def options(solver, **opts):
    """Set MTG_OPT_<name> options for the block; each goes back to its real default afterwards."""
    import mav_trajectory_generation_b200 as m
    try:
        for name, value in opts.items():
            solver.set_option(getattr(m.capi, "OPT_" + name), value)
        yield
    finally:
        for name in opts:
            solver.set_option(getattr(m.capi, "OPT_" + name), DEFAULT_OPTIONS[name])


def solve(solver, kernels, prob, t_d, f_d, coeffs=None, want=None, **opts):
    """solve_linear under the profiler -> (coeffs, d_free, status, kernel ids).  Outputs start as NaN / -1, so that an
    entry the kernel never writes cannot pass a comparison.  `want`: as launched_kernels."""
    import torch
    B = t_d.shape[0]
    if coeffs is None:
        coeffs = torch.full((B, prob.K, prob.D, prob.N), float("nan"), dtype=torch.float64, device="cuda")
    dfree = torch.full((B, prob.D, max(prob.n_free, 1)), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    with options(solver, **opts):
        _, ids = kernels(lambda: solver.solve_linear(prob, t_d, f_d, coeffs=coeffs, d_free=dfree, status=status),
                         want=want)
    return coeffs.cpu().numpy(), dfree.cpu().numpy(), status.cpu().numpy(), ids


def solve_fused(solver, kernels, N, r, pos, want=None, **opts):
    """solve_waypoints_nfabian (v_max 3, a_max 5, magic 6.5: the fixture's) under the profiler
    -> (coeffs, seg_times_out, status, kernel ids)"""
    import torch
    B, K1, D = pos.shape
    coeffs = torch.full((B, K1 - 1, D, N), float("nan"), dtype=torch.float64, device="cuda")
    t_out = torch.full((B, K1 - 1), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    p_d = torch.from_numpy(np.ascontiguousarray(pos)).cuda()
    with options(solver, **opts):
        _, ids = kernels(lambda: solver.solve_waypoints_nfabian(N, r, p_d, 3.0, 5.0, 6.5, coeffs=coeffs,
                                                                seg_times_out=t_out, status=status),
                         want=want)
    return coeffs.cpu().numpy(), t_out.cpu().numpy(), status.cpu().numpy(), ids


def to_dev(*arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


# ---------------------------------------------------------------------------------------------------------------------
# Shared checks

# Parametrisations where rule 2 of check_parity does not hold, on the 1-D (10, 4, 1) fixtures as in SWEEP_LOSS_CASES of
# test_large_k: one trajectory lands 1.04e-10 (v4, K = 8) and 1.22e-10 (fused v5, K = 14) from the reference-order
# oracle where the oracle is 8.4e-11 from exact, just under rule 2's 0.9e-10, while rule 1 holds.  There each
# trajectory is held to the bound of check_parity_or_sweep_loss, max(2e-10, 2 * err(oracle), 4 * err(banded kernel)),
# and the test also asserts that the exact solution moves by less than 1e-13 when every segment time moves by one ulp:
# the digits are lost to fp64 elimination, not to an ill-posed fixture.
RESIDENT_LOSS_CASES = {("v4", 10, 4, 1, 8), ("v5 early fused", 10, 4, 1, 14)}


def check_parity_or_loss(oracle, case, N, r, times, dfix, out, ref, exact, banded, label):
    """check_parity, or on a RESIDENT_LOSS_CASES parametrisation the bounded rule described there (`banded`: a thunk
    returning the banded generic kernel's result on the same inputs)"""
    if case not in RESIDENT_LOSS_CASES:
        check_parity(out, ref, exact, label)
        return
    moved = oracle.exact_solve_batch(N, r, np.nextafter(times, np.inf), dfix)
    e_mv = global_rel_err(moved, exact).max()
    gen = banded()
    assert np.isfinite(gen).all(), label
    e_ge, e_oe, e_be = global_rel_err(out, exact), global_rel_err(ref, exact), global_rel_err(gen, exact)
    b = int(np.argmax(e_ge))
    print(f"{label}: CUDA vs exact {e_ge[b]:.3e}, oracle {e_oe[b]:.3e}, banded kernel {e_be[b]:.3e}, exact moves "
          f"{e_mv:.1e} under one-ulp times")
    assert e_mv <= 1e-13, f"{label}: the exact solution moves by {e_mv:.3e} under one-ulp changes of the times"
    bad = e_ge > np.maximum(2e-10, np.maximum(2.0 * e_oe, 4.0 * e_be))
    assert not bad.any(), (f"{label}: CUDA vs exact {e_ge[bad].max():.3e} on trajectory {int(np.argmax(bad))} "
                           f"(oracle {e_oe[np.argmax(bad)]:.3e}, banded generic kernel {e_be[np.argmax(bad)]:.3e})")


def check_exact(oracle, N, r, pos, times, sd, ed, dfix, out, dfree, status, times_kind, label, case=None,
                banded=None):
    """status 0, finite outputs, check_parity (or check_parity_or_loss for `case`) against binary128 and the
    reference-order oracle, and d_free against the exact d_free under the rule of
    test_chunked_kernel_every_specialisation"""
    assert (status == 0).all(), (label, status)
    assert np.isfinite(out).all() and np.isfinite(dfree).all(), label
    exact, exact_free, _ = oracle.exact_solve_batch(N, r, times, dfix, want_free=True)
    ref, ref_free = oracle_solve(oracle, N, r, pos, times, sd, ed)
    check_parity_or_loss(oracle, case, N, r, times, dfix, out, ref, exact, banded, label)
    e_f, e_of = rel_err_free(dfree, exact_free), rel_err_free(ref_free, exact_free)
    flat = times_kind == "nfabian" and N <= 10
    bad = e_f > (1e-9 if flat else np.maximum(1e-9, 2.0 * e_of))
    assert not bad.any(), f"{label}: d_free vs exact {e_f[bad].max():.3e} (oracle vs exact {e_of[bad].max():.3e})"


def check_same(a, b, label, what):
    """(coeffs, d_free, status) triples bitwise equal"""
    assert same_bits(a[0], b[0]), f"{label}: coefficients differ from {what}"
    assert same_bits(a[1], b[1]), f"{label}: d_free differs from {what}"
    assert same_bits(a[2], b[2]), f"{label}: status differs from {what}"


def check_k3(solver, kernels, prob, t_d, f_d, res, label):
    """bitwise equal to the chunked kernel K3, which runs the same fold-carry arithmetic"""
    N, r, D = prob.N, prob.r, prob.D
    o, f, s, ids = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=5, want=k3_id(N, r, D))
    assert_ran(ids, k3_id(N, r, D), label + " K3")
    check_same(res, (o, f, s), label, "K3")


def check_fused(solver, kernels, oracle, N, r, pos, host_times, want_fused, want_plain, label, plain_opts=None,
                case=None, **opts):
    """The fused entry: exactly `want_fused` ran, seg_times_out within 4e-16 of the host Nfabian times, the plain entry
    (`want_plain`, run with `plain_opts`, default the same options) on the kernel's own times and the packed d_fixed
    gives the same bits, and the result passes check_parity."""
    import mav_trajectory_generation_b200 as m
    B, K1, D = pos.shape
    out, t_out, status, ids = solve_fused(solver, kernels, N, r, pos, want=want_fused, **opts)
    assert_ran(ids, want_fused, label)
    assert (status == 0).all(), (label, status)
    assert np.isfinite(out).all(), label
    np.testing.assert_allclose(t_out, host_times, rtol=4e-16, atol=0)  # device exp() vs glibc exp()
    dfix = oracle.waypoint_d_fixed(N, pos)  # what nfabian_pack_kernel packs: positions, zero end derivatives
    prob = m.Problem(N, r, K1 - 1, D)
    t_d, f_d = to_dev(t_out, dfix)
    o2, _, s2, ids2 = solve(solver, kernels, prob, t_d, f_d, want=want_plain,
                            **(opts if plain_opts is None else plain_opts))
    assert_ran(ids2, want_plain, label + " plain entry")
    assert same_bits(out, o2), f"{label}: fused entry differs from the plain entry on its own inputs"
    assert same_bits(status, s2), label
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, t_out, n_threads=oracle.hardware_threads())
    check_parity_or_loss(oracle, case, N, r, t_out, dfix, out, ref, oracle.exact_solve_batch(N, r, t_out, dfix),
                         lambda: banded_solve(solver, prob, t_d, f_d), label)
    return out


def fixture(oracle, N, r, K, D, B, times_kind, seed):
    import mav_trajectory_generation_b200 as m
    pos, times, sd, ed = waypoint_fixture(oracle, N, K, D, B, times_kind, seed)
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_WAYPOINT
    return prob, pos, times, sd, ed, dfix


# ---------------------------------------------------------------------------------------------------------------------
# 1. v3

V3_CASES = [  # K (None: V3_KMAX; capped at V3_KMAX: (12, 5, 4) runs v3 up to K = 4 only), B, segment times
    pytest.param(2, 1, "nfabian", id="K2-B1"),
    pytest.param(3, 33, "mixed", id="K3-B33"),      # partial 16-row box
    pytest.param(5, 70, "nfabian", id="K5-B70"),    # partial 64-row CTA tile
    pytest.param(None, 130, "mixed", id="Kmax-B130"),
]


def _v3_k(shape, K):
    return V3_KMAX[shape] if K is None else min(K, V3_KMAX[shape])


@pytest.mark.gpu
@pytest.mark.parametrize("K,B,times_kind", V3_CASES)
@pytest.mark.parametrize("N,r,D", WAYPOINT_SHAPES, ids=[_sid(s) for s in WAYPOINT_SHAPES])
def test_v3_every_shape(solver, kernels, oracle, N, r, D, K, B, times_kind):
    """Forced v3 at every registry shape: the instantiation by name, check_parity and d_free against binary128, and
    rounding-level agreement with K3 (v3 adds the end-derivative carry of the first sweep step first, the fold-carry
    kernels last): on the Nfabian fixture within the bounds of test_tma_input_kernel_bitwise_vs_resident.  On
    log-uniform times the one reordered addition is amplified up to 1e-8 (N = 10) and 8e-3 (N = 12, where both kernels
    are that far from exact too), so there the median bound stays and each trajectory's difference is held to the two
    kernels' own distances from exact: max(1e-10, 2 * (err(v3) + err(K3)))."""
    K = _v3_k((N, r, D), K)
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, times_kind, 50000 + 1000 * N + 100 * r + 10 * D + K)
    t_d, f_d = to_dev(times, dfix)
    label = f"v3 N={N} r={r} D={D} K={K} B={B} {times_kind}"
    out, dfree, status, ids = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=3, want=v3_id(N, r, D))
    assert_ran(ids, v3_id(N, r, D), label)
    check_exact(oracle, N, r, pos, times, sd, ed, dfix, out, dfree, status, times_kind, label)
    o3, _, _, ids = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=5, want=k3_id(N, r, D))
    assert_ran(ids, k3_id(N, r, D), label + " K3")
    dv = global_rel_err(out, o3)
    assert np.median(dv) <= (1e-14 if N < 12 else 1e-12), f"{label}: v3 vs K3 median {np.median(dv):.3e}"
    if times_kind == "nfabian":
        bound = 1e-10 if N < 12 else 1e-7
    else:
        exact = oracle.exact_solve_batch(N, r, times, dfix)
        bound = np.maximum(1e-10, 2.0 * (global_rel_err(out, exact) + global_rel_err(o3, exact)))
    assert (dv <= bound).all(), f"{label}: v3 vs K3 {dv.max():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("K,B", [pytest.param(2, 1, id="K2-B1"), pytest.param(5, 37, id="K5-B37")])
@pytest.mark.parametrize("N,r,D", WAYPOINT_SHAPES, ids=[_sid(s) for s in WAYPOINT_SHAPES])
def test_v3_fused_every_shape(solver, kernels, oracle, N, r, D, K, B):
    """solve_waypoints_nfabian with variant 3: the fused v3 instantiation, no pack fallback."""
    K = _v3_k((N, r, D), K)
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=51000 + 100 * N + 10 * r + D)
    check_fused(solver, kernels, oracle, N, r, pos, times, v3_id(N, r, D, fused=True), v3_id(N, r, D),
                f"v3 fused N={N} r={r} D={D} K={K} B={B}", WAYPOINT_VARIANT=3)


# ---------------------------------------------------------------------------------------------------------------------
# 2. v4 and v5: the fold-carry family

V4_CASES = [  # K (None: V4_KBIG), B, segment times
    pytest.param(2, 1, "nfabian", id="K2-B1"),
    pytest.param(3, 33, "mixed", id="K3-B33"),
    pytest.param(8, 70, "nfabian", id="K8-B70"),
    pytest.param(None, 45, "mixed", id="Kbig-B45"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("K,B,times_kind", V4_CASES)
@pytest.mark.parametrize("N,r,D", V45_SHAPES, ids=[_sid(s) for s in V45_SHAPES])
def test_v4(solver, kernels, oracle, N, r, D, K, B, times_kind):
    """Forced v4: by name, against binary128, bitwise equal to K3; the fused entry on the Nfabian fixture."""
    K = V4_KBIG[(N, r, D)] if K is None else K
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, times_kind, 52000 + 1000 * N + 100 * r + 10 * D + K)
    t_d, f_d = to_dev(times, dfix)
    label = f"v4 N={N} r={r} D={D} K={K} B={B} {times_kind}"
    res = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=4, want=v4_id(N, r, D))
    assert_ran(res[3], v4_id(N, r, D), label)
    check_exact(oracle, N, r, pos, times, sd, ed, dfix, *res[:3], times_kind, label, case=("v4", N, r, D, K),
                banded=lambda: banded_solve(solver, prob, t_d, f_d))
    check_k3(solver, kernels, prob, t_d, f_d, res[:3], label)
    pos_f, times_f = oracle.make_waypoint_batch(K, D, B, base_seed=53000 + 100 * N + 10 * K + D)
    check_fused(solver, kernels, oracle, N, r, pos_f, times_f, v4_id(N, r, D, fused=True), v4_id(N, r, D),
                f"v4 fused N={N} r={r} D={D} K={K} B={B}", WAYPOINT_VARIANT=4)


V5_DOUBLE_CASES = [  # K (None: V5_DOUBLE_KMAX), B (a multiple of 16), segment times
    pytest.param(2, 16, "nfabian", id="K2-B16"),
    pytest.param(3, 48, "mixed", id="K3-B48"),
    pytest.param(None, 80, "nfabian", id="Kmax-B80"),   # partial 64-row CTA tile
]


@pytest.mark.gpu
@pytest.mark.parametrize("K,B,times_kind", V5_DOUBLE_CASES)
@pytest.mark.parametrize("N,r,D", V45_SHAPES, ids=[_sid(s) for s in V45_SHAPES])
def test_v5_double_buffered(solver, kernels, oracle, N, r, D, K, B, times_kind):
    """Default routing with TMA_INPUTS = 1 takes v5 only with two tile buffers, so the v5 name proves double
    buffering.  Against binary128, bitwise equal to v4 and K3; the fused entry equal to the plain one."""
    K = V5_DOUBLE_KMAX[(N, r, D)] if K is None else K
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, times_kind, 54000 + 1000 * N + 100 * r + 10 * D + K)
    t_d, f_d = to_dev(times, dfix)
    label = f"v5 double N={N} r={r} D={D} K={K} B={B} {times_kind}"
    res = solve(solver, kernels, prob, t_d, f_d, TMA_INPUTS=1, want=v5_id(N, r, D))
    assert_ran(res[3], v5_id(N, r, D), label)
    check_exact(oracle, N, r, pos, times, sd, ed, dfix, *res[:3], times_kind, label)
    o4 = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=4, want=v4_id(N, r, D))
    assert_ran(o4[3], v4_id(N, r, D), label + " v4")
    check_same(res[:3], o4[:3], label, "v4")
    check_k3(solver, kernels, prob, t_d, f_d, res[:3], label)
    pos_f, times_f = oracle.make_waypoint_batch(K, D, B, base_seed=55000 + 100 * N + 10 * K + D)
    check_fused(solver, kernels, oracle, N, r, pos_f, times_f, v5_id(N, r, D, fused=True), v5_id(N, r, D),
                f"v5 double fused N={N} r={r} D={D} K={K} B={B}", TMA_INPUTS=1)


V5_EARLY_PLAIN_CASES = [(shape, K) for shape, Ks in V5_EARLY_PLAIN_K.items() for K in Ks]
V5_EARLY_FUSED_CASES = [(shape, K) for shape, Ks in V5_EARLY_FUSED_K.items() for K in Ks]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,K", V5_EARLY_PLAIN_CASES, ids=[f"{_sid(s)}-K{K}" for s, K in V5_EARLY_PLAIN_CASES])
def test_v5_single_buffer_early_refill(solver, kernels, oracle, shape, K):
    """Forced v5 (variant 6) where one tile buffer fits: the EARLY instantiation, and with EARLY_REFILL = -1 the
    instantiation without it on the same inputs (the buffer count does not depend on the option, so that one runs
    single buffered too).  Against binary128; EARLY, no EARLY, v4 (where it fits) and K3 bitwise equal."""
    N, r, D = shape
    B, times_kind = (32, "nfabian") if K % 2 else (80, "mixed")
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, times_kind, 56000 + 1000 * N + 100 * r + 10 * D + K)
    t_d, f_d = to_dev(times, dfix)
    label = f"v5 early N={N} r={r} D={D} K={K} B={B} {times_kind}"
    res = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=6, want=v5_id(N, r, D, early=2))
    assert_ran(res[3], v5_id(N, r, D, early=2), label)
    check_exact(oracle, N, r, pos, times, sd, ed, dfix, *res[:3], times_kind, label)
    late = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=6, EARLY_REFILL=-1, want=v5_id(N, r, D))
    assert_ran(late[3], v5_id(N, r, D), label + " no early refill")
    check_same(res[:3], late[:3], label, "v5 without the early refill")
    if K <= V4_KBIG[shape]:
        o4 = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=4, want=v4_id(N, r, D))
        assert_ran(o4[3], v4_id(N, r, D), label + " v4")
        check_same(res[:3], o4[:3], label, "v4")
    check_k3(solver, kernels, prob, t_d, f_d, res[:3], label)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,K", V5_EARLY_FUSED_CASES, ids=[f"{_sid(s)}-K{K}" for s, K in V5_EARLY_FUSED_CASES])
def test_v5_fused_single_buffer_early_refill(solver, kernels, oracle, shape, K):
    """The fused entry forced to v5 where one tile buffer fits: the fused EARLY instantiation, equal bit for bit to the
    fused instantiation without it and to the plain entry on the kernel's own times and the packed d_fixed -- the plain
    EARLY instantiation where it runs at this K, else K3, which runs the same fold-carry arithmetic."""
    N, r, D = shape
    B = 48 if K % 2 else 144
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=57000 + 100 * N + 10 * K + D)
    label = f"v5 early fused N={N} r={r} D={D} K={K} B={B}"
    if K in V5_EARLY_PLAIN_K[shape]:
        plain_id, plain_opts = v5_id(N, r, D, early=2), dict(WAYPOINT_VARIANT=6)
    else:
        plain_id, plain_opts = k3_id(N, r, D), dict(WAYPOINT_VARIANT=5)
    case = ("v5 early fused", N, r, D, K)
    early = check_fused(solver, kernels, oracle, N, r, pos, times, v5_id(N, r, D, fused=True, early=2), plain_id,
                        label, plain_opts=plain_opts, case=case, WAYPOINT_VARIANT=6)
    no_early = check_fused(solver, kernels, oracle, N, r, pos, times, v5_id(N, r, D, fused=True), plain_id,
                           label + " no early refill", plain_opts=plain_opts, case=case, WAYPOINT_VARIANT=6,
                           EARLY_REFILL=-1)
    assert same_bits(early, no_early), label


# ---------------------------------------------------------------------------------------------------------------------
# 3. The cost-only kernel

COST_CASES = [  # K (None: COST_KMAX), B, segment times
    pytest.param(2, 5, "nfabian", id="K2"),
    pytest.param(5, 7, "nfabian", id="K5"),
    pytest.param(None, 3, "nfabian", id="Kmax"),
    pytest.param(5, 5, "clamp", id="K5-clamp"),  # 0.12 s segments: t - 0.1 / (K-1) < 0.1 hits the lower bound
]


# (12, 5, 3) on the clamp fixture: the cost-only kernel's cost is 4.6e-8 from the binary128 cost, where the unfused path
# (expand + K3 + cost_kernel on the coefficients) is 1.6e-10 from it (H100 80GB HBM3).  The cost-only kernel evaluates
# 0.5 u^T H(1;r) u on the scaled vertex derivatives u, and at N = 12, r = 5 on 0.12 s segments that sum of
# alternating-sign terms cancels far more than the coefficient form.  The loss is in the formulation, not in an index
# or a factor (each of those moves the cost by O(1)); until the kernel evaluates the cost from coefficients, this case
# is held to 1e-7, the unfused path to 1e-9, and the two paths to agree within the sum.
COST_LOSS_CASES = {(12, 5, 3, "clamp")}


@pytest.mark.gpu
@pytest.mark.parametrize("K,B,times_kind", COST_CASES)
@pytest.mark.parametrize("N,r,D", COST_SHAPES, ids=[_sid(s) for s in COST_SHAPES])
def test_cost_only_kernel(solver, kernels, oracle, N, r, D, K, B, times_kind):
    """cost_gradient_mellinger on its default path runs the fused cost-only kernel and the gradient kernel, nothing
    else: the cost within 1e-10 relative of the binary128 cost (COST_LOSS_CASES aside), the gradient within 1e-6 of the
    binary128 forward differences on the same expanded time vectors, and the unfused path agreeing as in
    test_batched_mellinger_gradient."""
    import mav_trajectory_generation_b200 as m
    K = COST_KMAX[(N, r, D)] if K is None else K
    pos, times, sd, ed = waypoint_fixture(oracle, N, K, D, B, "nfabian", 58000 + 1000 * N + 100 * r + 10 * D + K)
    if times_kind == "clamp":
        times[:, ::2] = 0.12
        assert (mellinger_times(times)[:, 1:] == 0.1).any()
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = to_dev(times, dfix)
    label = f"cost-only N={N} r={r} D={D} K={K} {times_kind}"
    want, helpers = v3_id(N, r, D, cost=True), ("mellinger_gradient_kernel",)
    (cost, grad), ids = kernels(lambda: solver.cost_gradient_mellinger(prob, t_d, f_d), want=want, helpers=helpers)
    assert_ran(ids, want, label, helpers=helpers)
    cost, grad = cost.cpu().numpy(), grad.cpu().numpy()
    with options(solver, MELLINGER_UNFUSED=1):
        (cost_u, grad_u), ids = kernels(lambda: solver.cost_gradient_mellinger(prob, t_d, f_d))
    assert v3_id(N, r, D, cost=True) not in ids, label
    cost_u, grad_u = cost_u.cpu().numpy(), grad_u.cpu().numpy()
    _, _, c_exact = oracle.exact_solve_batch(N, r, times, dfix, want_cost=True)
    e_c = np.abs(cost - c_exact) / np.abs(c_exact)
    e_u = np.abs(cost_u - c_exact) / np.abs(c_exact)
    print(f"{label}: cost vs exact {e_c.max():.2e} (unfused path {e_u.max():.2e})")
    bound, agree = 1e-10, 1e-8
    if (N, r, D, times_kind) in COST_LOSS_CASES:
        bound, agree = 1e-7, 1e-7 + 1e-9
        assert (e_u <= 1e-9).all(), f"{label}: unfused cost vs exact {e_u.max():.3e}"
    assert (e_c <= bound).all(), f"{label}: cost vs exact {e_c.max():.3e} (unfused path {e_u.max():.3e})"
    c_ref, g_ref = mellinger_reference(oracle, N, r, times, dfix)
    e_g = np.abs(grad - g_ref).max(axis=1) / np.maximum(np.abs(c_ref), np.abs(g_ref).max(axis=1))
    assert (e_g <= 1e-6).all(), f"{label}: gradient vs exact {e_g.max():.3e}"
    assert np.abs(cost_u - cost).max() <= agree * np.abs(cost).max(), label
    assert np.abs(grad_u - grad).max() <= 1e-6 * max(np.abs(cost).max(), np.abs(grad).max()), label


# ---------------------------------------------------------------------------------------------------------------------
# 4. Tile independence with many tiles per warp

def _many_tiles_batch():
    """rows for >= 3 16-row tiles per warp even at the 8 resident 4-warp CTAs per SM the launch code allows"""
    import torch
    return 3 * 16 * 4 * 8 * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("dyn", [1, 2], ids=["dynamic", "static"])
def test_v5_early_many_tiles_rows_alone_and_split(solver, kernels, oracle, dyn):
    """v5 single buffered with the EARLY refill, every warp running >= 3 tiles (mbarrier phases flip, the parking area
    is reused): the whole batch equals 16 scattered rows solved as one batch (v5 needs whole 16-row boxes) and a batch
    split at a 16-row box that is not a 64-row CTA tile boundary, bit for bit; dynamic and static tile assignment agree;
    sampled rows pass check_parity."""
    N, r, D = 10, 4, 1
    K = V5_EARLY_PLAIN_K[(N, r, D)][0]
    B = _many_tiles_batch()
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, "nfabian", 59000 + dyn)
    t_d, f_d = to_dev(times, dfix)
    want = v5_id(N, r, D, early=2)
    label = f"v5 early many tiles K={K} B={B} dyn={dyn}"
    whole = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=6, DYNAMIC_TILES=dyn, want=want)
    assert_ran(whole[3], want, label)
    assert (whole[2] == 0).all(), label
    other = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=6, DYNAMIC_TILES=3 - dyn, want=want)
    assert_ran(other[3], want, label)
    check_same(whole[:3], other[:3], label, "the other tile assignment")
    rng = np.random.RandomState(dyn)
    rows = np.concatenate([[0, B - 1, 16, 63, 64], rng.choice(np.arange(65, B - 1), 11, replace=False)])
    rng.shuffle(rows)
    t_r, f_r = to_dev(times[rows], dfix[rows])
    alone = solve(solver, kernels, prob, t_r, f_r, WAYPOINT_VARIANT=6, DYNAMIC_TILES=dyn, want=want)
    assert_ran(alone[3], want, label + " rows")
    check_same(alone[:3], tuple(x[rows] for x in whole[:3]), label, "the same rows in the whole batch")
    cut = 16 * 37
    parts = []
    for sl in (slice(0, cut), slice(cut, B)):
        t_p, f_p = to_dev(times[sl], dfix[sl])
        part = solve(solver, kernels, prob, t_p, f_p, WAYPOINT_VARIANT=6, DYNAMIC_TILES=dyn, want=want)
        assert_ran(part[3], want, label + " split")
        parts.append(part)
    check_same(tuple(np.concatenate([p[i] for p in parts]) for i in range(3)), whole[:3], label, "the split batch")
    sub = rows[:8]
    check_exact(oracle, N, r, pos[sub], times[sub], sd[sub], ed[sub], dfix[sub], *(x[sub] for x in whole[:3]),
                "nfabian", label)


@pytest.mark.gpu
def test_v4_dynamic_tiles_rows_alone_and_split(solver, kernels, oracle):
    """v4 with the dynamic tile counter and with static round-robin, every warp running >= 3 tiles: identical bits,
    and equal to rows solved alone (B = 1) and to a batch split inside a tile."""
    N, r, K, D = 8, 3, 4, 3
    B = _many_tiles_batch() + 5
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, B, "nfabian", 59100)
    t_d, f_d = to_dev(times, dfix)
    label = f"v4 many tiles B={B}"
    dyn = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=4, DYNAMIC_TILES=1, want=v4_id(N, r, D))
    assert_ran(dyn[3], v4_id(N, r, D), label)
    assert (dyn[2] == 0).all(), label
    static = solve(solver, kernels, prob, t_d, f_d, WAYPOINT_VARIANT=4, DYNAMIC_TILES=2, want=v4_id(N, r, D))
    assert_ran(static[3], v4_id(N, r, D), label)
    check_same(dyn[:3], static[:3], label, "static tiles")
    for b in (0, 17, B // 2 + 3, B - 1):
        t_r, f_r = to_dev(times[b:b + 1], dfix[b:b + 1])
        one = solve(solver, kernels, prob, t_r, f_r, WAYPOINT_VARIANT=4, DYNAMIC_TILES=1, want=v4_id(N, r, D))
        assert_ran(one[3], v4_id(N, r, D), label)
        check_same(one[:3], tuple(x[b:b + 1] for x in dyn[:3]), f"{label} row {b}", "the whole batch")
    cut = 16 * 1001 + 7
    parts = []
    for sl in (slice(0, cut), slice(cut, B)):
        t_p, f_p = to_dev(times[sl], dfix[sl])
        part = solve(solver, kernels, prob, t_p, f_p, WAYPOINT_VARIANT=4, DYNAMIC_TILES=1, want=v4_id(N, r, D))
        assert_ran(part[3], v4_id(N, r, D), label + " split")
        parts.append(part)
    check_same(tuple(np.concatenate([p[i] for p in parts]) for i in range(3)), dyn[:3], label, "the split batch")
    sub = np.arange(0, B, B // 8)
    check_exact(oracle, N, r, pos[sub], times[sub], sd[sub], ed[sub], dfix[sub], *(x[sub] for x in dyn[:3]),
                "nfabian", label)


# ---------------------------------------------------------------------------------------------------------------------
# 5. Bad segment times

BAD_VALUES = [0.0, -0.0, -1.0, float("nan"), float("inf"), float("-inf")]
BAD_IDS = ["zero", "negzero", "neg", "nan", "inf", "neginf"]
# B = 160: 16-row boxes of v5, 64-row CTA tiles of v3 / v4 / v5; five bad rows inside the first box, five across tiles
BAD_B = 160
BAD_ROWS = [1, 4, 9, 14, 15, 40, 77, 100, 131, 159]
STATUS_K = 6  # v3 still runs at (10, 4, 3); meeting vertex M = 3: segments 2 and 3 are either side of it
STATUS_FAMILIES = [  # name, options, output slice offset (1: an 8-byte aligned output takes the banded kernel)
    ("v1", dict(WAYPOINT_VARIANT=1), 0),
    ("v2", dict(WAYPOINT_VARIANT=2), 0),
    ("v3", dict(WAYPOINT_VARIANT=3), 0),
    ("v4", dict(WAYPOINT_VARIANT=4), 0),
    ("K3", dict(WAYPOINT_VARIANT=5), 0),
    ("v5", dict(WAYPOINT_VARIANT=6), 0),
    ("default", {}, 0),
    ("banded", {}, 1),
]


def _is_v5(N, r, D, fused):
    """predicate: one launch of the v5 instantiation of (N, r, D, fused), either EARLY"""
    return lambda ids: ids in ([v5_id(N, r, D, fused)], [v5_id(N, r, D, fused, early=2)])


def _bad_segments(K, i):
    """segment(s) that row number i of BAD_ROWS gets the bad value in: 0, either side of M, K-1, every segment"""
    M = (K + 1) // 2
    return [[0], [M - 1], [M], [K - 1], list(range(K))][i % 5]


def _status_solve(solver, kernels, prob, times, dfix, offset, opts, want):
    import torch
    B = times.shape[0]
    coeffs = None
    if offset:
        n = B * prob.K * prob.D * prob.N
        big = torch.full((n + 1,), float("nan"), dtype=torch.float64, device="cuda")
        coeffs = big[1:].view(B, prob.K, prob.D, prob.N)
        assert coeffs.data_ptr() % 16 == 8
    t_d, f_d = to_dev(times, dfix)
    return solve(solver, kernels, prob, t_d, f_d, coeffs=coeffs, want=want, **opts)


def _check_bad_rows(res, clean, bad, want, n_free, label):
    """STATUS_BAD_TIME on every bad row; every other row status 0, finite and the bits of the repaired batch; both
    batches ran the kernel `want` (as assert_ran)"""
    import mav_trajectory_generation_b200 as m
    out, dfree, status, ids = res
    assert_ran(clean[3], want, label + " repaired batch")
    assert_ran(ids, want, label)
    assert all(status[b] & m.STATUS_BAD_TIME for b in bad), f"{label}: status {status[bad]} on the bad rows"
    good = np.setdiff1d(np.arange(out.shape[0]), bad)
    assert (status[good] == 0).all() and (clean[2] == 0).all(), label
    assert np.isfinite(out[good]).all(), label
    assert same_bits(out[good], clean[0][good]), f"{label}: good rows differ from the repaired batch"
    if n_free:
        assert np.isfinite(dfree[good]).all(), label
        assert same_bits(dfree[good], clean[1][good]), f"{label}: good d_free differs from the repaired batch"


@pytest.mark.gpu
@pytest.mark.parametrize("value", BAD_VALUES, ids=BAD_IDS)
@pytest.mark.parametrize("family,opts,offset", STATUS_FAMILIES, ids=[f[0] for f in STATUS_FAMILIES])
def test_bad_segment_time_sets_status(solver, kernels, oracle, family, opts, offset, value):
    """A bad segment time in segment 0, either side of the meeting vertex, segment K-1 or every segment, on rows inside
    one 16-row box and across CTA tiles, sets STATUS_BAD_TIME in every waypoint kernel family and in the banded
    kernel; the other rows keep the bits of the same batch with the bad rows repaired.  +inf passes !(T > 0): before
    the shared bad_segment_time() check, the waypoint kernels reported it as STATUS_NOT_SPD and the banded kernel as
    nothing at all."""
    N, r, K, D = 10, 4, STATUS_K, 3
    prob, pos, times, sd, ed, dfix = fixture(oracle, N, r, K, D, BAD_B, "nfabian", 60000)
    want = {"v1": kernel_id("waypoint_solve_kernel", N, r, D), "v2": kernel_id("twisted_solve_kernel", N, r, D),
            "v3": v3_id(N, r, D), "v4": v4_id(N, r, D), "K3": k3_id(N, r, D), "banded": "generic_solve_kernel",
            # v5 forced, and the default route: v5 at this K, with or without the EARLY refill
            "v5": _is_v5(N, r, D, False), "default": _is_v5(N, r, D, False)}[family]
    clean = _status_solve(solver, kernels, prob, times, dfix, offset, opts, want)
    bad_times = times.copy()
    for i, b in enumerate(BAD_ROWS):
        bad_times[b, _bad_segments(K, i)] = value
    res = _status_solve(solver, kernels, prob, bad_times, dfix, offset, opts, want)
    _check_bad_rows(res, clean, BAD_ROWS, want, prob.n_free, f"{family} value={value}")


@pytest.mark.gpu
@pytest.mark.parametrize("value", BAD_VALUES, ids=BAD_IDS)
def test_bad_segment_time_backsub(solver, kernels, oracle, value):
    """K = 1 waypoint problems have no free constraint and take backsub_kernel: the same rule."""
    N, r, K, D = 10, 4, 1, 3
    import mav_trajectory_generation_b200 as m
    pos, times = oracle.make_waypoint_batch(K, D, BAD_B, base_seed=61000)
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_NOFREE
    clean = _status_solve(solver, kernels, prob, times, dfix, 0, {}, "backsub_kernel")
    bad_times = times.copy()
    bad_times[BAD_ROWS, 0] = value
    res = _status_solve(solver, kernels, prob, bad_times, dfix, 0, {}, "backsub_kernel")
    _check_bad_rows(res, clean, BAD_ROWS, "backsub_kernel", prob.n_free, f"backsub value={value}")


@pytest.mark.gpu
@pytest.mark.parametrize("value", [float("nan"), float("inf")], ids=["nan", "inf"])
def test_bad_waypoint_fused_entry_sets_status(solver, kernels, oracle, value):
    """The fused Nfabian entry computes the times from the waypoints: a NaN or +inf waypoint (first, middle, last
    vertex, every vertex) gives NaN / +inf times on its segments and STATUS_BAD_TIME; the other rows keep the bits of
    the repaired batch."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D = 10, 4, STATUS_K, 3
    pos, _ = oracle.make_waypoint_batch(K, D, BAD_B, base_seed=62000)

    def run(p):
        coeffs = torch.full((BAD_B, K, D, N), float("nan"), dtype=torch.float64, device="cuda")
        status = torch.full((BAD_B,), -1, dtype=torch.int32, device="cuda")
        p_d = torch.from_numpy(np.ascontiguousarray(p)).cuda()
        _, ids = kernels(lambda: solver.solve_waypoints_nfabian(N, r, p_d, 3.0, 5.0, 6.5, coeffs=coeffs,
                                                                status=status), want=want)
        return coeffs.cpu().numpy(), status.cpu().numpy(), ids

    want = _is_v5(N, r, D, True)  # the default route of the fused entry at this K
    clean = run(pos)
    assert_ran(clean[2], want, "fused repaired batch")
    bad_pos = pos.copy()
    vertices = [[0], [(K + 1) // 2], [K], list(range(K + 1))]
    for i, b in enumerate(BAD_ROWS):
        bad_pos[b, vertices[i % 4], i % D] = value
    out, status, ids = run(bad_pos)
    assert_ran(ids, want, "fused")
    assert all(status[b] & m.STATUS_BAD_TIME for b in BAD_ROWS), f"status {status[BAD_ROWS]} on the bad rows"
    good = np.setdiff1d(np.arange(BAD_B), BAD_ROWS)
    assert (status[good] == 0).all() and np.isfinite(out[good]).all()
    assert same_bits(out[good], clean[0][good]), "good rows differ from the repaired batch"
