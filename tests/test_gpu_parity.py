"""Parity of the CUDA path (through the C-ABI) against the CPU oracle on identical inputs.

Tolerance (north_star): max |p_gpu - p_ref| / max |p_ref| over one trajectory's K*D*N
coefficients <= 1e-10 for the BASELINE configurations (N=10 snap, N=8 jerk).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL = 1e-10          # north_star: coefficients within 1e-10 (global-relative) of the reference path
BASELINE_SHAPES = {(10, 4, 16, 3), (10, 4, 8, 3), (8, 3, 4, 3), (10, 4, 2, 3)}   # C3, C2, C4, C1


def global_rel_err(a, b):
    """per-trajectory max|a-b| / max|b|   (a, b: [B][K][D][N])"""
    B = a.shape[0]
    num = np.abs(a - b).reshape(B, -1).max(axis=1)
    den = np.abs(b).reshape(B, -1).max(axis=1)
    return num / den


def check_parity(out, ref, exact, label, baseline=False):
    """The parity contract, PER TRAJECTORY, same rule for every shape (no shape-dependent loosening):

      (1) err(CUDA, exact) <= max(1e-10, 2 * err(oracle, exact))
          `exact` is the binary128 solve of the same equations (oracle/exact.cpp): the CUDA path is within the
          north-star tolerance of the TRUE solution, except on trajectories where the reference-order fp64
          arithmetic itself is further than that (N = 12, 1-D fixtures with sub-second segments) -- there it must
          still be no worse than twice the reference-order error.
      (2) err(CUDA, oracle) <= 1e-10 unless the oracle itself is >= 0.9e-10 from exact on that trajectory (then
          the excursion is the reference-order rounding, shown by (1) holding at the same time).

    For the BASELINE shapes additionally the distribution is pinned: median <= 1e-13, 99th percentile <= 2e-12
    against exact.
    Returns the three per-trajectory error arrays."""
    e_ge = global_rel_err(out, exact)
    e_go = global_rel_err(out, ref)
    e_oe = global_rel_err(ref, exact)
    bound = np.maximum(TOL, 2.0 * e_oe)
    bad = e_ge > bound
    assert not bad.any(), (f"{label}: CUDA vs exact {e_ge[bad].max():.3e} on trajectory {int(np.argmax(bad))} "
                           f"(oracle vs exact there {e_oe[np.argmax(bad)]:.3e})")
    unexplained = (e_go > TOL) & (e_oe < 0.9 * TOL)
    assert not unexplained.any(), (f"{label}: CUDA vs oracle {e_go[unexplained].max():.3e} where the oracle is only "
                                   f"{e_oe[unexplained].max():.3e} from exact")
    if baseline and len(e_ge) >= 1000:
        assert np.median(e_ge) <= 1e-13 and np.quantile(e_ge, 0.99) <= 2e-12, \
            (label, float(np.median(e_ge)), float(np.quantile(e_ge, 0.99)))
    return e_ge, e_go, e_oe


def run_waypoint(solver, oracle, N, r, K, D, B, base_seed=1000, want_free=True, variant=0):
    import torch
    import mav_trajectory_generation_b200 as m
    solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, variant)
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=base_seed)
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, times, n_threads=oracle.hardware_threads())
    prob = m.Problem(N, r, K, D)
    dfix = oracle.waypoint_d_fixed(N, pos)
    t_d = torch.from_numpy(times).cuda()
    f_d = torch.from_numpy(dfix).cuda()
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    dfree = torch.zeros((B, D, max(prob.n_free, 1)), dtype=torch.float64, device="cuda") if want_free else None
    out = solver.solve_linear(prob, t_d, f_d, d_free=dfree, status=status)
    torch.cuda.synchronize()
    solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 0)
    return prob, pos, times, ref, out.cpu().numpy(), status.cpu().numpy(), (dfree.cpu().numpy() if want_free else None)


@pytest.mark.parametrize("name,N,r,K,D", [("C3", 10, 4, 16, 3), ("C2", 10, 4, 8, 3), ("C4", 8, 3, 4, 3)])
def test_baseline_configs_8192_fixtures_vs_exact_and_oracle(solver, oracle, name, N, r, K, D):
    """>= 8192 bit-exact fixture trajectories (createRandomVertices seeds 1000+b, Nfabian v=3 a=5) for each
    single-GPU BASELINE configuration, default kernel, under the check_parity contract (every trajectory, no
    sampling): within 1e-10 of the binary128 solve, within 1e-10 of the reference-order oracle except where the
    oracle itself is that far from exact (reference LIN_impl.h:338-379 in fp64 loses ~5 digits on short
    segments: ONE C2 trajectory of 8192 sits at 1.08e-10 from the oracle, and the oracle sits at 1.08e-10 from
    exact there), distribution median <= 1e-13 / p99 <= 2e-12, and the CUDA path closer to exact than the
    reference-order arithmetic on >= 99 % of the trajectories."""
    B = 8192
    prob, pos, times, ref, out, status, _ = run_waypoint(solver, oracle, N, r, K, D, B, want_free=False)
    assert (status == 0).all()
    exact = oracle.exact_solve_batch(N, r, times, oracle.waypoint_d_fixed(N, pos))
    e_ge, e_go, e_oe = check_parity(out, ref, exact, name, baseline=True)
    assert (e_ge <= e_oe).mean() >= 0.99
    print(f"{name}: CUDA-exact max {e_ge.max():.2e}  CUDA-oracle max {e_go.max():.2e} (#>1e-10: {(e_go > TOL).sum()})  "
          f"oracle-exact max {e_oe.max():.2e}")


@pytest.mark.parametrize("variant", [1, 2, 3, 4, 6])  # 1: thread/trajectory, 2: twisted, 3: + shared-memory state and TMA stores, 4: persistent, 6: + TMA inputs
@pytest.mark.parametrize("N,r,K,D,B", [
    (10, 4, 16, 3, 4096),   # C3 headline shape, >= 4096 bit-exact fixture trajectories (SURVEY.md 8d)
    (10, 4, 8, 3, 2048),    # C2
    (8, 3, 4, 3, 4096),     # C4
    (10, 4, 2, 3, 257),     # C1 shape, ragged batch: only the middle vertex
    (10, 4, 3, 3, 129),     # unbalanced halves (1 + 0 vertices)
    (10, 4, 5, 3, 131),     # unbalanced halves (2 + 1)
    (10, 4, 50, 3, 48),     # the reference's largest test case (twisted only: v1 state does not fit)
    (10, 4, 16, 1, 300),
    (10, 3, 5, 3, 300),
    (12, 5, 6, 3, 300),
    (10, 4, 6, 2, 200),     # D = 2 / 4 specialisations
    (10, 4, 7, 4, 200),
    (8, 3, 6, 2, 150),
    (6, 2, 5, 3, 200),      # N = 6 min acceleration
    (12, 5, 4, 4, 100),
])
def test_waypoint_kernel_matches_oracle(solver, oracle, N, r, K, D, B, variant):
    import mav_trajectory_generation_b200 as m
    prob, pos, times, ref, out, status, dfree = run_waypoint(solver, oracle, N, r, K, D, B, variant=variant)
    # d_free output (getFreeConstraints order) is consistent with the coefficients: derivative k of the
    # polynomial at t=0 of segment v equals u_v[k]
    h = N // 2
    for v in range(1, K):
        for k in range(1, h):
            fact = float(np.prod(np.arange(1, k + 1)))
            got = dfree[:, :, (v - 1) * (h - 1) + (k - 1)]
            want = out[:, v, :, k] * fact
            assert np.abs(got - want).max() <= 1e-9 * (1.0 + np.abs(want).max())
    assert prob.kernel == m.KERNEL_WAYPOINT
    assert (status == 0).all()
    # One rule for every shape (check_parity): within 1e-10 of the binary128 solve, or -- where the
    # reference-order arithmetic itself is further than that from exact (1-D fixtures with sub-second segments,
    # N = 12) -- no worse than twice the oracle's own error on that trajectory.
    exact = oracle.exact_solve_batch(N, r, times, oracle.waypoint_d_fixed(N, pos))
    check_parity(out, ref, exact, f"N={N} r={r} K={K} D={D} variant={variant}", baseline=(N, r, K, D) in BASELINE_SHAPES)


@pytest.mark.parametrize("K,B,chunk", [(100, 48, 0), (50, 80, 0), (50, 33, 3), (33, 65, 2), (16, 130, 3), (16, 70, 1),
                                       (7, 40, 1), (2, 17, 1), (200, 20, 0)])
def test_large_k_chunked_kernel(solver, oracle, K, B, chunk):
    """K3: the chunked (checkpoint + recompute) twisted kernel.  K = 50 / 100 are the sizes of the reference's
    timing program (polynomial_timing_evaluation.cpp:114-129) and tests (test_polynomial_optimization.cpp:822-828);
    small chunks are forced on small K to exercise every chunk-boundary case (partial outer chunk, chunk = 1,
    odd / even K, K = 2 with no interior sweep).  Checked against the binary128 solve and the oracle under the
    check_parity contract, and -- where the resident kernel also runs (K <= 34) -- bitwise against it: the
    recomputation replays the identical arithmetic."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, D = 10, 4, 3
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=106)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_WAYPOINT
    dfix = oracle.waypoint_d_fixed(N, pos)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    dfree = torch.zeros((B, D, prob.n_free), dtype=torch.float64, device="cuda")
    solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 5)
    solver.set_option(m.capi.OPT_CHUNK_BLOCKS, chunk)
    try:
        out = solver.solve_linear(prob, t_d, f_d, status=status, d_free=dfree)
        torch.cuda.synchronize()
    finally:
        solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 0)
        solver.set_option(m.capi.OPT_CHUNK_BLOCKS, 0)
    assert (status.cpu().numpy() == 0).all()
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, times, n_threads=oracle.hardware_threads())
    exact, exact_free, _ = oracle.exact_solve_batch(N, r, times, dfix, want_free=True)
    check_parity(out.cpu().numpy(), ref, exact, f"chunked K={K} chunk={chunk}")
    e_f = np.abs(dfree.cpu().numpy() - exact_free).reshape(B, -1).max(axis=1) / np.abs(exact_free).reshape(B, -1).max(axis=1)
    if K > 1:
        assert e_f.max() <= 1e-9, e_f.max()
    if K <= 34:
        solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 3)
        try:
            res = solver.solve_linear(prob, t_d, f_d)
            torch.cuda.synchronize()
        finally:
            solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 0)
        assert torch.equal(res, out), "chunked kernel differs from the resident kernel"
    if K >= 50:  # default routing reaches the chunked kernel
        dflt = solver.solve_linear(prob, t_d, f_d)
        torch.cuda.synchronize()
        assert torch.equal(dflt, out) or chunk != 0


@pytest.mark.parametrize("N,r,K,D,B", [(10, 4, 8, 3, 65536), (10, 4, 2, 3, 4112), (10, 4, 7, 3, 16), (10, 4, 5, 3, 1600),
                                       (8, 3, 4, 3, 131072), (8, 3, 8, 3, 48), (10, 4, 6, 1, 2048), (10, 3, 3, 3, 320),
                                       (10, 4, 16, 3, 40000), (10, 4, 13, 3, 4800), (10, 4, 20, 3, 640), (12, 5, 10, 3, 1024)])
def test_tma_input_kernel_bitwise_vs_resident(solver, oracle, N, r, K, D, B):
    """K1v5 (inputs moved as whole tiles by cp.async.bulk + mbarrier, double buffered, persistent warps): bitwise
    equal to the persistent kernel v4 on the same inputs (identical arithmetic, only the input path differs) --
    many tiles per warp (buffer reuse, mbarrier phase flips), a single tile, odd K, dynamic and static tile
    assignment, NON-ZERO end derivatives; K <= 8 double-buffered tiles, K >= 10 a single tile buffer refilled
    during the last emission; d_free and
    status outputs included.  Against the per-tile kernel v3 the
    results agree to rounding only: v4/v5 add the end-derivative carry of the first sweep step last instead of
    first (the 2^+-600 folding)."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(K * 100 + D)
    pos = rng.uniform(-10, 10, size=(B, K + 1, D))
    dist = np.maximum(np.linalg.norm(np.diff(pos, axis=1), axis=2), 0.2)
    times = dist / 3.0 * 2 * (1.0 + 6.5 * 3.0 / 5.0 * np.exp(-dist / 3.0 * 2))
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    prob = m.Problem(N, r, K, D)
    t_d = torch.from_numpy(np.ascontiguousarray(times)).cuda()
    f_d = torch.from_numpy(oracle.waypoint_d_fixed(N, pos, sd, ed)).cuda()
    outs = {}
    for variant, dyn in ((3, 0), (4, 2), (6, 1), (6, 2)):
        solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, variant)
        solver.set_option(m.capi.OPT_DYNAMIC_TILES, dyn)
        try:
            st = torch.full((B,), -1, dtype=torch.int32, device="cuda")
            df = torch.zeros((B, D, max(prob.n_free, 1)), dtype=torch.float64, device="cuda")
            out = solver.solve_linear(prob, t_d, f_d, status=st, d_free=df)
            torch.cuda.synchronize()
        finally:
            solver.set_option(m.capi.OPT_WAYPOINT_VARIANT, 0)
            solver.set_option(m.capi.OPT_DYNAMIC_TILES, 0)
        assert bool((st == 0).all())
        outs[(variant, dyn)] = (out, df)
    for key in ((6, 1), (6, 2)):
        assert torch.equal(outs[key][0], outs[(4, 2)][0]), key
        assert torch.equal(outs[key][1], outs[(4, 2)][1]), key
    den = outs[(3, 0)][0].abs().reshape(B, -1).max(dim=1).values
    # rounding-level agreement with the per-tile kernel: median at the 1e-15 level, every trajectory inside the
    # parity tolerance (ill-conditioned fixtures amplify the one reordered addition)
    dv = ((outs[(6, 1)][0] - outs[(3, 0)][0]).abs().reshape(B, -1).max(dim=1).values / den)
    assert float(dv.median()) <= (1e-14 if N < 12 else 1e-12) and float(dv.max()) <= (1e-10 if N < 12 else 1e-7)
    sub = slice(0, min(B, 256))
    exact = oracle.exact_solve_batch(N, r, times[sub], oracle.waypoint_d_fixed(N, pos, sd, ed)[sub])
    e_ge = global_rel_err(outs[(6, 1)][0][sub].cpu().numpy(), exact)
    assert e_ge.max() <= (1e-10 if N < 12 else 1e-7), e_ge.max()


@pytest.mark.parametrize("N,r,K,D,seed", [(10, 4, 16, 3, 1000), (10, 4, 16, 1, 1003), (10, 3, 5, 3, 110), (10, 2, 5, 3, 109),
                                          (12, 5, 6, 3, 3), (8, 3, 4, 3, 1002)])
def test_gpu_vs_truth(solver, oracle, N, r, K, D, seed):
    """Against the 60-digit solve of the same equations (oracle/truth.py): the kernels' exact-table
    formulation is ~1e-13 from the exact answer, i.e. closer than the reference's own arithmetic."""
    import os
    import sys
    import torch
    import mav_trajectory_generation_b200 as m
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import truth
    B = 3
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    prob = m.Problem(N, r, K, D)
    out = solver.solve_linear(prob, torch.from_numpy(times).cuda(),
                              torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda()).cpu().numpy()
    for b in range(B):
        mask, values = oracle.waypoint_problem(N, pos[b])
        tru, _ = truth.solve(N, r, mask, values, times[b])
        err = np.abs(out[b] - tru).max() / np.abs(tru).max()
        assert err <= 2e-12, (b, err)


def test_generic_kernel_arbitrary_masks(solver, oracle):
    """Arbitrary Vertex constraint sets (interior velocity fixed, free end derivatives, non-zero end
    derivatives), several N: the generic kernel against the oracle and the d_free output against the
    oracle's getFreeConstraints."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(11)
    for trial in range(12):
        N = int(rng.choice([6, 8, 10, 12]))
        h = N // 2
        K = int(rng.randint(2, 9))
        D = int(rng.randint(1, 4))
        B = 33
        mask = (rng.rand(K + 1, h) < 0.35).astype(np.uint8)
        mask[:, 0] = 1
        mask[0, :] = 1
        prob = m.Problem(N, h - 1, K, D, fixed_mask=mask)
        if prob.n_free == 0:
            continue
        assert prob.kernel in (m.KERNEL_GENERIC, m.KERNEL_WAYPOINT)
        times = rng.uniform(2.0, 6.0, size=(B, K))
        values = rng.uniform(-2, 2, size=(B, K + 1, h, D)) * mask[None, :, :, None]
        values[:, :, 0, :] = rng.uniform(-10, 10, size=(B, K + 1, D))
        ref = np.zeros((B, K, D, N))
        dfix = np.zeros((B, D, prob.n_fixed))
        dfree_ref = np.zeros((B, D, prob.n_free))
        for b in range(B):
            res = oracle.solve(N, h - 1, mask, values[b], times[b])
            ref[b], dfix[b], dfree_ref[b] = res["coeffs"], res["d_fixed"], res["d_free"]
        status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        dfree = torch.zeros((B, D, prob.n_free), dtype=torch.float64, device="cuda")
        out = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda(), d_free=dfree,
                                  status=status)
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all()
        # every trajectory against the binary128 solve with the same mask; the oracle (whose QR works on the
        # cancellation-prone A^-T Q A^-1) only has to be as close to the kernel as it is to exact
        exact, exact_free, _ = oracle.exact_solve_batch(N, h - 1, times, dfix, mask=mask, want_free=True)
        check_parity(out.cpu().numpy(), ref, exact, f"mask trial {trial} N={N} K={K} D={D}")
        got_free = dfree.cpu().numpy()
        e_f = np.abs(got_free - exact_free).reshape(B, -1).max(axis=1) / np.abs(exact_free).reshape(B, -1).max(axis=1)
        e_of = np.abs(dfree_ref - exact_free).reshape(B, -1).max(axis=1) / np.abs(exact_free).reshape(B, -1).max(axis=1)
        assert (e_f <= np.maximum(1e-10, 2.0 * e_of)).all(), (trial, N, K, D, e_f.max(), e_of.max())


def test_waypoint_nonzero_end_derivatives_and_dfree(solver, oracle):
    """Start/end vertices with NON-zero velocity..snap (the general makeStartOrEnd-free case) through
    the waypoint kernel; also checks the optional d_free output."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(5)
    N, r, K, D, B = 10, 4, 6, 3, 65
    h = N // 2
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=2000)
    sd = rng.uniform(-1, 1, size=(B, h - 1, D))
    ed = rng.uniform(-1, 1, size=(B, h - 1, D))
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    assert prob.kernel == m.KERNEL_WAYPOINT
    ref = np.zeros((B, K, D, N))
    dfree_ref = np.zeros((B, D, prob.n_free))
    for b in range(B):
        mask, values = oracle.waypoint_problem(N, pos[b])
        values[0, 1:, :] = sd[b]
        values[-1, 1:, :] = ed[b]
        res = oracle.solve(N, r, mask, values, times[b])
        ref[b], dfree_ref[b] = res["coeffs"], res["d_free"]
        np.testing.assert_array_equal(res["d_fixed"], dfix[b])
    dfree = torch.zeros((B, D, prob.n_free), dtype=torch.float64, device="cuda")
    out = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda(), d_free=dfree)
    torch.cuda.synchronize()
    assert global_rel_err(out.cpu().numpy(), ref).max() <= TOL
    assert np.abs(dfree.cpu().numpy() - dfree_ref).max() <= 1e-9 * np.abs(dfree_ref).max()


def test_status_flags_and_edge_cases(solver, oracle):
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 4, 3, 40
    pos, times = oracle.make_waypoint_batch(K, D, B)
    times[3, 1] = 0.0       # reference: CHECK_GT(segment_time, 0) aborts (linear_impl.h:297)
    times[7, 2] = -1.0
    times[9, 0] = float("nan")
    prob = m.Problem(N, r, K, D)
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    out = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda(),
                              status=status)
    st = status.cpu().numpy()
    bad = [3, 7, 9]
    assert all(st[b] & m.STATUS_BAD_TIME for b in bad)
    good = [b for b in range(B) if b not in bad]
    assert (st[good] == 0).all()
    ref, _ = oracle.solve_waypoint_batch(N, r, pos[good], times[good])
    assert global_rel_err(out.cpu().numpy()[good], ref).max() <= TOL
    # empty batch is a no-op
    empty = solver.solve_linear(prob, torch.zeros((0, K), dtype=torch.float64, device="cuda"),
                                torch.zeros((0, D, prob.n_fixed), dtype=torch.float64, device="cuda"))
    assert empty.shape[0] == 0


def test_nofree_backsub_and_cost(solver, oracle):
    """n_free == 0 shortcut (linear_impl.h:343-349), setFreeConstraints path and computeCost()."""
    import torch
    import mav_trajectory_generation_b200 as m
    # fully constrained single segment, N = 12, 4-D (the reference's feasibility-test usage)
    rng = np.random.RandomState(2)
    N, r, K, D, B = 12, 5, 1, 4, 50
    h = N // 2
    mask = np.ones((2, h), dtype=np.uint8)
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_NOFREE
    values = rng.uniform(-1, 1, size=(B, 2, h, D))
    times = rng.uniform(1.0, 5.0, size=(B, 1))
    ref = np.zeros((B, K, D, N))
    dfix = np.zeros((B, D, prob.n_fixed))
    cost_ref = np.zeros(B)
    for b in range(B):
        res = oracle.solve(N, r, mask, values[b], times[b])
        ref[b], dfix[b], cost_ref[b] = res["coeffs"], res["d_fixed"], res["cost"]
    t_d = torch.from_numpy(times).cuda()
    out = solver.solve_linear(prob, t_d, torch.from_numpy(dfix).cuda())
    assert global_rel_err(out.cpu().numpy(), ref).max() <= TOL
    cost = solver.compute_cost(prob, t_d, out).cpu().numpy()
    np.testing.assert_allclose(cost, cost_ref, rtol=1e-7)  # c^T Q c cancels ~1e-9 for N=12 in either arithmetic
    # setFreeConstraints path on a problem with free constraints: feed the oracle's optimum back
    N, r, K, D, B = 10, 4, 5, 3, 20
    pos, times = oracle.make_waypoint_batch(K, D, B)
    prob = m.Problem(N, r, K, D)
    ref = np.zeros((B, K, D, N))
    dfree = np.zeros((B, D, prob.n_free))
    cost_ref = np.zeros(B)
    for b in range(B):
        mask, values = oracle.waypoint_problem(N, pos[b])
        res = oracle.solve(N, r, mask, values, times[b])
        ref[b], dfree[b], cost_ref[b] = res["coeffs"], res["d_free"], res["cost"]
    t_d = torch.from_numpy(times).cuda()
    out = solver.coeffs_from_constraints(prob, t_d, torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda(),
                                         torch.from_numpy(dfree).cuda())
    assert global_rel_err(out.cpu().numpy(), ref).max() <= TOL
    np.testing.assert_allclose(solver.compute_cost(prob, t_d, out).cpu().numpy(), cost_ref, rtol=1e-8)


def test_host_pointer_path_bitwise_equals_device_path(solver, oracle):
    """mtg_solve_linear_batch_host_f64 (what the C++ solveLinear() calls): chunked H2D/solve/D2H gives
    bit-identical results to the device-pointer call (each trajectory is solved independently)."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 8, 3, 100003  # > one pipeline chunk, ragged
    rng = np.random.RandomState(0)
    pos = rng.uniform(-10, 10, size=(B, K + 1, D))
    dist = np.maximum(np.linalg.norm(np.diff(pos, axis=1), axis=2), 0.2)
    times = dist / 3.0 * 2 * (1.0 + 6.5 * 3.0 / 5.0 * np.exp(-dist / 3.0 * 2))
    dfix = oracle.waypoint_d_fixed(N, pos)
    prob = m.Problem(N, r, K, D)
    dev = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()).cpu().numpy()
    host = np.zeros((B, K, D, N))
    status = np.full(B, -1, dtype=np.int32)
    solver.solve_linear_host(prob, np.ascontiguousarray(times), dfix, host, status=status)
    assert (status == 0).all()
    assert np.array_equal(host, dev)
    ref, _ = oracle.solve_waypoint_batch(N, r, pos[:512], times[:512], n_threads=oracle.hardware_threads())
    assert global_rel_err(host[:512], ref).max() <= TOL


def test_full_size_properties_c3(solver):
    """BASELINE C3 at full size (262 144 x 16 segments): size-independent properties instead of an
    oracle pass -- position constraints met, derivatives 0..4 continuous at every interior vertex,
    zero end derivatives, shard-concatenation == whole-batch (bitwise), computeCost linear in D."""
    import torch
    import mav_trajectory_generation_b200 as m
    import bench
    N, r, K, D, B = 10, 4, 16, 3, 262144
    dev = torch.device("cuda:0")
    pos, times, dfix = bench.synth_batch(torch, N, K, D, B, dev, seed=7)
    prob = m.Problem(N, r, K, D)
    status = torch.full((B,), -1, dtype=torch.int32, device=dev)
    out = solver.solve_linear(prob, times, dfix, status=status)
    assert bool((status == 0).all())
    # evaluate derivatives at t = 0 and t = T with torch (independent of the kernels)
    T = times[:, :, None, None]                                   # [B][K][1][1]
    powers = torch.arange(N, device=dev, dtype=torch.float64)
    scale = pos.abs().max()
    for k in range(5):
        fall = torch.ones(N, device=dev, dtype=torch.float64)
        for q in range(k):
            fall = fall * (powers - q).clamp_min(0)
        at0 = out[..., k] * fall[k]
        atT = (out * fall * T ** (powers - k).clamp_min(0)).sum(dim=-1)   # [B][K][D]
        tol = 1e-7 * float(scale)
        if k == 0:
            assert (at0 - pos[:, :-1]).abs().max() <= tol and (atT - pos[:, 1:]).abs().max() <= tol
        else:
            assert at0[:, 0].abs().max() <= tol and atT[:, -1].abs().max() <= tol
        assert (atT[:, :-1] - at0[:, 1:]).abs().max() <= tol   # continuity at interior vertices
    # sharding: solving two halves separately gives the same bits
    half = B // 2
    a = solver.solve_linear(prob, times[:half].contiguous(), dfix[:half].contiguous())
    b = solver.solve_linear(prob, times[half:].contiguous(), dfix[half:].contiguous())
    assert torch.equal(torch.cat([a, b]), out)


@pytest.mark.parametrize("N,r,K,D,B", [(10, 4, 16, 3, 1024), (8, 3, 4, 3, 777), (10, 4, 5, 2, 130), (10, 4, 6, 5, 64),
                                       (10, 4, 100, 3, 24)])
def test_fused_nfabian_waypoint_entry(solver, oracle, N, r, K, D, B):
    """SURVEY.md 8f-1: positions in, estimateSegmentTimesNfabian + constraint packing on the device.  The
    last two cases have no fused specialisation (D = 5: generic kernel; K = 100: state too large) and go
    through the pack-kernel fallback."""
    import torch
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=4000)   # v_max 3, a_max 5, magic 6.5
    ref, _ = oracle.solve_waypoint_batch(N, r, pos, times, n_threads=oracle.hardware_threads())
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    t_out = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    out = solver.solve_waypoints_nfabian(N, r, torch.from_numpy(pos).cuda(), 3.0, 5.0, 6.5, seg_times_out=t_out,
                                         status=status)
    torch.cuda.synchronize()
    assert (status.cpu().numpy() == 0).all()
    # device exp() vs glibc exp(): at most a couple of ulps apart
    np.testing.assert_allclose(t_out.cpu().numpy(), times, rtol=4e-16, atol=0)
    exact = oracle.exact_solve_batch(N, r, times, oracle.waypoint_d_fixed(N, pos))
    check_parity(out.cpu().numpy(), ref, exact, f"fused N={N} K={K} D={D}")


@pytest.mark.parametrize("N,r,K,D,B", [(10, 4, 16, 3, 40), (10, 4, 5, 3, 33), (8, 3, 4, 3, 50), (10, 4, 1, 3, 5)])
def test_batched_mellinger_gradient(solver, oracle, N, r, K, D, B):
    """SURVEY.md 8f-2: batched getCostAndGradientMellinger against the oracle's restatement of the
    reference loop (K+1 re-solves per trajectory).  Costs agree to 1e-8 relative (c^T Q c cancels ~1e-10 in the
    reference-order arithmetic); the gradient is a difference of two costs divided by 0.1, so its absolute
    error is ~20x the cost error."""
    import torch
    import mav_trajectory_generation_b200 as m
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=6000)
    prob = m.Problem(N, r, K, D)
    cost, grad = solver.cost_gradient_mellinger(prob, torch.from_numpy(times).cuda(),
                                                torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda())
    torch.cuda.synchronize()
    cost, grad = cost.cpu().numpy(), grad.cpu().numpy()
    for b in range(B):
        c_ref, g_ref = oracle.cost_gradient_mellinger(N, r, pos[b], times[b])
        assert abs(cost[b] - c_ref) <= 1e-8 * abs(c_ref)
        assert np.abs(grad[b] - g_ref).max() <= 1e-6 * max(abs(c_ref), np.abs(g_ref).max())
    # the fused cost-only path evaluates 0.5 d^T H d from the exact tables: against the binary128 cost it is far
    # tighter than the reference's own c^T Q c arithmetic
    _, _, c_exact = oracle.exact_solve_batch(N, r, times, oracle.waypoint_d_fixed(N, pos), want_cost=True)
    assert np.abs(cost - c_exact).max() <= 1e-10 * np.abs(c_exact).max()
    # and the round-1 path (expand + solve + cost kernels) agrees with it
    solver.set_option(m.capi.OPT_MELLINGER_UNFUSED, 1)
    try:
        cost_u, grad_u = solver.cost_gradient_mellinger(prob, torch.from_numpy(times).cuda(),
                                                        torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda())
        torch.cuda.synchronize()
    finally:
        solver.set_option(m.capi.OPT_MELLINGER_UNFUSED, 0)
    cost_u, grad_u = cost_u.cpu().numpy(), grad_u.cpu().numpy()
    assert np.abs(cost_u - cost).max() <= 1e-8 * np.abs(cost).max()
    if K > 1:
        assert np.abs(grad_u - grad).max() <= 1e-6 * max(np.abs(cost).max(), np.abs(grad).max())


def test_batched_evaluate(solver, oracle):
    """SURVEY.md 8f-3: batched Trajectory::evaluate against a numpy Horner evaluation with the reference's
    segment-selection conventions (vertex times belong to the right segment, the end time to the last one,
    beyond the end -> zeros)."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 37
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=8000)
    prob = m.Problem(N, r, K, D)
    t_d = torch.from_numpy(times).cuda()
    coeffs = solver.solve_linear(prob, t_d, torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda())
    c = coeffs.cpu().numpy()
    S, dt = 257, 0.25
    for der in (0, 1, 2, 4):
        got = solver.evaluate(t_d, coeffs, der, 0.0, dt, S).cpu().numpy()
        want = np.zeros((B, S, D))
        for b in range(B):
            ends = np.cumsum(times[b])
            for s_i in range(S):
                t = s_i * dt
                if t > ends[-1]:
                    continue
                i = int(np.searchsorted(ends, t, side="right"))
                i = min(i, K - 1)
                tl = t - (ends[i] - times[b, i])
                for d in range(D):
                    acc = 0.0
                    for j in range(N - 1, der - 1, -1):
                        acc = acc * tl + np.prod(np.arange(j - der + 1, j + 1, dtype=np.float64)) * c[b, i, d, j]
                    want[b, s_i, d] = acc
        scale = max(1.0, np.abs(want).max())
        assert np.abs(got - want).max() <= 1e-11 * scale, der
    # positions at the vertices are the waypoints (t on a vertex -> right segment, value continuous)
    pos0 = solver.evaluate(t_d, coeffs, 0, 0.0, 1.0, 1).cpu().numpy()[:, 0, :]
    assert np.abs(pos0 - pos[:, 0, :]).max() <= 1e-9


def test_small_orders_n2_n4(solver, oracle):
    """N = 2 (piecewise linear: every constraint fixed, back-substitution only) and N = 4 (cubic, velocity free
    at interior vertices -> generic kernel), the smallest orders the reference template accepts."""
    import torch
    import mav_trajectory_generation_b200 as m
    rng = np.random.RandomState(4)
    for N, r in ((2, 0), (4, 1), (4, 0)):
        h = N // 2
        K, D, B = 5, 3, 21
        mask = np.zeros((K + 1, h), dtype=np.uint8)
        mask[:, 0] = 1
        mask[0, :] = 1
        mask[-1, :] = 1
        prob = m.Problem(N, r, K, D, fixed_mask=mask)
        times = rng.uniform(1.0, 3.0, size=(B, K))
        values = rng.uniform(-1, 1, size=(B, K + 1, h, D)) * mask[None, :, :, None]
        ref = np.zeros((B, K, D, N))
        dfix = np.zeros((B, D, prob.n_fixed))
        for b in range(B):
            res = oracle.solve(N, r, mask, values[b], times[b])
            ref[b], dfix[b] = res["coeffs"], res["d_fixed"]
        status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        out = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda(), status=status)
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all(), (N, r)
        assert global_rel_err(out.cpu().numpy(), ref).max() <= 1e-11, (N, r)


# ---------------------------------------------------------------------------------------------------------
# Host-pointer pipeline: chunks run concurrently on 3 streams.  Round 1 shared ONE band / pack scratch between
# them (a data race on generic topologies and on the Nfabian pack fallback).  These tests use PINNED buffers
# (pageable copies serialise and hide the race) and B > one pipeline chunk.

def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


def test_host_pipeline_generic_mask_bitwise_equals_device_path(solver, oracle):
    """Generic (non-waypoint) mask -- interior velocity fixed as well -- B = 100 003, pinned host buffers:
    the pipelined host path must be bit-identical to one device-pointer launch, and correct vs exact."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 100003
    h = N // 2
    mask = np.zeros((K + 1, h), dtype=np.uint8)
    mask[:, 0] = 1
    mask[:, 1] = 1          # velocity fixed at every vertex
    mask[0, :] = 1
    mask[-1, :] = 1
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC
    rng = np.random.RandomState(3)
    times = rng.uniform(2.0, 6.0, size=(B, K))
    dfix = rng.uniform(-2, 2, size=(B, D, prob.n_fixed))
    dev = solver.solve_linear(prob, torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda())
    torch.cuda.synchronize()
    dev = dev.cpu().numpy()
    for rep in range(2):
        host = torch.zeros((B, K, D, N), dtype=torch.float64).pin_memory()
        status = torch.full((B,), -1, dtype=torch.int32).pin_memory()
        solver.solve_linear_host(prob, _pinned(times), _pinned(dfix), host, status=status)
        assert bool((status == 0).all())
        assert np.array_equal(host.numpy(), dev), f"host pipeline differs from the device path (rep {rep})"
    sub = rng.choice(B, size=256, replace=False)
    exact = oracle.exact_solve_batch(N, r, times[sub], dfix[sub], mask=mask)
    assert global_rel_err(dev[sub], exact).max() <= 1e-10


@pytest.mark.parametrize("N,r,K,D,B", [(10, 4, 6, 5, 20011), (10, 4, 100, 3, 6007)])
def test_nfabian_host_pipeline_pack_fallback_bitwise(solver, oracle, N, r, K, D, B):
    """mtg_solve_waypoints_nfabian_batch_host_f64 on shapes WITHOUT a fused kernel (D = 5; K = 100): pack kernel +
    solve per chunk on 3 streams, B > 4096, pinned buffers -- bit-identical to one device-pointer call."""
    import torch
    rng = np.random.RandomState(8)
    pos = rng.uniform(-10, 10, size=(B, K + 1, D))
    dev_t = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    dev = solver.solve_waypoints_nfabian(N, r, torch.from_numpy(pos).cuda(), 3.0, 5.0, 6.5, seg_times_out=dev_t)
    torch.cuda.synchronize()
    host = torch.zeros((B, K, D, N), dtype=torch.float64).pin_memory()
    host_t = torch.zeros((B, K), dtype=torch.float64).pin_memory()
    status = torch.full((B,), -1, dtype=torch.int32).pin_memory()
    solver.solve_waypoints_nfabian_host(N, r, _pinned(pos), 3.0, 5.0, 6.5, host, seg_times_out=host_t, status=status)
    assert bool((status == 0).all())
    assert np.array_equal(host_t.numpy(), dev_t.cpu().numpy())
    assert np.array_equal(host.numpy(), dev.cpu().numpy())


def test_mellinger_odd_offsets_and_unaligned_output(solver, oracle):
    """ADVICE r1: (10,4,16,3) with B = 33 put the expanded coefficient buffer at an odd double offset (TMA
    tensor maps need 16 bytes) -> MTG_ERR_CUDA.  Sub-buffers are now 256-byte aligned; and a caller buffer that
    is only 8-byte aligned takes the scalar-store generic kernel instead of failing."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 33
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=6100)
    prob = m.Problem(N, r, K, D)
    t_d = torch.from_numpy(times).cuda()
    f_d = torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda()
    cost, grad = solver.cost_gradient_mellinger(prob, t_d, f_d)
    torch.cuda.synchronize()
    c_ref, g_ref = oracle.cost_gradient_mellinger(N, r, pos[0], times[0])
    assert abs(float(cost[0]) - c_ref) <= 1e-8 * abs(c_ref)
    assert np.abs(grad[0].cpu().numpy() - g_ref).max() <= 1e-6 * max(abs(c_ref), np.abs(g_ref).max())
    # 8-byte aligned output slice
    aligned = solver.solve_linear(prob, t_d, f_d)
    big = torch.zeros(B * K * D * N + 1, dtype=torch.float64, device="cuda")
    odd = big[1:].view(B, K, D, N)
    assert odd.data_ptr() % 16 == 8
    solver.solve_linear(prob, t_d, f_d, coeffs=odd)
    torch.cuda.synchronize()
    exact = oracle.exact_solve_batch(N, r, times, oracle.waypoint_d_fixed(N, pos))
    assert global_rel_err(odd.cpu().numpy(), exact).max() <= 1e-10
    assert global_rel_err(aligned.cpu().numpy(), exact).max() <= 1e-10


def test_batched_evaluate_range_bitwise_vs_oracle(solver, oracle):
    """SURVEY.md 8f-3: mtg_evaluate_range_batch_f64 replays Trajectory::evaluateRange (reference
    src/trajectory.cpp:81-141) -- sequential walk, quirks included -- and Polynomial::evaluate's arithmetic: the
    sample count, the sampling times and every sample are BIT-IDENTICAL to the oracle's literal restatement,
    for t_start = 0 (sampleWholeTrajectory), a mid-trajectory start, a start on a vertex, a range that runs past
    the end, and a start beyond the end (n = -1)."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 41
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=8100)
    prob = m.Problem(N, r, K, D)
    t_d = torch.from_numpy(times).cuda()
    coeffs = solver.solve_linear(prob, t_d, torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).cuda())
    c = coeffs.cpu().numpy()
    total = times.sum(axis=1)
    cases = [(0.0, float(total.min()), 0.01), (1.2345, 9.5, 0.1), (float(times[0, 0]), 7.0, 0.25),
             (3.0, 1e9, 0.5), (float(total.max()) + 1.0, float(total.max()) + 2.0, 0.1)]
    derivs = (0, 1, 2, 3, 4)
    for t0, t1, dt in cases:
        S = int(float(total.max()) / dt) + 8   # the walk never outlives the trajectory
        out, n, st = solver.evaluate_range(t_d, coeffs, t0, t1, dt, derivs=derivs, max_samples=S, want_times=True)
        torch.cuda.synchronize()
        out, n, st = out.cpu().numpy(), n.cpu().numpy(), st.cpu().numpy()
        for b in range(B):
            for q, der in enumerate(derivs):
                n_ref, o_ref, st_ref = oracle.evaluate_range(times[b], c[b], t0, t1, dt, der, S)
                assert n[b] == n_ref, (t0, t1, dt, b, n[b], n_ref)
                if n_ref > 0:
                    k = min(n_ref, S)
                    assert np.array_equal(out[b, :k, q, :], o_ref[:k]), (t0, b, der)
                    assert np.array_equal(st[b, :k], st_ref[:k])
                    assert not out[b, k:].any()


def test_one_handle_two_caller_streams_dynamic_tiles(solver, oracle):
    """Two large solves of one handle enqueued on two different caller streams: the persistent kernel's dynamic tile
    counter is per handle slot, so the second launch must be ordered behind the first (event), not race on the counter --
    both results equal the single-stream solve bit for bit."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 16, 3, 180000 // 16 * 16
    prob = m.Problem(N, r, K, D)
    pos, times = oracle.make_waypoint_batch(K, D, 2048, base_seed=77)
    dev = torch.device("cuda:0")
    t_small = torch.from_numpy(times).to(dev)
    f_small = torch.from_numpy(oracle.waypoint_d_fixed(N, pos)).to(dev)
    idx_a = torch.arange(B, device=dev) % 2048
    idx_b = (torch.arange(B, device=dev) * 7 + 3) % 2048
    ta, fa = t_small[idx_a].contiguous(), f_small[idx_a].contiguous()
    tb, fb = t_small[idx_b].contiguous(), f_small[idx_b].contiguous()
    solver.set_option(m.capi.OPT_DYNAMIC_TILES, 1)
    try:
        want_a = solver.solve_linear(prob, ta, fa)
        want_b = solver.solve_linear(prob, tb, fb)
        out_a, out_b = torch.zeros_like(want_a), torch.zeros_like(want_b)
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        for _ in range(3):
            solver.solve_linear(prob, ta, fa, coeffs=out_a, stream=s1.cuda_stream)
            solver.solve_linear(prob, tb, fb, coeffs=out_b, stream=s2.cuda_stream)
        torch.cuda.synchronize()
    finally:
        solver.set_option(m.capi.OPT_DYNAMIC_TILES, 0)
    assert torch.equal(out_a, want_a) and torch.equal(out_b, want_b)
