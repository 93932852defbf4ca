"""The host-pointer entry points beyond their bit-for-bit parity with the device entries (test_generic_kernels.py §5,
test_time_scaling.py, test_time_objective.py and the host-pipeline tests):

  1. every nullable output of a host entry may be omitted (NULL): the outputs that are given stay bit for bit those of
     the device call with every output given;
  2. a host call whose arguments its device entry's check refuses returns MTG_ERR_BAD_ARG before any copy or launch;
  3. every compute entry point, device and host, right after a refused allocation has left an error in the library's
     CUDA runtime, returns MTG_OK with the outputs of a clean call.
"""
import numpy as np
import pytest

from test_large_k import _pinned, same_bits
from test_masked_kernel import waypoint_mask

pytestmark = pytest.mark.gpu
NAN = float("nan")


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _dev(shape, dtype=None):
    import torch
    return torch.full(shape, -1, dtype=dtype or torch.float64, device="cuda")


def _host(shape, dtype=np.float64):
    return np.full(shape, -1, dtype=dtype)


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _waypoints(oracle, N, K, D, B, seed):
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    return pos, times, oracle.waypoint_d_fixed(N, pos)


# ---------------------------------------------------------------------------------------------------------------------
# 1. Nullable outputs given and omitted.  Each case returns (device outputs, host(given) -> host outputs in the same
# order, None where omitted).

def _solve_generic(solver, oracle):
    """a generic mask (velocity fixed at every vertex) at B = 9001: three pipeline chunks; d_free and status"""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 6, 3, 9001
    mask = np.array(waypoint_mask(N, K), dtype=np.uint8)
    mask[:, 1] = 1
    prob = m.Problem(N, r, K, D, fixed_mask=mask)
    assert prob.kernel == m.KERNEL_GENERIC and prob.n_free > 0
    rng = np.random.RandomState(3)
    times, dfix = rng.uniform(2.0, 6.0, size=(B, K)), rng.uniform(-2, 2, size=(B, D, prob.n_fixed))
    free, st = _dev((B, D, prob.n_free)), _dev((B,), torch.int32)
    dev = [solver.solve_linear(prob, _cuda(times), _cuda(dfix), d_free=free, status=st), free, st]

    def host(given):
        c = _pinned(_host((B, K, D, N)))
        free = _pinned(_host((B, D, prob.n_free))) if given else None
        st = _pinned(_host((B,), np.int32)) if given else None
        solver.solve_linear_host(prob, _pinned(times), _pinned(dfix), c, d_free=free, status=st)
        return [c, free, st]
    return dev, host


def _solve_waypoint(solver, oracle):
    """the waypoint kernel, one chunk; d_free and status"""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B = 10, 4, 5, 3, 1000
    prob = m.Problem(N, r, K, D)
    _, times, dfix = _waypoints(oracle, N, K, D, B, 19000)
    free, st = _dev((B, D, prob.n_free)), _dev((B,), torch.int32)
    dev = [solver.solve_linear(prob, _cuda(times), _cuda(dfix), d_free=free, status=st), free, st]

    def host(given):
        c = _host((B, K, D, N))
        free = _host((B, D, prob.n_free)) if given else None
        st = _host((B,), np.int32) if given else None
        solver.solve_linear_host(prob, times, dfix, c, d_free=free, status=st)
        return [c, free, st]
    return dev, host


def _nfabian_pack(solver, oracle):
    """D = 5 has no fused kernel (pack fallback), B = 5003: pipelined; seg_times_out and status"""
    import torch
    N, r, K, D, B = 10, 4, 6, 5, 5003
    pos = np.random.RandomState(8).uniform(-10, 10, size=(B, K + 1, D))
    t, st = _dev((B, K)), _dev((B,), torch.int32)
    dev = [solver.solve_waypoints_nfabian(N, r, _cuda(pos), 3.0, 5.0, 6.5, seg_times_out=t, status=st), t, st]

    def host(given):
        c = _pinned(_host((B, K, D, N)))
        t = _pinned(_host((B, K))) if given else None
        st = _pinned(_host((B,), np.int32)) if given else None
        solver.solve_waypoints_nfabian_host(N, r, _pinned(pos), 3.0, 5.0, 6.5, c, seg_times_out=t, status=st)
        return [c, t, st]
    return dev, host


def _nfabian_fused(solver, oracle):
    """the fused Nfabian kernel, one chunk; seg_times_out and status"""
    import torch
    N, r, K, D, B = 10, 4, 5, 3, 1000
    pos, _, _ = _waypoints(oracle, N, K, D, B, 19100)
    t, st = _dev((B, K)), _dev((B,), torch.int32)
    dev = [solver.solve_waypoints_nfabian(N, r, _cuda(pos), 3.0, 5.0, 6.5, seg_times_out=t, status=st), t, st]

    def host(given):
        c = _host((B, K, D, N))
        t = _host((B, K)) if given else None
        st = _host((B,), np.int32) if given else None
        solver.solve_waypoints_nfabian_host(N, r, pos, 3.0, 5.0, 6.5, c, seg_times_out=t, status=st)
        return [c, t, st]
    return dev, host


def _solved(solver, oracle, seed, B=1001):
    import mav_trajectory_generation_b200 as m
    N, r, K, D = 10, 4, 5, 3
    prob = m.Problem(N, r, K, D)
    _, times, dfix = _waypoints(oracle, N, K, D, B, seed)
    coeffs = _np(solver.solve_linear(prob, _cuda(times), _cuda(dfix)))
    return prob, times, dfix, coeffs


def _max_magnitude(solver, oracle):
    """time, segment and status"""
    _, times, _, coeffs = _solved(solver, oracle, 19200)
    B = times.shape[0]
    dev = list(solver.max_magnitude(_cuda(times), _cuda(coeffs), (1, 2)))

    def host(given):
        v = _host((B, 2))
        t, s, st = (_host((B, 2)), _host((B, 2), np.int32), _host((B,), np.int32)) if given else (None,) * 3
        solver.max_magnitude_host(times, coeffs, (1, 2), v, t, s, st)
        return [v, t, s, st]
    return dev, host


def _time_objective(solver, oracle):
    """terms and status"""
    import mav_trajectory_generation_b200 as m
    prob, times, dfix, _ = _solved(solver, oracle, 19300)
    B, cons = times.shape[0], ((1, 2.0), (2, 3.0))
    obj, terms, coeffs, st = solver.time_objective(prob, _cuda(times), _cuda(dfix), constraints=cons)
    dev = [coeffs, obj, terms, st]

    def host(given):
        c, o = _host((B, prob.K, prob.D, prob.N)), _host((B,))
        tm, st = (_host((B, 3)), _host((B,), np.int32)) if given else (None, None)
        solver.time_objective_host(prob, times, dfix, None, m.time_objective_params(constraints=cons), c, o, tm, st)
        return [c, o, tm, st]
    return dev, host


def _scale_to_constraints(solver, oracle):
    """within_range, maxima and status"""
    _, times, _, coeffs = _solved(solver, oracle, 19400)
    B = times.shape[0]
    dev = list(solver.scale_to_constraints(_cuda(times), _cuda(coeffs), 2.0, 3.0))

    def host(given):
        t, c = _host(times.shape), _host(coeffs.shape)
        w, mx, st = (_host((B,), np.int32), _host((B, 2)), _host((B,), np.int32)) if given else (None,) * 3
        solver.scale_to_constraints_host(times, coeffs, 2.0, 3.0, t, c, w, mx, st)
        return [t, c, w, mx, st]
    return dev, host


def _scale_with_violation(solver, oracle):
    """within_range, maxima and status"""
    prob, times, dfix, coeffs = _solved(solver, oracle, 19500)
    B = times.shape[0]
    dev = list(solver.scale_times_with_violation(prob, _cuda(times), _cuda(dfix), 2.0, 3.0))

    def host(given):
        c, t = _host(coeffs.shape), _host(times.shape)
        w, mx, st = (_host((B,), np.int32), _host((B, 2)), _host((B,), np.int32)) if given else (None,) * 3
        solver.scale_times_with_violation_host(prob, times, dfix, 2.0, 3.0, c, t, w, mx, st)
        return [c, t, w, mx, st]
    return dev, host


def _mellinger(solver, oracle):
    """cost, on the fused cost-only path (K > 1)"""
    prob, times, dfix, _ = _solved(solver, oracle, 19600, B=37)
    dev = list(solver.cost_gradient_mellinger(prob, _cuda(times), _cuda(dfix)))

    def host(given):
        cost, grad = _host((times.shape[0],)) if given else None, _host(times.shape)
        solver.cost_gradient_mellinger_host(prob, times, dfix, cost, grad)
        return [cost, grad]
    return dev, host


OPTIONAL_CASES = {
    "solve_generic": _solve_generic, "solve_waypoint": _solve_waypoint, "nfabian_pack": _nfabian_pack,
    "nfabian_fused": _nfabian_fused, "max_magnitude": _max_magnitude, "time_objective": _time_objective,
    "scale_to_constraints": _scale_to_constraints, "scale_times_with_violation": _scale_with_violation,
    "mellinger": _mellinger,
}


@pytest.mark.parametrize("case", list(OPTIONAL_CASES))
def test_nullable_outputs_given_and_omitted(solver, oracle, case):
    """The host entry with its nullable outputs given and omitted: every output it returns equals the device call's
    bit for bit."""
    import torch
    dev, host = OPTIONAL_CASES[case](solver, oracle)
    torch.cuda.synchronize()
    dev = [_np(x) for x in dev]
    for given in (True, False):
        got = host(given)
        assert given == all(g is not None for g in got)
        for i, (g, d) in enumerate(zip(got, dev)):
            if g is not None:
                assert same_bits(_np(g), d), f"{case}: output {i} differs (optional outputs given: {given})"


# ---------------------------------------------------------------------------------------------------------------------
# 2. Refused before any copy

@pytest.mark.parametrize("kind", ["pageable", "pinned"])
def test_host_arguments_refused_before_copies(solver, kind):
    """evaluateRange with dt = 0 and Nfabian with v_max = 0: the device entries' checks refuse them, and so do the host
    entries -- MTG_ERR_BAD_ARG, no launch, every host output untouched."""
    def buf(shape, dtype=np.float64, fill=NAN):
        a = np.full(shape, fill, dtype=dtype)
        return _pinned(a) if kind == "pinned" else a

    launches = solver.launch_count
    N, K, D, B, S = 8, 2, 3, 5, 4
    out, n = buf((B, S, 1, D)), buf((B,), np.int32, -7)
    with pytest.raises(RuntimeError, match="bad argument"):
        solver.evaluate_range_host(buf((B, K), fill=1.0), buf((B, K, D, N), fill=0.0), 0.0, 1.0, 0.0, [0], out, n)
    N, r, K, D, B = 10, 4, 3, 3, 5
    coeffs, t_out, status = buf((B, K, D, N)), buf((B, K)), buf((B,), np.int32, -7)
    with pytest.raises(RuntimeError, match="bad argument"):
        solver.solve_waypoints_nfabian_host(N, r, buf((B, K + 1, D), fill=0.0), 0.0, 5.0, 6.5, coeffs,
                                            seg_times_out=t_out, status=status)
    assert solver.launch_count == launches
    assert np.isnan(_np(out)).all() and (_np(n) == -7).all()
    assert np.isnan(_np(coeffs)).all() and np.isnan(_np(t_out)).all() and (_np(status) == -7).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. A stale error in the library's CUDA runtime

def test_entry_points_ignore_a_stale_runtime_error(solver, oracle):
    """libmtg_b200.so links the CUDA runtime statically, so a runtime call of the library that failed -- here an
    mtg_device_alloc of 1 PiB, which cudaMalloc refuses on the host side -- leaves its error in the library's own
    last-error state.  Each of the 11 device and 10 host compute entry points, called right after such a refusal,
    returns MTG_OK (the wrappers raise otherwise) with outputs bit for bit those of a clean call.  The Mellinger
    gradient runs at (10, 4, 5, 3), where it takes the fused cost-only kernel; Nfabian at D = 5, where it takes the
    pack fallback."""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, K, D, B, S = 10, 4, 5, 3, 37, 80
    prob = m.Problem(N, r, K, D)
    _, times, dfix = _waypoints(oracle, N, K, D, B, 18000)
    pos5 = np.random.RandomState(18).uniform(-10, 10, size=(B, K + 1, 5))
    t_d, f_d, p5_d = _cuda(times), _cuda(dfix), _cuda(pos5)
    free_d = torch.empty((B, D, prob.n_free), dtype=torch.float64, device="cuda")
    c_d = solver.solve_linear(prob, t_d, f_d, d_free=free_d)
    coeffs, d_free = c_d.cpu().numpy(), free_d.cpu().numpy()
    cons = ((1, 2.0), (2, 3.0))
    v_max, a_max = 2.0, 3.0

    def solve():
        fr, st = _dev((B, D, prob.n_free)), _dev((B,), torch.int32)
        return solver.solve_linear(prob, t_d, f_d, d_free=fr, status=st), fr, st

    def nfabian():
        t, st = _dev((B, K)), _dev((B,), torch.int32)
        return solver.solve_waypoints_nfabian(N, r, p5_d, 3.0, 5.0, 6.5, seg_times_out=t, status=st), t, st

    def solve_host():
        c, fr, st = _host((B, K, D, N)), _host((B, D, prob.n_free)), _host((B,), np.int32)
        solver.solve_linear_host(prob, times, dfix, c, d_free=fr, status=st)
        return c, fr, st

    def nfabian_host():
        c, t, st = _host((B, K, 5, N)), _host((B, K)), _host((B,), np.int32)
        solver.solve_waypoints_nfabian_host(N, r, pos5, 3.0, 5.0, 6.5, c, seg_times_out=t, status=st)
        return c, t, st

    def coeffs_host():
        c = _host((B, K, D, N))
        solver.coeffs_from_constraints_host(prob, times, dfix, d_free, c)
        return (c,)

    def cost_host():
        c = _host((B,))
        solver.compute_cost_host(prob, times, coeffs, c)
        return (c,)

    def mellinger_host():
        c, g = _host((B,)), _host((B, K))
        solver.cost_gradient_mellinger_host(prob, times, dfix, c, g)
        return c, g

    def range_host():
        o, n, st = _host((B, S, 2, D)), _host((B,), np.int32), _host((B, S))
        solver.evaluate_range_host(times, coeffs, 0.1, 3.0, 0.05, (0, 2), o, n, sampling_times=st)
        return o, n, st

    def extrema_host():
        v, t, s, st = _host((B, 2)), _host((B, 2)), _host((B, 2), np.int32), _host((B,), np.int32)
        solver.max_magnitude_host(times, coeffs, (1, 2), v, t, s, st)
        return v, t, s, st

    def objective_host():
        c, o, tm, st = _host((B, K, D, N)), _host((B,)), _host((B, 3)), _host((B,), np.int32)
        solver.time_objective_host(prob, times, dfix, None, m.time_objective_params(constraints=cons), c, o, tm, st)
        return c, o, tm, st

    def scale_host():
        t, c, w, mx, st = _host((B, K)), _host((B, K, D, N)), _host((B,), np.int32), _host((B, 2)), _host((B,), np.int32)
        solver.scale_to_constraints_host(times, coeffs, v_max, a_max, t, c, w, mx, st)
        return t, c, w, mx, st

    def violation_host():
        c, t, w, mx, st = _host((B, K, D, N)), _host((B, K)), _host((B,), np.int32), _host((B, 2)), _host((B,), np.int32)
        solver.scale_times_with_violation_host(prob, times, dfix, v_max, a_max, c, t, w, mx, st)
        return c, t, w, mx, st

    cases = {
        "solve_linear": solve,
        "nfabian_pack_fallback": nfabian,
        "coeffs_from_constraints": lambda: (solver.coeffs_from_constraints(prob, t_d, f_d, free_d),),
        "compute_cost": lambda: (solver.compute_cost(prob, t_d, c_d),),
        "evaluate": lambda: (solver.evaluate(t_d, c_d, 1, 0.1, 0.05, S),),
        "evaluate_range": lambda: solver.evaluate_range(t_d, c_d, 0.1, 3.0, 0.05, (0, 2), S, True),
        "mellinger_fused": lambda: solver.cost_gradient_mellinger(prob, t_d, f_d),
        "max_magnitude": lambda: solver.max_magnitude(t_d, c_d, (1, 2)),
        "time_objective": lambda: solver.time_objective(prob, t_d, f_d, constraints=cons),
        "scale_to_constraints": lambda: solver.scale_to_constraints(t_d, c_d, v_max, a_max),
        "scale_times_with_violation": lambda: solver.scale_times_with_violation(prob, t_d, f_d, v_max, a_max),
        "solve_linear_host": solve_host,
        "nfabian_pack_fallback_host": nfabian_host,
        "coeffs_from_constraints_host": coeffs_host,
        "compute_cost_host": cost_host,
        "mellinger_fused_host": mellinger_host,
        "evaluate_range_host": range_host,
        "max_magnitude_host": extrema_host,
        "time_objective_host": objective_host,
        "scale_to_constraints_host": scale_host,
        "scale_times_with_violation_host": violation_host,
    }

    def run(call):
        outs = call()
        torch.cuda.synchronize()
        return [_np(x) for x in outs]

    failed = []
    for name, call in cases.items():
        clean = run(call)
        assert not solver.lib.mtg_device_alloc(solver.h, 1 << 50), "a 1 PiB allocation succeeded"
        try:
            stale = run(call)
        except RuntimeError as e:
            failed.append(f"{name}: {e}")
            continue
        if not all(same_bits(a, b) for a, b in zip(stale, clean)):
            failed.append(f"{name}: outputs differ from the clean call")
    assert not failed, "\n".join(failed)
