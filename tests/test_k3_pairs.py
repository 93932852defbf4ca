"""The chunked kernel K3 in warp pairs (twisted_chunked_pair_kernel) against the one-warp K3.

The paired form runs one tile's inward sweep beside the previous tile's outward sweep on one tile's resident blocks;
the slot of a vertex alternates with the tile's parity and the parking area has one half per parity.  It calls the
same sweep functions with the same arguments, so its coefficients, d_free and status must be bitwise equal to the
one-warp K3 (WAYPOINT_VARIANT = 5).  Each case proves by name which kernel ran, from the CUDA profiler in a child
process that makes the same calls (the route depends on the shape, B, alignment and options, not on the values), so
that this process never starts a profiler session of its own:
  * the default route of the headline shape (N = 10, r = 4, D = 3, K = 16) launches the paired form;
  * 3 pairs per SM forced:
    - the shapes of test_k3_parking.py, with a ragged batch where every pair runs at least three tiles, so that
      both slot maps repeat;
    - odd K (15, 17), forced chunks 1 and 2, and a chunk with nothing parked;
  * a batch of a single tile, and rows solved alone;
  * bad segment times (where NaN meets NaN only the NaN mask is compared: the bits of a NaN, its sign among them, are
    not part of the result).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_k3_parking import SHAPES
from test_large_k import same_bits
from test_resident_kernels import k3_id, kernel_id

PAIRS_PER_SM = 3  # forced in the cases below (the default route runs 2)
TILES_PER_PAIR = 3
N_ALONE = 64


def pair_id(N, r, D):
    return kernel_id("twisted_chunked_pair_kernel", N, r, D, 3)  # ring depth 3


# The child process: for each (N, r, D, K, B, options), the ids of the kernels one solve_linear launched
_ROUTES = r"""
import json, sys
import torch
import mav_trajectory_generation_b200 as m
from test_resident_kernels import launched_kernels
s = m.Solver(0)
out = []
for N, r, D, K, B, opts in json.loads(sys.stdin.read()):
    prob = m.Problem(N, r, K, D)
    t = torch.ones((B, K), dtype=torch.float64, device="cuda")
    f = torch.zeros((B, D, prob.n_fixed), dtype=torch.float64, device="cuda")
    for name, value in opts.items():
        s.set_option(getattr(m.capi, "OPT_" + name), value)
    _, ids = launched_kernels(lambda: s.solve_linear(prob, t, f))
    for name in opts:
        s.set_option(getattr(m.capi, "OPT_" + name), 0)
    out.append(ids)
print(json.dumps(out))
"""


def _routes(calls):
    """kernel ids launched by solve_linear for each (N, r, D, K, B, options), from a child process"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
    res = subprocess.run([sys.executable, "-c", _ROUTES], input=json.dumps(calls), capture_output=True, text=True,
                         env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


def _solve(solver, prob, t_d, f_d, **opts):
    """solve_linear with the options (each back to 0 afterwards) -> (coeffs, d_free, status) as numpy.  Outputs start
    as NaN / -1."""
    import torch
    import mav_trajectory_generation_b200 as m
    B = t_d.shape[0]
    coeffs = torch.full((B, prob.K, prob.D, prob.N), float("nan"), dtype=torch.float64, device="cuda")
    dfree = torch.full((B, prob.D, prob.n_free), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    try:
        for name, value in opts.items():
            solver.set_option(getattr(m.capi, "OPT_" + name), value)
        solver.solve_linear(prob, t_d, f_d, coeffs=coeffs, d_free=dfree, status=status)
        torch.cuda.synchronize()
    finally:
        for name in opts:
            solver.set_option(getattr(m.capi, "OPT_" + name), 0)
    return coeffs.cpu().numpy(), dfree.cpu().numpy(), status.cpu().numpy()


def _batch(oracle, N, D, K, B, seed, bad_times=False):
    rng = np.random.RandomState(seed)
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    sd[1::2] = 0.0
    if bad_times:  # one bad segment per affected row, at every position of the sweep
        for i, value in enumerate([0.0, -0.0, -1.0, np.nan, np.inf, -np.inf]):
            rows = np.arange(i, B, 7)
            times[rows, (rows // 7) % K] = value
    return times, oracle.waypoint_d_fixed(N, pos, sd, ed)


def _same_bits_or_both_nan(a, b):
    if a.dtype != np.float64:
        return same_bits(a, b)
    both = np.isnan(a) & np.isnan(b)
    return np.array_equal(np.isnan(a), np.isnan(b)) and same_bits(np.where(both, 0.0, a), np.where(both, 0.0, b))


def _compare(solver, N, r, D, K, times, dfix, label, opts=None, expect_ok=True):
    """the paired form (default route, with `opts`) against the one-warp K3, bitwise (with expect_ok False, up to the
    bits of NaNs); returns the paired result"""
    import torch
    import mav_trajectory_generation_b200 as m
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    B = times.shape[0]
    ids = _routes([[N, r, D, K, B, opts or {}], [N, r, D, K, B, dict(WAYPOINT_VARIANT=5)]])
    assert ids == [[pair_id(N, r, D)], [k3_id(N, r, D)]], f"{label}: launched {ids}, expected the paired, then the " \
                                                          "one-warp K3"
    got = _solve(solver, prob, t_d, f_d, **(opts or {}))
    ref = _solve(solver, prob, t_d, f_d, WAYPOINT_VARIANT=5)
    same = same_bits if expect_ok else _same_bits_or_both_nan
    for what, a, b in zip(("coefficients", "d_free", "status"), got, ref):
        assert same(a, b), f"{label}: {what} of the paired K3 differ from the one-warp K3"
    if expect_ok:
        assert (got[2] == 0).all(), f"{label}: non-zero status"
        assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all(), label
    return got, (prob, t_d, f_d)


def _many_tiles(sms):
    return TILES_PER_PAIR * PAIRS_PER_SM * sms * 16


@pytest.mark.gpu
def test_default_route_launches_pairs_at_the_headline_shape(solver, oracle):
    """no option set: nothing parked, two pairs per SM, many tiles per pair"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 7
    times, dfix = _batch(oracle, 10, 3, 16, B, 8100)
    _compare(solver, 10, 4, 3, 16, times, dfix, f"default route N=10 r=4 D=3 K=16 B={B}")


@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K", SHAPES, ids=["N{}r{}D{}-K{}".format(*s) for s in SHAPES])
def test_pairs_many_tiles_and_rows_alone(solver, oracle, N, r, D, K):
    """every pair runs >= 3 tiles of a ragged batch (3 pairs per SM forced, so that every shape takes the paired
    form); then the same rows alone, one tile per pair at most"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 5
    label = f"paired K3 N={N} r={r} D={D} K={K} B={B}"
    times, dfix = _batch(oracle, N, D, K, B, 8200 + 100 * N + 10 * D + K)
    got, (prob, t_d, f_d) = _compare(solver, N, r, D, K, times, dfix, label, dict(CTAS_PER_SM=6))
    rng = np.random.RandomState(K)
    rows = np.sort(np.concatenate([[0, B - 1], 1 + rng.choice(B - 2, N_ALONE - 2, replace=False)]))
    idx = torch.from_numpy(rows).cuda()
    ids = _routes([[N, r, D, K, len(rows), dict(CTAS_PER_SM=6)]])
    assert ids == [[pair_id(N, r, D)]], f"{label}: rows alone launched {ids}"
    alone = _solve(solver, prob, t_d[idx].contiguous(), f_d[idx].contiguous(), CTAS_PER_SM=6)
    for what, a, b in zip(("coefficients", "d_free", "status"), alone, got):
        assert same_bits(a, b[rows]), f"{label}: {what} of rows solved alone differ from the batch"


# (K, forced chunk): odd K on both sides of the headline, small chunks, and C = 7 = n at K = 16 (nothing parked)
CASES = [(15, 0), (17, 0), (16, 1), (16, 2), (16, 7), (33, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("K,chunk", CASES, ids=["K{}-C{}".format(*c) for c in CASES])
def test_pairs_odd_k_and_chunks(solver, oracle, K, chunk):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 9
    times, dfix = _batch(oracle, 10, 3, K, B, 8300 + K + 50 * chunk)
    _compare(solver, 10, 4, 3, K, times, dfix, f"paired K3 K={K} C={chunk} B={B}",
             dict(CHUNK_BLOCKS=chunk, CTAS_PER_SM=6))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [16, 5])
def test_pairs_single_tile(solver, oracle, B):
    times, dfix = _batch(oracle, 10, 3, 16, B, 8400 + B)
    _compare(solver, 10, 4, 3, 16, times, dfix, f"paired K3 one tile B={B}")


@pytest.mark.gpu
def test_pairs_bad_segment_times(solver, oracle):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 3
    times, dfix = _batch(oracle, 10, 3, 16, B, 8500, bad_times=True)
    got, _ = _compare(solver, 10, 4, 3, 16, times, dfix, "paired K3 bad segment times", expect_ok=False)
    bad = ~np.isfinite(times).all(axis=1) | (times <= 0).any(axis=1)
    assert (got[2][bad] != 0).all() and (got[2][~bad] == 0).all(), "status does not flag exactly the bad rows"
