"""The chunked kernel K3 over batches where every resident warp runs several tiles.

K3 parks the outer vertex blocks of each lane's sweep in a global area that every thread reuses from tile to tile,
and prefetches the next tile's prologue inputs at the end of a tile.  Both can only go wrong when a warp runs more
than one tile, so the batch here is large enough for every resident warp to run at least three tiles, and ragged.
Checked at each shape:
  * the same rows solved alone (a small batch) are bitwise equal to the rows of the large batch;
  * forced chunks 1, 2 and auto give bitwise equal coefficients, d_free and status;
  * status is zero everywhere;
  * 256 sampled rows pass check_parity against the binary128 solve.
"""
import numpy as np
import pytest

from test_gpu_parity import check_parity
from test_large_k import oracle_solve, options

# (N, r, D, K): the headline shape at K = 16 and 50, and the shape of K3 with the most register pressure
SHAPES = [(10, 4, 3, 16), (10, 4, 3, 50), (12, 5, 4, 16)]
# K3 is launched at two CTAs of 4 warps per SM at most (__launch_bounds__(128, 2), about 250 registers per thread)
K3_WARPS_PER_SM = 2 * 4
TILES_PER_WARP = 3
N_SAMPLE = 256


def _solve(solver, prob, t_d, f_d, chunk):
    """K3 at a forced chunk (0 = auto) -> (coeffs, d_free, status) on the device; outputs start as NaN / -1"""
    import torch
    B = t_d.shape[0]
    coeffs = torch.full((B, prob.K, prob.D, prob.N), float("nan"), dtype=torch.float64, device="cuda")
    dfree = torch.full((B, prob.D, prob.n_free), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    with options(solver, WAYPOINT_VARIANT=5, CHUNK_BLOCKS=chunk):
        solver.solve_linear(prob, t_d, f_d, coeffs=coeffs, d_free=dfree, status=status)
        torch.cuda.synchronize()
    return coeffs, dfree, status


def _same_bits(a, b):
    import torch
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == torch.float64:
        a, b = a.contiguous().view(torch.int64), b.contiguous().view(torch.int64)
    return torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K", SHAPES, ids=["N{}r{}D{}-K{}".format(*s) for s in SHAPES])
def test_k3_many_tiles_per_warp(solver, oracle, N, r, D, K):
    import torch
    import mav_trajectory_generation_b200 as m
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = TILES_PER_WARP * K3_WARPS_PER_SM * sms * 16 + 5  # ragged last tile
    seed = 7000 + 100 * N + 10 * D + K
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    rng = np.random.RandomState(seed)
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    sd[1::2] = 0.0
    ed[1::2] = 0.0
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    label = f"K3 N={N} r={r} D={D} K={K} B={B}"

    out, dfree, status = _solve(solver, prob, t_d, f_d, 0)
    assert int((status != 0).sum().item()) == 0, f"{label}: non-zero status"
    assert bool(torch.isfinite(out).all().item()) and bool(torch.isfinite(dfree).all().item()), label

    # forced chunks
    for c in (1, 2):
        o2, f2, s2 = _solve(solver, prob, t_d, f_d, c)
        assert _same_bits(o2, out), f"{label}: coefficients differ with chunk {c}"
        assert _same_bits(f2, dfree), f"{label}: d_free differs with chunk {c}"
        assert _same_bits(s2, status), f"{label}: status differs with chunk {c}"
        del o2, f2, s2

    # the same rows alone: first, last (ragged tile) and a random sample
    rows = np.sort(np.concatenate([[0, B - 1], 1 + rng.choice(B - 2, N_SAMPLE - 2, replace=False)]))
    idx = torch.from_numpy(rows).cuda()
    o_s, f_s, s_s = _solve(solver, prob, t_d[idx].contiguous(), f_d[idx].contiguous(), 0)
    assert _same_bits(o_s, out[idx]), f"{label}: rows solved alone differ from the same rows in the batch"
    assert _same_bits(f_s, dfree[idx]), f"{label}: d_free of rows solved alone differs"
    assert _same_bits(s_s, status[idx]), f"{label}: status of rows solved alone differs"

    # parity of the sampled rows against the binary128 solve
    exact, _, _ = oracle.exact_solve_batch(N, r, times[rows], dfix[rows], want_free=True)
    ref, _ = oracle_solve(oracle, N, r, pos[rows], times[rows], sd[rows], ed[rows])
    check_parity(out[idx].cpu().numpy(), ref, exact, label)
