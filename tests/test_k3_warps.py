"""The chunked kernel K3 at every warp layout: one-warp and four-warp CTAs, capped warps per SM, L2 hints on and off.

K3's warps are independent: warps per CTA (MTG_OPT_CHUNK_WARPS), the cap on resident warps per SM
(MTG_OPT_CTAS_PER_SM) and the evict-first L2 hints (MTG_OPT_L2_HINTS) change which warp runs which tile, how the
parking area is laid out and what L2 keeps, never the arithmetic.  The batch is ragged and large enough for every
warp to run at least three tiles at 8 warps per SM.  At each shape of test_k3_parking.py, coefficients, d_free and
status must be bitwise equal:
  * across W = 1 and W = 4;
  * across warp caps 4, 6 and as many as fit;
  * with the hints on and off;
  * to the same rows solved alone.
"""
import numpy as np
import pytest

from test_k3_parking import SHAPES, _same_bits
from test_large_k import options

WARPS_PER_SM = 8
TILES_PER_WARP = 3
N_ALONE = 256

# (W, warp cap, L2 hints on): the auto layout first, every other one is compared with it
# (a cap of 8 is as many as fit)
LAYOUTS = [(0, 0, 0), (1, 8, 0), (4, 0, 0), (1, 4, 0), (1, 6, 0), (4, 8, 0), (1, 8, 1), (4, 0, 1)]


def _solve(solver, prob, t_d, f_d, warps, cap, hints):
    import torch
    B = t_d.shape[0]
    coeffs = torch.full((B, prob.K, prob.D, prob.N), float("nan"), dtype=torch.float64, device="cuda")
    dfree = torch.full((B, prob.D, prob.n_free), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    with options(solver, WAYPOINT_VARIANT=5, CHUNK_WARPS=warps, CTAS_PER_SM=cap, L2_HINTS=hints):
        solver.solve_linear(prob, t_d, f_d, coeffs=coeffs, d_free=dfree, status=status)
        torch.cuda.synchronize()
    return coeffs, dfree, status


@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K", SHAPES, ids=["N{}r{}D{}-K{}".format(*s) for s in SHAPES])
def test_k3_warp_layouts(solver, oracle, N, r, D, K):
    import torch
    import mav_trajectory_generation_b200 as m
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = TILES_PER_WARP * WARPS_PER_SM * sms * 16 + 11  # ragged last tile
    seed = 9100 + 100 * N + 10 * D + K
    pos, times = oracle.make_waypoint_batch(K, D, B, base_seed=seed)
    rng = np.random.RandomState(seed)
    sd = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    ed = rng.uniform(-1, 1, size=(B, N // 2 - 1, D))
    sd[1::2] = 0.0
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    label = f"K3 N={N} r={r} D={D} K={K} B={B}"

    out, dfree, status = _solve(solver, prob, t_d, f_d, *LAYOUTS[0])
    assert int((status != 0).sum().item()) == 0, f"{label}: non-zero status"
    assert bool(torch.isfinite(out).all().item()) and bool(torch.isfinite(dfree).all().item()), label

    for lay in LAYOUTS[1:]:
        what = "W={} warp cap={} hints {}".format(lay[0], lay[1], "on" if lay[2] else "off")
        o2, f2, s2 = _solve(solver, prob, t_d, f_d, *lay)
        assert _same_bits(o2, out), f"{label}: coefficients differ at {what}"
        assert _same_bits(f2, dfree), f"{label}: d_free differs at {what}"
        assert _same_bits(s2, status), f"{label}: status differs at {what}"
        del o2, f2, s2

    # the same rows alone (one warp tile at most per CTA): first, last (ragged tile) and a random sample
    rows = np.sort(np.concatenate([[0, B - 1], 1 + rng.choice(B - 2, N_ALONE - 2, replace=False)]))
    idx = torch.from_numpy(rows).cuda()
    for lay in (LAYOUTS[1], LAYOUTS[2]):
        o_s, f_s, s_s = _solve(solver, prob, t_d[idx].contiguous(), f_d[idx].contiguous(), *lay)
        assert _same_bits(o_s, out[idx]), f"{label}: rows solved alone (W={lay[0]}) differ from the batch"
        assert _same_bits(f_s, dfree[idx]), f"{label}: d_free of rows solved alone (W={lay[0]}) differs"
        assert _same_bits(s_s, status[idx]), f"{label}: status of rows solved alone (W={lay[0]}) differs"
