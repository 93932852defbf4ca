"""The chunked kernel K3 in warp pairs (twisted_chunked_pair_kernel) at every compiled (N, r, D) of the waypoint
registry.

The paired form is the default route of plain waypoint solves at the K where the resident kernels no longer fit
(rule 5 of plan_waypoint, then plan_chunked), and each registry row has its own instantiation.  Everything in it that
depends on the shape -- ChunkedPairLayout (prologue, final-segment inputs, the h*D handoff, the block slots), the slot
map that alternates with the tile's parity, the parking columns of each parity half and the outward warp's staging
tile -- is checked here at every row:
  1. the default route map over K in ROUTE_K and B in ROUTE_B, as observed on an H100 80GB HBM3 (DEFAULT_ROUTES);
  2. the paired form (3 pairs per SM forced) bitwise equal to the one-warp K3 on a ragged batch where every pair runs
     >= 3 tiles, at the four K of PAIR_K (the smallest K at which the paired form runs, odd and even K, K = 16), on the
     Nfabian and the log-uniform times, half of the rows with non-zero start and end derivatives; 64 of its rows
     solved alone give the same bits;
  3. blocks parked in both parity halves: forced chunks 1 and 3 at K = 16 (or the smallest paired K beyond), and
     chunk 3 at K = 33 for one shape per N;
  4. 128 rows of each case of 2 against the binary128 solve (check_parity, d_free as in
     test_chunked_kernel_every_specialisation);
  5. a partial tile (B = 5) and one full tile (B = 16) at the default route, where that route is the paired form;
  6. bad segment times at one shape per N: the bits of K3 up to NaN bits, status on exactly the bad rows.
Every case proves by name which kernel ran; the routes of all cases come from one child process (see _routes in
test_k3_pairs.py).
"""
import json

import numpy as np
import pytest

from test_gpu_parity import check_parity, global_rel_err
from test_k3_pairs import _batch, _many_tiles, _routes, _same_bits_or_both_nan, _solve, pair_id
from test_large_k import WAYPOINT_SHAPES, oracle_solve, rel_err_free, same_bits, waypoint_fixture
from test_resident_kernels import k3_id, kernel_id

PAIRS = dict(CTAS_PER_SM=6)  # 3 pairs per SM at most: every shape takes the paired form at the K of PAIR_K
K3 = dict(WAYPOINT_VARIANT=5)
N_PARITY = 128
N_ALONE = 64

# ---------------------------------------------------------------------------------------------------------------------
# 1. The default route map

ROUTE_K = (3, 4, 7, 9, 12, 15, 16, 17)
ROUTE_B = (100, 112)  # B % 16 != 0 rules v5 out (rule 3 of plan_waypoint); B % 16 == 0 admits it

# The kernel family the default route (no option set) launches for each registry row, at ROUTE_K, for B = 100 and
# B = 112.  Observed on an H100 80GB HBM3 (132 SMs).  The rule of plan_waypoint (csrc/mtg_capi.cu) that gives each:
#   v5  rule 3: B % 16 == 0, 16-byte aligned inputs and a v5 instantiation, >= 2 resident CTAs per SM
#   v4  rule 4: K <= 8 and a v4 instantiation, >= 2 resident CTAs per SM
#   v3  rule 5: v3's factor leaves >= 2 CTAs per SM
#   P   rule 5, then plan_chunked: v3 does not fit, nmax = ceil(K/2) - 1 <= kPairMaxBlocks = 7 and kAutoPairs = 2 pairs
#       per SM fit with every block resident -- the paired form, twisted_chunked_pair_kernel<N, r, D, 3>
#   K3  rule 5, then plan_chunked: the one-warp K3, twisted_chunked_kernel<N, r, D, 3, 1> (K = 17: nmax = 8 > 7)
DEFAULT_ROUTES = {
    (10, 4, 3): ("v4 v4 P P P P P K3", "v5 v5 P P P P P K3"),
    (10, 4, 1): ("v4 v4 v4 v3 v3 P P K3", "v5 v5 v5 v5 v5 P P K3"),
    (10, 4, 2): ("v3 v3 v3 v3 P P P K3", "v3 v3 v3 v3 P P P K3"),
    (10, 4, 4): ("v3 v3 P P P P P K3", "v3 v3 P P P P P K3"),
    (10, 3, 3): ("v4 v4 P P P P P K3", "v5 v5 P P P P P K3"),
    (10, 3, 1): ("v3 v3 v3 v3 v3 P P K3", "v3 v3 v3 v3 v3 P P K3"),
    (10, 2, 3): ("v4 v4 P P P P P K3", "v5 v5 P P P P P K3"),
    (10, 2, 1): ("v3 v3 v3 v3 v3 P P K3", "v3 v3 v3 v3 v3 P P K3"),
    (8, 3, 3): ("v4 v4 v4 v3 P P P K3", "v5 v5 v5 v5 P P P K3"),
    (8, 3, 1): ("v3 v3 v3 v3 v3 v3 v3 v3", "v3 v3 v3 v3 v3 v3 v3 v3"),  # v3 fits up to K = 20
    (8, 3, 2): ("v3 v3 v3 v3 v3 P P K3", "v3 v3 v3 v3 v3 P P K3"),
    (8, 3, 4): ("v3 v3 v3 P P P P K3", "v3 v3 v3 P P P P K3"),
    (12, 5, 3): ("v4 v4 P P P P P K3", "v5 v5 P P P P P K3"),
    (12, 5, 1): ("v3 v3 v3 v3 P P P K3", "v3 v3 v3 v3 P P P K3"),
    (12, 5, 4): ("v3 v3 P P P P P K3", "v3 v3 P P P P P K3"),
    (6, 2, 3): ("v3 v3 v3 v3 v3 P P K3", "v3 v3 v3 v3 v3 P P K3"),
    (6, 2, 1): ("v3 v3 v3 v3 v3 v3 v3 v3", "v3 v3 v3 v3 v3 v3 v3 v3"),  # v3 fits up to K = 30
}

_FAMILIES = {"twisted_chunked_pair_kernel": "P", "twisted_chunked_kernel": "K3", "twisted_tmem_kernel": "v3",
             "twisted_tmem_v4_kernel": "v4", "twisted_tmem_v5_kernel": "v5"}


def _check_same_as_k3(got, ref, label, expect_ok=True):
    """(coeffs, d_free, status) of the paired form bitwise equal to those of the one-warp K3 (with expect_ok False, up
    to the bits of NaNs), as _compare of test_k3_pairs; with expect_ok, status 0 and finite outputs"""
    same = same_bits if expect_ok else _same_bits_or_both_nan
    for what, a, b in zip(("coefficients", "d_free", "status"), got, ref):
        assert same(a, b), f"{label}: {what} of the paired K3 differ from the one-warp K3"
    if expect_ok:
        assert (got[2] == 0).all(), f"{label}: non-zero status"
        assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all(), label


def _sid(shape):
    return "N{}r{}D{}".format(*shape)


def _family(ids, N, r, D):
    """the DEFAULT_ROUTES code of one launch of the instantiation of (N, r, D); anything else as the ids themselves"""
    if len(ids) == 1:
        for base, code in _FAMILIES.items():
            if ids[0].startswith(kernel_id(base, N, r, D)[:-1] + ","):
                return code
    return "+".join(ids) or "nothing"


def _default_route(shape, K, B):
    """the committed default route of (shape, K, B): B stands for its class (B % 16 != 0 or == 0), as the route
    depends on B only through that test"""
    if shape not in DEFAULT_ROUTES:
        return None
    return DEFAULT_ROUTES[shape][int(B % 16 == 0)].split()[ROUTE_K.index(K)]


# ---------------------------------------------------------------------------------------------------------------------
# The cases of 2-6

# CTAS_PER_SM does not override rules 3-5 of plan_waypoint: below the K at which v3's factor no longer leaves 2 CTAs per
# SM (and where v4 takes K <= 8), a solve runs v3 or v4 whatever the option, so the paired form cannot run at K = 3 or 4
# at any registry shape.  PAIR_K: per row, the smallest K at which the paired form runs with CTAS_PER_SM = 6 (B = 100;
# it runs at every K above, up to 100 -- observed on an H100 80GB HBM3), the next K and two more, K = 16 among them
# wherever the paired form runs there (beyond K = 16, nmax > 7: blocks are parked at the auto chunk).
PAIR_K = {
    (10, 4, 3): (7, 8, 11, 16), (10, 4, 1): (15, 16, 17, 24), (10, 4, 2): (11, 12, 13, 16), (10, 4, 4): (7, 8, 13, 16),
    (10, 3, 3): (7, 8, 9, 16), (10, 3, 1): (15, 16, 17, 20), (10, 2, 3): (7, 8, 15, 16), (10, 2, 1): (15, 16, 19, 24),
    (8, 3, 3): (11, 12, 13, 16), (8, 3, 1): (21, 22, 23, 33), (8, 3, 2): (15, 16, 17, 22), (8, 3, 4): (9, 10, 11, 16),
    (12, 5, 3): (7, 8, 9, 16), (12, 5, 1): (11, 12, 15, 16), (12, 5, 4): (5, 6, 7, 16), (6, 2, 3): (15, 16, 17, 25),
    (6, 2, 1): (31, 32, 33, 40),
}
assert list(PAIR_K) == WAYPOINT_SHAPES

KINDS = ("nfabian", "mixed")
PAIR_CASES = [(shape, K, KINDS[(j + i) % 2]) for i, shape in enumerate(WAYPOINT_SHAPES)
              for j, K in enumerate(PAIR_K[shape])]
CHUNKS = (1, 3)
# (N, r, D, K, forced chunks): every row at K = 16, or at its smallest paired K where that is larger; one row per N at
# K = 33, where 13 blocks per lane are parked
PARK_CASES = [(*shape, max(16, PAIR_K[shape][0]), CHUNKS) for shape in WAYPOINT_SHAPES] + \
             [(6, 2, 3, 33, (3,)), (8, 3, 2, 33, (3,)), (10, 4, 4, 33, (3,)), (12, 5, 3, 33, (3,))]
SINGLE_TILE_K = 16
# a partial tile and one full tile, where the default route at K = 16 is the paired form
SINGLE_TILE_CASES = [(shape, B) for shape in WAYPOINT_SHAPES for B in (5, 16)
                     if _default_route(shape, SINGLE_TILE_K, B) == "P"]
# (N, r, D, K, forced chunk): one row per N, two with blocks parked
BAD_CASES = [(6, 2, 3, 15, 0), (8, 3, 3, 16, 2), (10, 3, 1, 15, 2), (12, 5, 4, 16, 0)]


def _bad_opts(chunk):
    return dict(PAIRS, CHUNK_BLOCKS=chunk) if chunk else PAIRS


def _seed(N, r, D, K, base):
    return base + 1000 * N + 100 * r + 10 * D + K


def _case_calls(sms):
    """every call of the cases of 2-6, as _routes takes it: [N, r, D, K, B, options]"""
    big, bad = _many_tiles(sms) + 5, _many_tiles(sms) + 3
    out = []
    for (N, r, D), K, _ in PAIR_CASES:
        out += [[N, r, D, K, big, PAIRS], [N, r, D, K, big, K3], [N, r, D, K, N_ALONE, PAIRS]]
    for N, r, D, K, chunks in PARK_CASES:
        out += [[N, r, D, K, big, dict(PAIRS, CHUNK_BLOCKS=c)] for c in chunks] + [[N, r, D, K, big, K3]]
    for (N, r, D), B in SINGLE_TILE_CASES:
        out += [[N, r, D, SINGLE_TILE_K, B, {}], [N, r, D, SINGLE_TILE_K, B, K3]]
    for N, r, D, K, c in BAD_CASES:
        out += [[N, r, D, K, bad, _bad_opts(c)], [N, r, D, K, bad, K3]]
    return out


def _route_calls():
    return [[N, r, D, K, B, {}] for (N, r, D) in WAYPOINT_SHAPES for K in ROUTE_K for B in ROUTE_B]


def _key(call):
    return json.dumps(call, sort_keys=True)


@pytest.fixture(scope="module")
def routes():
    """the kernel ids of every call of this file (the route map's and those of the cases), from one child process"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    calls = {_key(c): c for c in _route_calls() + _case_calls(sms)}
    ids = _routes(list(calls.values()))
    return dict(sms=sms, ids=dict(zip(calls, ids)))


def _assert_ran(routes, N, r, D, K, B, opts, want, label):
    ids = routes["ids"][_key([N, r, D, K, B, opts])]
    assert ids == [want], f"{label}: {opts or 'the default route'} launched {ids}, expected {want}"


# ---------------------------------------------------------------------------------------------------------------------
# 1.

@pytest.mark.gpu
def test_default_route_map(routes):
    """The default route of every registry row at ROUTE_K x ROUTE_B is DEFAULT_ROUTES: each paired instantiation that
    the default route reaches is listed, and a routing change has to update the map on purpose.  At K = 17 (nmax = 8)
    the route is never the paired form."""
    seen = {}
    for N, r, D in WAYPOINT_SHAPES:
        seen[(N, r, D)] = tuple(" ".join(_family(routes["ids"][_key([N, r, D, K, B, {}])], N, r, D) for K in ROUTE_K)
                                for B in ROUTE_B)
    table = "\n".join(f"    {shape}: {codes}," for shape, codes in seen.items())
    for shape, codes in seen.items():
        for B, row in zip(ROUTE_B, codes):
            assert row.split()[ROUTE_K.index(17)] != "P", f"{_sid(shape)} B={B}: the paired form at K = 17"
    assert seen == DEFAULT_ROUTES, f"default routes (K = {ROUTE_K}; B = {ROUTE_B}) differ from DEFAULT_ROUTES:\n{table}"


# ---------------------------------------------------------------------------------------------------------------------
# 2 and 4. Paired against the one-warp K3, rows alone, and against binary128

# Rows where rule 1 of check_parity does not hold for the sweep arithmetic, which the paired form shares bit for bit
# with K3: on the 1-D (12, 5, 1) Nfabian fixture at K = 16 a trajectory lands 1.8e-8 from exact where the
# reference-order oracle is 3.6e-9 from it -- the loss of fp64 elimination that SWEEP_LOSS_CASES of test_large_k
# describes at K = 50 (d_free as far from exact on the same trajectory).  There each trajectory is held to the rule of
# check_parity_or_sweep_loss, the banded kernel sharing no code with the sweep:
#     err(CUDA, exact) <= max(2e-10, 2 * err(oracle, exact), 4 * err(banded generic kernel, exact)),
# and d_free to the rule of test_chunked_kernel_every_specialisation or 4 * the banded kernel's d_free error.
LOSS_SHAPES = {(12, 5, 1)}


def _banded(solver, prob, t_d, f_d):
    """(coefficients, d_free) of the banded generic kernel: an output that is only 8-byte aligned takes it (as
    banded_solve of test_large_k)"""
    import torch
    B = t_d.shape[0]
    big = torch.full((B * prob.K * prob.D * prob.N + 1,), float("nan"), dtype=torch.float64, device="cuda")
    out = big[1:].view(B, prob.K, prob.D, prob.N)
    assert out.data_ptr() % 16 == 8
    dfree = torch.full((B, prob.D, prob.n_free), float("nan"), dtype=torch.float64, device="cuda")
    solver.solve_linear(prob, t_d, f_d, coeffs=out, d_free=dfree)
    torch.cuda.synchronize()
    return out.cpu().numpy(), dfree.cpu().numpy()

@pytest.mark.gpu
@pytest.mark.parametrize("shape,K,times_kind", PAIR_CASES,
                         ids=[f"{_sid(s)}-K{K}-{kind}" for s, K, kind in PAIR_CASES])
def test_pairs_every_shape(solver, oracle, routes, shape, K, times_kind):
    """3 pairs per SM forced, every pair running >= 3 tiles: bitwise equal to the one-warp K3, rows alone bitwise
    equal to the batch, and 128 rows against binary128"""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, D = shape
    B = _many_tiles(routes["sms"]) + 5
    label = f"paired K3 N={N} r={r} D={D} K={K} B={B} {times_kind}"
    _assert_ran(routes, N, r, D, K, B, PAIRS, pair_id(N, r, D), label)
    _assert_ran(routes, N, r, D, K, B, K3, k3_id(N, r, D), label)
    pos, times, sd, ed = waypoint_fixture(oracle, N, K, D, B, times_kind, _seed(N, r, D, K, 70000))
    dfix = oracle.waypoint_d_fixed(N, pos, sd, ed)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    got = _solve(solver, prob, t_d, f_d, **PAIRS)
    _check_same_as_k3(got, _solve(solver, prob, t_d, f_d, **K3), label)

    # rows alone: at most one tile per pair
    rng = np.random.RandomState(K)
    rows = np.sort(np.concatenate([[0, B - 1], 1 + rng.choice(B - 2, N_ALONE - 2, replace=False)]))
    _assert_ran(routes, N, r, D, K, N_ALONE, PAIRS, pair_id(N, r, D), label + " rows alone")
    idx = torch.from_numpy(rows).cuda()
    alone = _solve(solver, prob, t_d[idx].contiguous(), f_d[idx].contiguous(), **PAIRS)
    for what, a, b in zip(("coefficients", "d_free", "status"), alone, got):
        assert same_bits(a, b[rows]), f"{label}: {what} of rows solved alone differ from the batch"

    # binary128 on the first, the last and random rows
    rows = np.sort(np.concatenate([[0, B - 1], 1 + rng.choice(B - 2, N_PARITY - 2, replace=False)]))
    idx = torch.from_numpy(rows).cuda()
    exact, exact_free, _ = oracle.exact_solve_batch(N, r, times[rows], dfix[rows], want_free=True)
    ref, ref_free = oracle_solve(oracle, N, r, pos[rows], times[rows], sd[rows], ed[rows])
    e_f, e_of = rel_err_free(got[1][rows], exact_free), rel_err_free(ref_free, exact_free)
    flat = times_kind == "nfabian" and N <= 10
    bound_free = 1e-9 if flat else np.maximum(1e-9, 2.0 * e_of)
    if shape not in LOSS_SHAPES:
        check_parity(got[0][rows], ref, exact, label)
    else:
        gen, gen_free = _banded(solver, prob, t_d[idx].contiguous(), f_d[idx].contiguous())
        assert np.isfinite(gen).all() and np.isfinite(gen_free).all(), label
        e_ge, e_oe, e_be = global_rel_err(got[0][rows], exact), global_rel_err(ref, exact), global_rel_err(gen, exact)
        bad = e_ge > np.maximum(2e-10, np.maximum(2.0 * e_oe, 4.0 * e_be))
        assert not bad.any(), (f"{label}: CUDA vs exact {e_ge[bad].max():.3e} on trajectory {int(np.argmax(bad))} "
                               f"(oracle {e_oe[np.argmax(bad)]:.3e}, banded generic kernel {e_be[np.argmax(bad)]:.3e})")
        bound_free = np.maximum(bound_free, 4.0 * rel_err_free(gen_free, exact_free))
    bad = e_f > bound_free
    assert not bad.any(), f"{label}: d_free vs exact {e_f[bad].max():.3e} (oracle vs exact {e_of[bad].max():.3e})"


# ---------------------------------------------------------------------------------------------------------------------
# 3. Parked blocks in both parity halves

@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K,chunks", PARK_CASES, ids=["N{}r{}D{}-K{}".format(*c[:4]) for c in PARK_CASES])
def test_pairs_parked_every_shape(solver, oracle, routes, N, r, D, K, chunks):
    """forced small chunks: tile j parks its outer blocks in the half of parity j % 2 while tile j-1 refills from the
    other; every pair runs >= 3 tiles, so that both halves are written and read twice"""
    import torch
    import mav_trajectory_generation_b200 as m
    B = _many_tiles(routes["sms"]) + 5
    times, dfix = _batch(oracle, N, D, K, B, _seed(N, r, D, K, 71000))
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    label = f"paired K3 N={N} r={r} D={D} K={K} B={B}"
    _assert_ran(routes, N, r, D, K, B, K3, k3_id(N, r, D), label)
    ref = _solve(solver, prob, t_d, f_d, **K3)
    for c in chunks:
        opts = dict(PAIRS, CHUNK_BLOCKS=c)
        _assert_ran(routes, N, r, D, K, B, opts, pair_id(N, r, D), f"{label} chunk {c}")
        _check_same_as_k3(_solve(solver, prob, t_d, f_d, **opts), ref, f"{label} chunk {c}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. One tile at the default route

@pytest.mark.gpu
@pytest.mark.parametrize("shape,B", SINGLE_TILE_CASES, ids=[f"{_sid(s)}-B{B}" for s, B in SINGLE_TILE_CASES])
def test_pairs_single_tile_default_route(solver, oracle, routes, shape, B):
    """a partial tile and one full tile at K = 16 without options, where DEFAULT_ROUTES has the paired form there:
    bitwise equal to the one-warp K3"""
    import torch
    import mav_trajectory_generation_b200 as m
    N, r, D = shape
    label = f"paired K3 default route N={N} r={r} D={D} K={SINGLE_TILE_K} B={B}"
    _assert_ran(routes, N, r, D, SINGLE_TILE_K, B, {}, pair_id(N, r, D), label)
    _assert_ran(routes, N, r, D, SINGLE_TILE_K, B, K3, k3_id(N, r, D), label)
    times, dfix = _batch(oracle, N, D, SINGLE_TILE_K, B, _seed(N, r, D, B, 72000))
    prob = m.Problem(N, r, SINGLE_TILE_K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    _check_same_as_k3(_solve(solver, prob, t_d, f_d), _solve(solver, prob, t_d, f_d, **K3), label)


# ---------------------------------------------------------------------------------------------------------------------
# 6. Bad segment times

@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K,chunk", BAD_CASES, ids=["N{}r{}D{}-K{}-C{}".format(*c) for c in BAD_CASES])
def test_pairs_bad_segment_times_every_n(solver, oracle, routes, N, r, D, K, chunk):
    """0, -0, -1, NaN, +inf, -inf in one segment of 6 rows in 7, at every position of the sweep: the bits of K3 up to
    the bits of NaNs, and STATUS_BAD_TIME on exactly the bad rows"""
    import torch
    import mav_trajectory_generation_b200 as m
    B = _many_tiles(routes["sms"]) + 3
    opts = _bad_opts(chunk)
    label = f"paired K3 bad segment times N={N} r={r} D={D} K={K} chunk={chunk} B={B}"
    _assert_ran(routes, N, r, D, K, B, opts, pair_id(N, r, D), label)
    _assert_ran(routes, N, r, D, K, B, K3, k3_id(N, r, D), label)
    times, dfix = _batch(oracle, N, D, K, B, _seed(N, r, D, K, 73000), bad_times=True)
    prob = m.Problem(N, r, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    got = _solve(solver, prob, t_d, f_d, **opts)
    _check_same_as_k3(got, _solve(solver, prob, t_d, f_d, **K3), label, expect_ok=False)
    bad = ~np.isfinite(times).all(axis=1) | (times <= 0).any(axis=1)
    assert bad.sum() == B - B // 7, label  # the fixture: every row but one in 7
    assert (got[2][bad] & m.STATUS_BAD_TIME != 0).all() and (got[2][~bad] == 0).all(), \
        f"{label}: status does not flag exactly the bad rows"
