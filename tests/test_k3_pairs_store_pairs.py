"""The paired chunked kernel's coefficient stores (TmaPairEmitter) against the one-warp K3.

The outward warp of twisted_chunked_pair_kernel stores two consecutive global segments (2i, 2i+1) per 16-row box and
a segment whose partner belongs to the other half alone, from two staging buffers per half.  Which segments pair up
depends on K: n = ceil(K/2) - 1 even leaves the forward half's first segment alone, ceil(K/2) odd the backward half's
first one, K odd its last one, and at odd K the backward half is idle in the first outward step.  Every case here is
bitwise against the one-warp K3 (WAYPOINT_VARIANT = 5) and proves by name which kernels ran (_routes of
test_k3_pairs.py, from a child process):
  * every K from 7 to 16 at the headline shape (N = 10, r = 4, D = 3), 3 pairs per SM asked for, on a ragged batch
    where every pair runs at least three tiles, and K = 17 and 24, where blocks are parked; K = 15 and 16 at D = 1.
    Below K = 7 no row that stores pairs runs the paired form (v3 or v4 takes those K whatever the options: see
    test_k3_pairs_every_shape.py), and rows with D*N > 32 store one segment per box as before;
  * an output at an 8-byte offset, which the TMA cannot store to: it goes to the banded generic kernel, which agrees
    with the paired form to 1e-10 of each trajectory's largest coefficient;
  * the headline's default route still launches twisted_chunked_pair_kernel<10,4,3,3>.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_k3_pairs import _batch, _compare, _many_tiles, pair_id

PAIRS = dict(CTAS_PER_SM=6)
# (N, r, D, K)
EVERY_K = [(10, 4, 3, K) for K in range(7, 17)] + [(10, 4, 3, 17), (10, 4, 3, 24), (10, 4, 1, 15), (10, 4, 1, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,r,D,K", EVERY_K, ids=["N{}r{}D{}-K{}".format(*c) for c in EVERY_K])
def test_store_pairs_every_k(solver, oracle, N, r, D, K):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 11
    times, dfix = _batch(oracle, N, D, K, B, 8600 + 100 * N + K)
    _compare(solver, N, r, D, K, times, dfix, f"paired K3 stores N={N} r={r} D={D} K={K} B={B}", PAIRS)


@pytest.mark.gpu
def test_store_pairs_default_route_headline(solver, oracle):
    """no option set at the headline shape: the paired form, bitwise equal to the one-warp K3"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 13
    times, dfix = _batch(oracle, 10, 3, 16, B, 8700)
    _compare(solver, 10, 4, 3, 16, times, dfix, f"paired K3 stores, default route B={B}")
    assert pair_id(10, 4, 3) == "twisted_chunked_pair_kernel<10,4,3,3>"


# The child process: the kernel ids that one solve_linear into an output at an 8-byte offset launched
_OFFSET_ROUTE = r"""
import json, sys
import torch
import mav_trajectory_generation_b200 as m
from test_resident_kernels import launched_kernels
N, r, D, K, B = json.loads(sys.stdin.read())
s = m.Solver(0)
prob = m.Problem(N, r, K, D)
t = torch.ones((B, K), dtype=torch.float64, device="cuda")
f = torch.zeros((B, D, prob.n_fixed), dtype=torch.float64, device="cuda")
big = torch.empty((B * K * D * N + 1,), dtype=torch.float64, device="cuda")
out = big[1:].view(B, K, D, N)
assert out.data_ptr() % 16 == 8
_, ids = launched_kernels(lambda: s.solve_linear(prob, t, f, coeffs=out))
print(json.dumps(ids))
"""


@pytest.mark.gpu
def test_store_pairs_offset_output_takes_the_banded_kernel(solver, oracle):
    import torch
    N, r, D, K = 10, 4, 3, 16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = _many_tiles(sms) + 3
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
    res = subprocess.run([sys.executable, "-c", _OFFSET_ROUTE], input=json.dumps([N, r, D, K, B]), capture_output=True,
                         text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    ids = json.loads(res.stdout.strip().splitlines()[-1])
    assert any(i.startswith("generic_solve_kernel") for i in ids) and not any(i.startswith("twisted_") for i in ids), \
        f"8-byte offset output launched {ids}"

    times, dfix = _batch(oracle, N, D, K, B, 8800)
    got, (prob, t_d, f_d) = _compare(solver, N, r, D, K, times, dfix, f"paired K3 stores B={B}")
    big = torch.full((B * K * D * N + 1,), float("nan"), dtype=torch.float64, device="cuda")
    out = big[1:].view(B, K, D, N)
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    solver.solve_linear(prob, t_d, f_d, coeffs=out, status=status)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    assert (status.cpu().numpy() == 0).all()
    ref = got[0].reshape(B, -1)
    err = np.abs(out.reshape(B, -1) - ref).max(axis=1) / np.abs(ref).max(axis=1)
    assert err.max() <= 1e-10, f"banded kernel vs paired form: {err.max():.3e}"
