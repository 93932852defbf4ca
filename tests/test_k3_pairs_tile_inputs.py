"""The paired chunked kernel's tile input buffer, filled both ways, against the one-warp K3.

twisted_chunked_pair_kernel reads every input of a tile from one shared-memory buffer that holds the tile's
seg_times[16][K] and d_fixed[16][D][n_fixed] as they lie in global memory.  A whole tile with 16-byte aligned inputs
arrives by two bulk copies; the ragged last tile, and every tile of inputs that are only 8-byte aligned, arrive by
per-lane 8-byte copies into the same layout.  Each case is bitwise equal to the one-warp K3 (WAYPOINT_VARIANT = 5),
with status 0:
  * whole tiles only (bulk copies), at the headline K = 16 and at odd K = 15;
  * a ragged last tile, B = 16k + 1 ... 16k + 15;
  * inputs offset by 8 bytes, so that every tile takes the per-lane copies, with whole and ragged batches;
  * blocks parked (forced chunk 3) beside both kinds of fill.
Every batch has at least three tiles per pair at up to four pairs per SM (the most the kernel's registers allow), so
that the buffer and its refill are reused.  Each case proves by name, from a child process (as in test_k3_pairs.py),
which kernel ran: the default route of N = 10, r = 4, D = 3 at K = 15 and 16 is twisted_chunked_pair_kernel<10,4,3,3>.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_k3_pairs import _batch, _solve, pair_id
from test_large_k import same_bits
from test_resident_kernels import k3_id

N, R, D = 10, 4, 3
MAX_PAIRS_PER_SM = 4
TILES_PER_PAIR = 3
K3 = dict(WAYPOINT_VARIANT=5)

# (K, B % 16, inputs offset by 8 bytes, forced chunk or 0)
CASES = ([(16, 0, False, 0), (15, 0, False, 0)] + [(16, rem, False, 0) for rem in range(1, 16)] +
         [(15, 5, False, 0), (16, 0, True, 0), (16, 9, True, 0), (15, 0, True, 0), (16, 0, False, 3),
          (16, 11, True, 3)])


def _ids(case):
    K, rem, offset, chunk = case
    return f"K{K}-rem{rem}" + ("-offset8" if offset else "") + (f"-C{chunk}" if chunk else "")


# The child process: for each (K, B, options, offset), the ids of the kernels one solve_linear launched
_ROUTES = r"""
import json, sys
import torch
import mav_trajectory_generation_b200 as m
from test_resident_kernels import launched_kernels
s = m.Solver(0)
out = []
for N, r, D, K, B, opts, offset in json.loads(sys.stdin.read()):
    prob = m.Problem(N, r, K, D)
    t = torch.ones(B * K + offset, dtype=torch.float64, device="cuda")[offset:].view(B, K)
    f = torch.zeros(B * D * prob.n_fixed + offset, dtype=torch.float64, device="cuda")[offset:].view(B, D, prob.n_fixed)
    for name, value in opts.items():
        s.set_option(getattr(m.capi, "OPT_" + name), value)
    _, ids = launched_kernels(lambda: s.solve_linear(prob, t, f))
    for name in opts:
        s.set_option(getattr(m.capi, "OPT_" + name), 0)
    out.append(ids)
print(json.dumps(out))
"""


def _batch_size(sms, rem):
    return TILES_PER_PAIR * MAX_PAIRS_PER_SM * sms * 16 + rem


def _opts(chunk):
    return dict(CHUNK_BLOCKS=chunk) if chunk else {}


def _calls(sms):
    out = []
    for K, rem, offset, chunk in CASES:
        B = _batch_size(sms, rem)
        out += [[N, R, D, K, B, _opts(chunk), int(offset)], [N, R, D, K, B, K3, int(offset)]]
    return out


@pytest.fixture(scope="module")
def routes():
    """the kernel ids of every call of this file, from one child process"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    calls = _calls(sms)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
    res = subprocess.run([sys.executable, "-c", _ROUTES], input=json.dumps(calls), capture_output=True, text=True,
                         env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    ids = json.loads(res.stdout.strip().splitlines()[-1])
    return dict(sms=sms, ids={json.dumps(c, sort_keys=True): i for c, i in zip(calls, ids)})


def _offset8(x):
    """a copy of x whose storage starts 8 bytes past a 16-byte boundary"""
    import torch
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    out = flat[1:].view(x.shape)
    out.copy_(x)
    assert out.data_ptr() % 16 == 8
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_tile_inputs_same_as_k3(solver, oracle, routes, case):
    import torch
    import mav_trajectory_generation_b200 as m
    K, rem, offset, chunk = case
    B = _batch_size(routes["sms"], rem)
    label = f"paired K3 tile inputs K={K} B={B} offset8={offset} chunk={chunk}"
    for opts, want in ((_opts(chunk), pair_id(N, R, D)), (K3, k3_id(N, R, D))):
        ids = routes["ids"][json.dumps([N, R, D, K, B, opts, int(offset)], sort_keys=True)]
        assert ids == [want], f"{label}: {opts or 'the default route'} launched {ids}, expected {want}"
    times, dfix = _batch(oracle, N, D, K, B, 8600 + 100 * K + 10 * rem + chunk + (5 if offset else 0))
    prob = m.Problem(N, R, K, D)
    t_d, f_d = torch.from_numpy(times).cuda(), torch.from_numpy(dfix).cuda()
    if offset:
        t_d, f_d = _offset8(t_d), _offset8(f_d)
    got = _solve(solver, prob, t_d, f_d, **_opts(chunk))
    ref = _solve(solver, prob, t_d, f_d, **K3)
    for what, a, b in zip(("coefficients", "d_free", "status"), got, ref):
        assert same_bits(a, b), f"{label}: {what} of the paired K3 differ from the one-warp K3"
    assert (got[2] == 0).all(), f"{label}: non-zero status"
    assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all(), label
