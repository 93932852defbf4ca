"""Kernel attributes are shared by every handle of a process.

A kernel's dynamic shared memory limit (cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to the function, not to
the handle that set it, while each handle remembers what it has set.  One handle must therefore never lower the limit
below what another handle already relies on."""
import numpy as np
import pytest


def _solve(solver, N, r, K, D, B, seed):
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=seed)
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    out = solver.solve_linear(m.Problem(N, r, K, D), torch.from_numpy(times).cuda(),
                              torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda(), status=status)
    torch.cuda.synchronize()
    return out.cpu().numpy(), status.cpu().numpy()


@pytest.mark.gpu
def test_second_handle_does_not_lower_a_kernels_shared_memory_limit():
    """Handle a launches the persistent kernel v4 of (N, r, D) = (8, 3, 3) at K = 8, handle b the same kernel at K = 1
    (less shared memory), then a at K = 7: a's launch must still be allowed, and give b's bits."""
    import torch
    import mav_trajectory_generation_b200 as m
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (no CPU fallback exists)")
    a, b = m.Solver(0), m.Solver(0)
    try:
        for s in (a, b):
            s.set_option(m.capi.OPT_WAYPOINT_VARIANT, 4)
        N, r, D, B = 8, 3, 3, 64
        for solver, K in ((a, 8), (b, 1)):
            _, st = _solve(solver, N, r, K, D, B, 500 + K)
            assert (st == 0).all()
        out_a, st_a = _solve(a, N, r, 7, D, B, 507)
        out_b, st_b = _solve(b, N, r, 7, D, B, 507)
        assert (st_a == 0).all() and (st_b == 0).all()
        assert np.array_equal(out_a.view(np.uint8), out_b.view(np.uint8))
    finally:
        a.close()
        b.close()
