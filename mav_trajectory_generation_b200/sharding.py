"""Multi-GPU sharding of a trajectory batch (one process per GPU, torch.distributed).

The batch is embarrassingly parallel (each trajectory is a closed problem; reference
impl/polynomial_optimization_linear_impl.h:338-379 touches only its own members), so ranks own
contiguous slices and the solve itself needs NO collective.  A collective appears only when one rank
holds the whole batch (BASELINE.json config C5: "NCCL over NVLink only to scatter the vertex batch and
gather the solved coefficients"): `scatter_solve_gather` below.

Design of the exchange (NCCL has no native scatter/gather; these are grouped ncclSend/ncclRecv issued
through torch.distributed.batch_isend_irecv):

  * every rank's slice is cut into `chunks` pieces; step c of the pipeline is ONE NCCL group per rank that
    carries the inputs of piece c root->rank AND the coefficients of piece c-1 rank->root, so the root's
    NVLink egress (inputs) and ingress (coefficients) run full duplex and the solve of piece c overlaps
    the gather of piece c-1;
  * the root receives straight into slices of the preallocated [total][K][D][N] output (no staging
    tensors, no torch.cat) and sends straight from slices of its input tensors;
  * the root solves its own slice in place on its compute stream while the exchange progresses.

The same code runs on the gloo backend with CPU tensors, which is how the bookkeeping is tested without
GPUs (tests/test_sharding_gloo.py).
"""
import os

import torch
import torch.distributed as dist


def shard_bounds(total, world):
    """Contiguous, balanced slices: rank r owns [bounds[r], bounds[r+1])."""
    return [total * r // world for r in range(world + 1)]


def chunk_bounds(lo, hi, chunks):
    """Piece c of the slice [lo, hi) is [b[c], b[c+1])."""
    n = hi - lo
    return [lo + n * c // chunks for c in range(chunks + 1)]


def _wait_all(works):
    for w in works:
        w.wait()


def scatter_solve_gather(solve_fn, times_root, dfix_root, out_root, total, K, D, N, n_fixed, device,
                         root=0, chunks=4, local_buffers=None):
    """BASELINE C5 data path.  On `root`: times_root [total][K], dfix_root [total][D][n_fixed] and the
    preallocated out_root [total][K][D][N]; other ranks pass None for the three.  solve_fn(times, d_fixed,
    coeffs) solves one contiguous piece into `coeffs` (asynchronously on the current stream).
    Returns out_root on the root, None elsewhere.  `local_buffers` (non-root): dict reused across calls."""
    world, rank = dist.get_world_size(), dist.get_rank()
    bounds = shard_bounds(total, world)
    if rank == root:
        works = []
        peers = [r for r in range(world) if r != root]
        pieces = {r: chunk_bounds(bounds[r], bounds[r + 1], chunks) for r in peers}
        for c in range(chunks + 1):
            ops = []
            for r in peers:
                b = pieces[r]
                if c < chunks and b[c + 1] > b[c]:
                    ops.append(dist.P2POp(dist.isend, times_root[b[c]:b[c + 1]], r))
                    ops.append(dist.P2POp(dist.isend, dfix_root[b[c]:b[c + 1]], r))
                if c >= 1 and b[c] > b[c - 1]:
                    ops.append(dist.P2POp(dist.irecv, out_root[b[c - 1]:b[c]], r))
            if ops:
                works += dist.batch_isend_irecv(ops)
            if c == 0 and bounds[root + 1] > bounds[root]:
                # the root's own slice: solved in place, concurrently with the exchange
                lo, hi = bounds[root], bounds[root + 1]
                solve_fn(times_root[lo:hi], dfix_root[lo:hi], out_root[lo:hi])
        _wait_all(works)
        return out_root
    lo, hi = bounds[rank], bounds[rank + 1]
    n = hi - lo
    buf = local_buffers if local_buffers is not None else {}
    if buf.get("n") != n or buf.get("shape") != (K, D, N, n_fixed):
        buf["t"] = torch.empty((n, K), dtype=torch.float64, device=device)
        buf["f"] = torch.empty((n, D, n_fixed), dtype=torch.float64, device=device)
        buf["c"] = torch.empty((n, K, D, N), dtype=torch.float64, device=device)
        buf["n"], buf["shape"] = n, (K, D, N, n_fixed)
    b = [x - lo for x in chunk_bounds(lo, hi, chunks)]
    works = []
    for c in range(chunks + 1):
        ops = []
        if c < chunks and b[c + 1] > b[c]:
            ops.append(dist.P2POp(dist.irecv, buf["t"][b[c]:b[c + 1]], root))
            ops.append(dist.P2POp(dist.irecv, buf["f"][b[c]:b[c + 1]], root))
        if c >= 1 and b[c] > b[c - 1]:
            ops.append(dist.P2POp(dist.isend, buf["c"][b[c - 1]:b[c]], root))
        if not ops:
            continue
        step = dist.batch_isend_irecv(ops)
        if c < chunks and b[c + 1] > b[c]:
            _wait_all(step)  # stream-ordered for NCCL: the solve below waits for piece c's inputs
            solve_fn(buf["t"][b[c]:b[c + 1]], buf["f"][b[c]:b[c + 1]], buf["c"][b[c]:b[c + 1]])
        else:
            works += step
    _wait_all(works)
    return None


def solve_scattered(solve_fn, times_root, dfix_root, total, K, D, N, n_fixed, device, root=0, chunks=4):
    """Convenience wrapper that allocates the output on the root (tests; bench.py preallocates)."""
    out = None
    if dist.get_rank() == root:
        out = torch.empty((total, K, D, N), dtype=torch.float64, device=device)
    return scatter_solve_gather(solve_fn, times_root, dfix_root, out, total, K, D, N, n_fixed, device, root=root,
                                chunks=chunks)


# ---- fused solve + gather over NVLink peer memory (no collective, no intermediate buffers) --------------------------
#
# The peer-memory form of "gather the solved coefficients": every rank maps the ROOT's output tensor into its own
# address space (CUDA IPC) and hands the solver a slice of it as the coefficient buffer -- the kernels' TMA tensor
# stores then travel over NVLink / NVSwitch straight into their final place in the root's HBM while the sweep of
# the following tiles continues.  The transfer overlaps the math tile by tile inside ONE kernel; there is no gather
# step, no staging copy and no NCCL call on the data path (torch.distributed only carries the 64-byte IPC handle
# once, and the barrier).  Inputs go the other way with one DMA per rank (peer copy of its contiguous slice).
# The mapping is opened through the C-ABI (mtg_ipc_import) with the RANK's device current, which is what makes the
# root's memory addressable from this rank's kernels (torch's own IPC rebuild opens it under the owner's device).

_ipc_open = {}  # IPC handle bytes -> [base pointer, reference count]: a handle may be opened once per process


class PeerBuffer:
    """A device buffer of rank `root`, addressable from this rank: `.ptr` is a raw device pointer (the root's own
    tensor on the root, an NVLink peer mapping elsewhere).  Keep the root tensor alive while mappings exist."""

    def __init__(self, solver, tensor, root=0):
        rank = dist.get_rank()
        payload = [solver.ipc_export(tensor) if rank == root else None]
        dist.broadcast_object_list(payload, src=root)
        self.solver = solver
        self.tensor = tensor if rank == root else None
        self.base = None
        if rank == root:
            self.ptr = tensor.data_ptr()
        else:
            handle, offset = payload[0]
            ent = _ipc_open.get(handle)
            if ent is None:  # opened with THIS rank's device current
                _, base = solver.ipc_import(handle, 0)
                ent = _ipc_open[handle] = [base, 0]
            ent[1] += 1
            self.base, self.handle = ent[0], handle
            self.ptr = ent[0] + offset

    def close(self):
        if self.base is not None:
            ent = _ipc_open[self.handle]
            ent[1] -= 1
            if ent[1] == 0:
                self.solver.ipc_close(ent[0])
                del _ipc_open[self.handle]
            self.base = None


def peer_solve_into_root(solver, prob, times_pb, dfix_pb, out_pb, total, device, root=0, local_buffers=None):
    """One step of the fused path: every rank pulls its input slice from the root with one peer DMA per array, then
    solves with `coeffs` pointing INTO the root's output buffer (PeerBuffer) -- the kernels' TMA stores are the
    gather.  The caller brackets steps with a barrier + synchronize."""
    world, rank = dist.get_world_size(), dist.get_rank()
    bounds = shard_bounds(total, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    n = hi - lo
    if n <= 0:
        return
    K, D, N, nf = prob.K, prob.D, prob.N, prob.n_fixed
    stream = torch.cuda.current_stream(device).cuda_stream
    out_ptr = out_pb.ptr + lo * K * D * N * 8
    if rank == root:
        solver.solve_linear_ptr(prob, n, times_pb.ptr + lo * K * 8, dfix_pb.ptr + lo * D * nf * 8, out_ptr, stream)
        return
    buf = local_buffers if local_buffers is not None else {}
    if buf.get("n") != n:
        buf["t"] = torch.empty((n, K), dtype=torch.float64, device=device)
        buf["f"] = torch.empty((n, D, nf), dtype=torch.float64, device=device)
        buf["n"] = n
    solver.memcpy_d2d(buf["t"].data_ptr(), times_pb.ptr + lo * K * 8, n * K * 8, stream)          # peer DMA, NVLink
    solver.memcpy_d2d(buf["f"].data_ptr(), dfix_pb.ptr + lo * D * nf * 8, n * D * nf * 8, stream)
    solver.solve_linear_ptr(prob, n, buf["t"].data_ptr(), buf["f"].data_ptr(), out_ptr, stream)    # stores land at the root


def peer_dma_solve_gather(solver, prob, times_pb, dfix_pb, out_pb, total, device, root=0, chunks=4,
                          local_buffers=None):
    """Scatter / solve / gather with the copy engines doing the exchange (no collective, no SM time spent on the
    transfer): every rank cuts its slice into `chunks` pieces and runs a three-stream pipeline
        copy-in stream : peer DMA PULL of piece c's inputs from the root
        compute stream : solve piece c into a local buffer (full-rate local TMA stores)
        copy-out stream: peer DMA PUSH of piece c's coefficients into their final place in the root's output
    so the root's NVLink ingress carries full-size write packets from all peers while the solves and the input pulls
    overlap it.  The root solves its own slice in place.  Events order the three streams; the call returns with
    everything joined on the current stream (the caller brackets steps with a barrier + synchronize)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    bounds = shard_bounds(total, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    n = hi - lo
    if n <= 0:
        return
    K, D, N, nf = prob.K, prob.D, prob.N, prob.n_fixed
    cur = torch.cuda.current_stream(device)
    if rank == root:
        solver.solve_linear_ptr(prob, n, times_pb.ptr + lo * K * 8, dfix_pb.ptr + lo * D * nf * 8,
                                out_pb.ptr + lo * K * D * N * 8, cur.cuda_stream)
        return
    buf = local_buffers if local_buffers is not None else {}
    if buf.get("n") != n or "c" not in buf:
        buf["t"] = torch.empty((n, K), dtype=torch.float64, device=device)
        buf["f"] = torch.empty((n, D, nf), dtype=torch.float64, device=device)
        buf["c"] = torch.empty((n, K, D, N), dtype=torch.float64, device=device)
        buf["n"] = n
    if "s_in" not in buf:
        buf["s_in"], buf["s_out"] = torch.cuda.Stream(device), torch.cuda.Stream(device)
    s_in, s_out = buf["s_in"], buf["s_out"]
    s_in.wait_stream(cur)   # the previous step's solves have read the input buffers
    s_out.wait_stream(cur)
    b = chunk_bounds(0, n, chunks)
    row_t, row_f, row_c = K * 8, D * nf * 8, K * D * N * 8
    for c in range(chunks):
        a, e = b[c], b[c + 1]
        if e <= a:
            continue
        solver.memcpy_d2d(buf["t"].data_ptr() + a * row_t, times_pb.ptr + (lo + a) * row_t, (e - a) * row_t, s_in.cuda_stream)
        solver.memcpy_d2d(buf["f"].data_ptr() + a * row_f, dfix_pb.ptr + (lo + a) * row_f, (e - a) * row_f, s_in.cuda_stream)
        ev_in = torch.cuda.Event()
        ev_in.record(s_in)
        cur.wait_event(ev_in)
        solver.solve_linear_ptr(prob, e - a, buf["t"].data_ptr() + a * row_t, buf["f"].data_ptr() + a * row_f,
                                buf["c"].data_ptr() + a * row_c, cur.cuda_stream)
        ev_solved = torch.cuda.Event()
        ev_solved.record(cur)
        s_out.wait_event(ev_solved)
        solver.memcpy_d2d(out_pb.ptr + (lo + a) * row_c, buf["c"].data_ptr() + a * row_c, (e - a) * row_c, s_out.cuda_stream)
    cur.wait_stream(s_out)


# ---- host side: NUMA placement of a rank's pinned buffers ------------------------------------------------

def gpu_numa_node(index):
    """NUMA node of CUDA device `index` from sysfs (None when unknown / single node)."""
    try:
        p = torch.cuda.get_device_properties(index)
        path = "/sys/bus/pci/devices/%04x:%02x:%02x.0/numa_node" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
        with open(path) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


def _parse_cpulist(text):
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        a, _, b = part.partition("-")
        cpus.update(range(int(a), int(b or a) + 1))
    return cpus


def bind_to_gpu_numa_node(index):
    """Restrict this process to the CPUs of the GPU's NUMA node, so that pinned host buffers allocated
    afterwards are first-touched on that node and the H2D/D2H copies do not cross the inter-socket link.
    Returns (node, previous affinity set) -- pass the set to os.sched_setaffinity(0, .) to undo -- or
    (None, None) when nothing was changed."""
    node = gpu_numa_node(index)
    if node is None:
        return None, None
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        prev = os.sched_getaffinity(0)
        want = cpus & prev
        if not want or want == prev:
            return node, None
        os.sched_setaffinity(0, want)
        return node, prev
    except Exception:
        return None, None
