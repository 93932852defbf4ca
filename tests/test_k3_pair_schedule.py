"""The schedule of the paired chunked kernel (twisted_chunked_pair_kernel), walked on the host.

The kernel runs two warps per CTA: the inward warp runs tile j's inward sweep while the outward warp runs tile j-1's
outward sweep, on one tile's C resident vertex blocks in shared memory and a parking area with one half per tile
parity.  The model below restates, operation by operation, what each warp reads and writes in the storage the two
share (resident slots with their segment times, the two parking halves, the handoff) and its mbarrier handshakes
and cp.async refills, as mtg_twisted_chunked_kernel.cuh does.  Every resident or parked block carries a tag (tile,
vertex).  The two warps are interleaved by several policies (one warp as far ahead as it can go, the other, and
seeded random choices), a refill's global read and shared write may happen anywhere between its issue and the
wait that retires it, and the walk checks that
  * every read finds the tag the kernel means to read: nothing is read before it is written or after it has been
    overwritten, and no refill lands in a slot the other warp writes meanwhile;
  * every mbarrier wait is met by an arrival, no side runs two phases ahead of the other's wait, and both warps run
    to the end (no deadlock).
"""
import random

import pytest


class Violation(Exception):
    pass


def inward_ops(K, C, tiles):
    """operations of the inward warp (the kernel's `if (inward)` branch), in program order"""
    n = (K + 1) // 2 - 1
    npark = n - C
    for j in range(tiles):
        for v in range(1, n + 1):
            if v <= npark:
                yield ("write", ("park", j & 1, v - 1), (j, v))
            else:
                b = slot_of(n, C, v, j)
                if j > 0:
                    yield ("wait", ("freed", b), j - 1)
                yield ("write", ("slot", b), (j, v))
        yield ("write", ("hand",), (j, "ed"))
        yield ("arrive", ("ready",))


def outward_ops(K, C, tiles):
    """operations of the outward warp, in program order; cp.async groups as ("commit", refill or None)"""
    n = (K + 1) // 2 - 1
    npark = n - C
    for j in range(tiles):
        yield ("commit", None)  # the final segment's inputs (private to this warp)
        yield ("wait", ("ready",), j)
        yield ("read", ("hand",), (j, "ed"))
        for v in range(n, 0, -1):
            b = slot_of(n, C, v, j)
            if v <= npark:
                yield ("wait_groups", min(max(C - 1, 0), 3))  # cp_async_wait_at_most(C - 1)
            yield ("read", ("slot", b), (j, v))
            if v - C >= 1:
                yield ("commit", (("park", j & 1, v - C - 1), ("slot", b), (j, v - C)))
            else:
                yield ("arrive", ("freed", b))
                yield ("commit", None)
        yield ("wait_groups", 0)


def slot_of(n, C, v, j):
    return (n - v) % C if j & 1 else (v - 1) % C


def walk(K, C, tiles, policy, seed=0):
    """run both warps under `policy` ("inward", "outward" or "random"); raises Violation"""
    rng = random.Random(seed)
    mem = {}
    inflight_dst = {}  # slot -> refill tag while a refill into it is in flight
    phases = {}        # barrier -> completed phases
    groups = []        # outward warp's cp.async groups not yet retired, oldest first
    warps = {"I": inward_ops(K, C, tiles), "O": outward_ops(K, C, tiles)}
    pending = {w: next(g, None) for w, g in warps.items()}

    def retire(keep):
        while len(groups) > keep:
            g = groups.pop(0)
            if g is None:
                continue
            src, dst, tag = g
            if mem.get(src) != tag:
                raise Violation(f"refill reads {src} after it was overwritten: {mem.get(src)} instead of {tag}")
            mem[dst] = tag
            del inflight_dst[dst]

    def ready(op):
        if op[0] == "wait":
            done = phases.get(op[1], 0)
            if done > op[2] + 1:
                raise Violation(f"{op[1]} ran two phases ahead of its wait for phase {op[2]}")
            return done == op[2] + 1
        return True

    def step(op):
        kind = op[0]
        if kind == "write":
            if op[1] in inflight_dst:
                raise Violation(f"write to {op[1]} while a refill into it is in flight")
            mem[op[1]] = op[2]
        elif kind == "read":
            if mem.get(op[1]) != op[2]:
                raise Violation(f"read of {op[1]} finds {mem.get(op[1])} instead of {op[2]}")
        elif kind == "arrive":
            phases[op[1]] = phases.get(op[1], 0) + 1
        elif kind == "commit":
            g = op[1]
            if g is not None:
                src, dst, tag = g
                if mem.get(src) != tag:
                    raise Violation(f"refill of {dst} issued before {src} holds {tag}")
                inflight_dst[dst] = tag
            groups.append(g)
        elif kind == "wait_groups":
            retire(op[1])

    while any(op is not None for op in pending.values()):
        runnable = [w for w, op in pending.items() if op is not None and ready(op)]
        if not runnable:
            raise Violation(f"deadlock: {pending}")
        if policy == "inward":
            w = "I" if "I" in runnable else "O"
        elif policy == "outward":
            w = "O" if "O" in runnable else "I"
        else:
            w = rng.choice(runnable)
        if w == "O" and policy == "random" and rng.random() < 0.3:
            retire(max(0, len(groups) - 1))  # a refill may land early, too
        step(pending[w])
        pending[w] = next(warps[w], None)
    if inflight_dst:
        raise Violation("refills still in flight at the end")


def chunks(K):
    n = (K + 1) // 2 - 1
    return sorted({c for c in range(1, 25) if c <= n + 1})


@pytest.mark.parametrize("K", range(3, 101))
def test_pair_schedule(K):
    for C in chunks(K):
        for tiles in (1, 2, 3):
            for policy, seed in (("inward", 0), ("outward", 0), ("random", 1), ("random", 2)):
                try:
                    walk(K, C, tiles, policy, seed)
                except Violation as e:
                    pytest.fail(f"K={K} C={C} tiles={tiles} {policy}/{seed}: {e}")


def test_pair_schedule_needs_an_inward_sweep():
    """at K = 2 there is no vertex to hand a slot over with, and the inward warp can run two tiles ahead; the
    planner does not pick the paired form there"""
    with pytest.raises(Violation):
        walk(2, 1, 3, "inward")


def test_model_catches_a_missing_handshake():
    """the walk is not vacuous: without the wait on a freed slot, the inward warp overwrites a resident block
    before the outward warp has read it"""
    real = inward_ops

    def no_wait(K, C, tiles):
        return (op for op in real(K, C, tiles) if op[0] != "wait")

    globals()["inward_ops"] = no_wait
    try:
        with pytest.raises(Violation):
            walk(16, 5, 2, "inward")
    finally:
        globals()["inward_ops"] = real
